"""CPU tests of the two helpers of tests/test_gpu_corr_tc_schedule.py: the model of the tensor-core correlation's work
assignment (tests/corr_tc_schedule.py) and the explicit fp64 correlation (tests/torch_ref.py)."""
import numpy as np
import pytest
import torch

import corr_tc_schedule as sch
import torch_ref
from oracle import cpu as orc


@pytest.mark.parametrize("sms", [132, 114])
def test_each_regime_is_reached(sms):
    """The batch picked for each regime puts the forward schedule in that regime, and its CTAs run more than one tile
    in both directions wherever there are more tiles than SMs."""
    for name, (what, pred) in sch.REGIMES.items():
        B, H, W = sch.pick(name, sms)
        f = sch.Forward(sch.ntiles(B, H, W), sms)
        assert pred(f), "%s (%s) not reached by B=%d %dx%d" % (name, what, B, H, W)
        if f.nt > sms:
            assert f.tiles_per_cta() > 1 and sch.Backward(f.nt, sms, True, False).tiles_per_cta() > 1, name
            assert sch.Backward(f.nt, sms, False, True).tiles_per_cta() > 1, name


@pytest.mark.parametrize("sms", [132, 114, 7])
def test_forward_segments_cover_every_unit_once(sms):
    """For every tile count up to 1000, the modelled segments deal each (tile, unit) pair exactly once (the model
    asserts no pair twice), in ascending unit order within a segment, never running past a tile's last unit, and each
    CTA's partial-round share is `wper` consecutive pairs."""
    for nt in range(1, 1001):
        f = sch.Forward(nt, sms)
        assert len(f.owner) == nt * sch.NU, nt
        assert set(f.owner) == {(t, u) for t in range(nt) for u in range(sch.NU)}, nt
        for cta, segs in enumerate(f.segs):
            part = [s for s in segs if s[0] >= f.full]
            assert all(0 <= ua < ub <= sch.NU for _, ua, ub in segs), nt
            assert all(s[0] < f.full and s[1:] == (0, sch.NU) for s in segs[:len(segs) - len(part)]), nt
            assert sum(ub - ua for _, ua, ub in part) <= f.wper, nt
            for (t0, _, ub0), (t1, ua1, _) in zip(part, part[1:]):
                assert (t1, ua1) == (t0 + 1, 0) and ub0 == sch.NU, nt


@pytest.mark.parametrize("sms", [132, 114, 7])
def test_backward_tiles_cover_every_tile_once(sms):
    for nt in range(4, 1001, 4):
        for need1, need2 in ((True, True), (True, False), (False, True)):
            b = sch.Backward(nt, sms, need1, need2)
            want = {(g, t) for g in range(2) if (need1, need2)[g] for t in range(nt)}
            assert set(b.owner) == want, (nt, need1, need2)


def test_locate_names_the_tile_and_unit():
    # B = 38 at 132 SMs: tile 150 is in the partial round (full = 132); its units 0..1 are
    # pairs w = 126, 127 of the round, CTA 126 / wper = 63's share, after that CTA's whole tile 63
    f = sch.Forward(sch.ntiles(38, 16, 32), 132)
    nxt, nyt = sch.tile_grid(16, 32)
    n, py, px, yc0, xc0 = sch.decode(150, nxt, nyt)
    y, x = 2 * yc0 + py, 2 * xc0 + px
    assert sch.tile_of(n, y, x, nxt, nyt) == (150, 0)
    assert "tile 150 unit 0 CTA 63 segment 1 [units 0..1, partial round]" in sch.locate_forward(f, 16, 32, n, 0, y, x)
    # displacement row tj = 10 of tile row 6: unit (10 + 6) // 4 = 4
    s = sch.locate_forward(f, 16, 32, n, 10 * 21, y + 12, x)
    assert "unit 4" in s
    b = sch.Backward(f.nt, 132)
    assert "tile 150 warpgroup 1 CTA" in sch.locate_backward(b, 16, 32, 1, n, y + 12, x)


# ------------------------------------------------------------------------------------------------
# The explicit fp64 correlation
# ------------------------------------------------------------------------------------------------
# (B, C, H, W, pad, md, s2): FlowNetC's configuration on ragged (odd, not tile-multiple) shapes, C not a power of two,
# stride2 1, and pads smaller and larger than the displacement
SHAPES = [(2, 3, 7, 9, 20, 20, 2), (1, 5, 10, 6, 4, 4, 1), (2, 6, 9, 11, 6, 8, 2), (1, 3, 6, 5, 5, 4, 2)]


@pytest.mark.parametrize("shape", SHAPES, ids=["B%d-C%d-%dx%d-pad%d-md%d-s%d" % s for s in SHAPES])
def test_fp64_correlation_k1(shape):
    """Against fp64 autograd through torch_ref.correlation (to fp64 rounding), and against the CPU oracle within the
    bound of its fp32 sums: |oracle - ref| <= 2 (n + 2) 2^-24 S, n = the products in one sum and S the same sum over
    |a|, |b|, |g|."""
    B, C, H, W, pad, md, s2 = shape
    g = torch.Generator().manual_seed(C * 100 + H)
    a, b = torch.randn(B, C, H, W, generator=g).double(), torch.randn(B, C, H, W, generator=g).double()
    prm = (pad, 1, md, 1, s2)
    out = torch_ref.correlation64(a, b, pad, 1, md, 1, s2)
    go = torch.randn(out.shape, generator=g).double()
    g1, g2 = torch_ref.correlation64_backward(a, b, go, pad, 1, md, 1, s2)
    a_, b_ = a.clone().requires_grad_(), b.clone().requires_grad_()
    r = torch_ref.correlation(a_, b_, *prm)
    r.backward(go)
    assert r.shape == out.shape
    for x, ref in ((out, r.detach()), (g1, a_.grad), (g2, b_.grad)):
        assert torch.allclose(x, ref, rtol=1e-12, atol=1e-13)

    S = torch_ref.correlation64(a.abs(), b.abs(), pad, 1, md, 1, s2)
    S1, S2 = torch_ref.correlation64_backward(a.abs(), b.abs(), go.abs(), pad, 1, md, 1, s2)
    a32, b32, g32 = (t.float().numpy() for t in (a, b, go))
    o = orc.correlation_forward(a32, b32, *prm)
    o1, o2 = orc.correlation_backward(a32, b32, g32, *prm)
    D = out.size(1)
    for x, ref, s, n in ((o, out, S, C), (o1, g1, S1, D), (o2, g2, S2, D)):
        err = np.abs(x - ref.numpy())
        assert (err <= 2 * (n + 2) * 2.0 ** -24 * s.numpy()).all(), err.max()
        assert err.max() > 0                             # the oracle sums in fp32: the check is not vacuous
