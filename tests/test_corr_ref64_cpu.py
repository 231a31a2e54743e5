"""CPU pins of the fp64 restatements the GPU tests judge the FP32-FMA correlation and ChannelNorm kernels against
(tests/torch_ref.py): correlation64 / correlation64_backward over the reference's parameter space, the deliberately
wrong variants used as negative controls, and the fp32 / 16-bit ChannelNorm restatements."""
import glob
import os

import numpy as np
import pytest
import torch

import torch_ref
from oracle import cpu as orc

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
U = 2.0 ** -24

# (B, C, H, W, pad, k, md, s1, s2): every kernel_size, stride1 and stride2 the GPU catalogue uses, md 0 (D = 1) and
# md < s2 (D = 1), pad 0, pad < md, pad = md and pad > md + kr (outputs whose every tap is in the padding)
CATALOGUE = [
    (1, 6, 10, 9, 4, 3, 4, 1, 2), (2, 5, 8, 6, 3, 1, 3, 1, 1), (1, 33, 7, 8, 6, 1, 4, 1, 2),
    (1, 4, 12, 13, 2, 1, 4, 1, 2), (1, 3, 8, 8, 5, 1, 5, 1, 2), (2, 3, 9, 11, 1, 3, 4, 1, 2),
    (1, 2, 13, 12, 0, 5, 3, 1, 1), (1, 3, 8, 9, 3, 2, 3, 1, 2), (1, 3, 11, 13, 4, 1, 4, 2, 2),
    (1, 2, 14, 15, 5, 3, 4, 3, 1), (1, 4, 9, 10, 7, 1, 5, 1, 3), (1, 3, 5, 6, 2, 1, 0, 1, 1),
    (2, 1, 6, 7, 2, 1, 1, 1, 2), (1, 9, 10, 13, 10, 5, 7, 1, 3), (1, 4, 9, 12, 8, 5, 5, 1, 2),
    (1, 5, 12, 13, 5, 3, 3, 2, 1), (1, 4, 13, 14, 3, 1, 3, 3, 3), (1, 9, 11, 10, 6, 2, 5, 3, 2),
]
IDS = ["B%d-C%d-%dx%d-pad%d-k%d-md%d-s%d-%d" % c for c in CATALOGUE]


def _inputs(B, C, H, W, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(B, C, H, W, generator=g).double(), torch.randn(B, C, H, W, generator=g).double(), g


def _k2(prm):
    return prm[1] ** 2


@pytest.mark.parametrize("case", CATALOGUE, ids=IDS)
def test_correlation64_vs_autograd_and_oracle(case):
    """Against fp64 autograd through torch_ref.correlation (to fp64 rounding), and against the C oracle within the bound
    of its fp32 sums, 2 (n + 2) 2^-24 S with n = k^2 C products per output (k^2 D per gradient) and S the restatement of
    |a|, |b|, |g|; elements whose S is 0 must be 0 in both."""
    B, C, H, W = case[:4]
    prm = case[4:]
    a, b, g = _inputs(B, C, H, W, sum(case))
    out = torch_ref.correlation64(a, b, *prm)
    a_, b_ = a.clone().requires_grad_(), b.clone().requires_grad_()
    r = torch_ref.correlation(a_, b_, *prm)
    assert r.shape == out.shape and out.shape[2:] == torch.Size(torch_ref.corr_geometry(H, W, *prm)[2:])
    assert torch.allclose(out, r.detach(), rtol=1e-12, atol=1e-13)
    S = torch_ref.correlation64(a.abs(), b.abs(), *prm)
    o = orc.correlation_forward(a.float().numpy(), b.float().numpy(), *prm)
    err = np.abs(o - out.numpy())
    assert (err <= 2 * (_k2(prm) * C + 2) * U * S.numpy()).all()
    assert (o[S.numpy() == 0] == 0).all()
    if prm[3] != 1:
        return
    go = torch.randn(out.shape, generator=g).double()
    g1, g2 = torch_ref.correlation64_backward(a, b, go, *prm)
    r.backward(go)
    assert torch.allclose(g1, a_.grad, rtol=1e-12, atol=1e-13) and torch.allclose(g2, b_.grad, rtol=1e-12, atol=1e-13)
    S1, S2 = torch_ref.correlation64_backward(a.abs(), b.abs(), go.abs(), *prm)
    o1, o2 = orc.correlation_backward(a.float().numpy(), b.float().numpy(), go.float().numpy(), *prm)
    D = out.size(1)
    for x, ref, s in ((o1, g1, S1), (o2, g2, S2)):
        assert (np.abs(x - ref.numpy()) <= 2 * (_k2(prm) * D + 2) * U * s.numpy()).all()
        assert (x[s.numpy() == 0] == 0).all()


@pytest.mark.parametrize("path", sorted(glob.glob(os.path.join(GOLDEN, "correlation_*.npz"))),
                         ids=lambda p: os.path.basename(p))
def test_correlation64_vs_reference_kernel_fixtures(path):
    """The reference's own kernels' results (tests/golden/make_golden.py), within the fp32 bound above."""
    z = np.load(path)
    prm = tuple(int(v) for v in z["params"])
    a, b = (torch.from_numpy(z[n]).double() for n in ("input1", "input2"))
    go = torch.from_numpy(z["grad_output"]).double()
    C = a.size(1)
    out = torch_ref.correlation64(a, b, *prm)
    S = torch_ref.correlation64(a.abs(), b.abs(), *prm)
    g1, g2 = torch_ref.correlation64_backward(a, b, go, *prm)
    S1, S2 = torch_ref.correlation64_backward(a.abs(), b.abs(), go.abs(), *prm)
    D = out.size(1)
    for name, ref, s, n in (("output", out, S, _k2(prm) * C), ("grad_input1", g1, S1, _k2(prm) * D),
                            ("grad_input2", g2, S2, _k2(prm) * D)):
        x = z[name]
        assert x.shape == tuple(ref.shape), name
        assert (np.abs(x - ref.numpy()) <= 2 * (n + 2) * U * s.numpy()).all(), name


def test_correlation64_known_answers():
    """Worked by hand."""
    a = torch.tensor([[[[1.0, 2.0], [3.0, 4.0]]]], dtype=torch.float64)
    b = torch.tensor([[[[5.0, 6.0], [7.0, 8.0]]]], dtype=torch.float64)
    # C = 1, 2x2, pad 1, md 1, s2 1: D = 9 planes of 2x2; plane (tj, ti) at (y, x) is a[y, x] b[y + tj, x + ti]
    out = torch_ref.correlation64(a, b, 1, 1, 1, 1, 1)
    assert out.shape == (1, 9, 2, 2)
    assert out[0, 4].tolist() == [[5.0, 12.0], [21.0, 32.0]]          # (0, 0)
    assert out[0, 8].tolist() == [[8.0, 0.0], [0.0, 0.0]]             # (1, 1): only a[0, 0] b[1, 1]
    assert out[0, 5].tolist() == [[6.0, 0.0], [24.0, 0.0]]            # (0, 1)
    assert out[0, 0].tolist() == [[0.0, 0.0], [0.0, 20.0]]            # (-1, -1): only a[1, 1] b[0, 0]
    # k = 2 (kr = 0: one tap) divides by k^2 C = 4: pad 0, md 0 -> D = 1, out = a * b / 4
    out = torch_ref.correlation64(a, b, 0, 2, 0, 1, 1)
    assert out.shape == (1, 1, 2, 2) and out[0, 0].tolist() == [[1.25, 3.0], [5.25, 8.0]]
    # md < s2: D = 1; two channels, divided by C = 2
    a2, b2 = torch.cat([a, 2 * a], 1), torch.cat([b, b], 1)
    out = torch_ref.correlation64(a2, b2, 1, 1, 1, 1, 2)
    assert out.shape == (1, 1, 2, 2) and out[0, 0].tolist() == [[7.5, 18.0], [31.5, 48.0]]
    g1, g2 = torch_ref.correlation64_backward(a2, b2, torch.ones(1, 1, 2, 2, dtype=torch.float64), 1, 1, 1, 1, 2)
    assert torch.equal(g1, b2 / 2) and torch.equal(g2, a2 / 2)
    # stride1 2 on a 5x5 input, pad 0, md 0: oH = oW = ceil(5 / 2) = 3, taps at 0, 2, 4
    x = torch.arange(25, dtype=torch.float64).view(1, 1, 5, 5)
    out = torch_ref.correlation64(x, torch.ones_like(x), 0, 1, 0, 2, 1)
    assert out.shape == (1, 1, 3, 3) and out[0, 0].tolist() == [[0, 2, 4], [10, 12, 14], [20, 22, 24]]

    # kernel_size 3, pad 1, md 0: output (0, 0)'s patch is centred on padded (0, 0) = input (-1, -1), not on input
    # (0, 0), so a[0, 0] b[0, 0] is its one tap inside; output (1, 1) sums all four products; both / 9
    out = torch_ref.correlation64(a, b, 1, 3, 0, 1, 1)
    assert out.shape == (1, 1, 2, 2)
    assert torch.allclose(out[0, 0], torch.tensor([[5.0, 17.0], [26.0, 70.0]], dtype=torch.float64) / 9, rtol=1e-15)
    o = orc.correlation_forward(a.float().numpy(), b.float().numpy(), 1, 3, 0, 1, 1)
    assert np.allclose(o[0, 0], out[0, 0].numpy(), rtol=1e-6)


# (variant, catalogue case on whose edge it acts)
VARIANT_CASES = [
    ("replicate", (1, 3, 8, 9, 3, 2, 3, 1, 2)), ("replicate", (1, 2, 13, 12, 0, 5, 3, 1, 1)),
    ("replicate", (1, 4, 12, 13, 2, 1, 4, 1, 2)), ("centre_br", (2, 3, 9, 11, 1, 3, 4, 1, 2)),
    ("norm_odd", (1, 3, 8, 9, 3, 2, 3, 1, 2)), ("drop_tail8", (1, 33, 7, 8, 6, 1, 4, 1, 2)),
    ("drop_tail64", (1, 70, 6, 8, 2, 1, 2, 1, 1)), ("drop_tail64", (1, 9, 10, 13, 10, 5, 7, 1, 3)),
    ("swap_planes", (1, 6, 10, 9, 4, 3, 4, 1, 2)), ("mirror2", (1, 4, 9, 10, 7, 1, 5, 1, 3)),
]


@pytest.mark.parametrize("variant,case", VARIANT_CASES, ids=["%s-%d" % (v, i) for i, (v, _) in enumerate(VARIANT_CASES)])
def test_variants_differ_only_on_their_edge(variant, case):
    """Each negative-control variant differs from the restatement somewhere on its edge (torch_ref.variant_edges) and
    is bit-equal to it everywhere else, in the forward and in both gradients."""
    B, C, H, W = case[:4]
    prm = case[4:]
    a, b, g = _inputs(B, C, H, W, 7 + sum(case))
    ref = torch_ref.correlation64(a, b, *prm)
    go = torch.randn(ref.shape, generator=g).double()
    refs = (ref,) + torch_ref.correlation64_backward(a, b, go, *prm)
    var = (torch_ref.correlation64(a, b, *prm, variant=variant),) + \
        torch_ref.correlation64_backward(a, b, go, *prm, variant=variant)
    masks = torch_ref.variant_edges(variant, a.shape, *prm)
    hit = False
    for what, r, v, m in zip(("forward", "grad1", "grad2"), refs, var, masks):
        assert torch.equal(r[~m], v[~m]), "%s: %s differs off its edge" % (variant, what)
        hit |= bool((r != v)[m].any())
    assert hit, "%s never differs on its edge" % variant


def test_replicate_edge_is_the_padding():
    """The replicate edge of a k = 1 forward with pad = md is the frame of outputs whose displacements reach the
    padding: all but the interior whose every shifted partner is inside."""
    fwd, g1, g2 = torch_ref.variant_edges("replicate", (1, 2, 12, 13), 4, 1, 4, 1, 2)
    # plane (0, 0) never reads padding; plane (tj, ti) = (2, 2) reads it for y or x >= H - 4
    assert not bool(fwd[0, 12].any())
    p = fwd[0, 24]
    assert bool(p[8:].all()) and bool(p[:, 9:].all()) and not bool(p[:8, :9].any())


# ------------------------------------------------------------------------------------------------
# ChannelNorm
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("shape", [(2, 3, 16, 24), (1, 2, 7, 9), (2, 3, 64, 128)])
def test_channelnorm16_vs_reference_kernel_fixtures(shape):
    """The 16-bit restatement reproduces the reference's own half kernels bit for bit, forward and backward, on the
    seeded inputs of tests/golden/make_golden.py (the backward from the recorded output)."""
    z = np.load(os.path.join(GOLDEN, "refk_channelnorm_half_%s.npz" % "x".join(map(str, shape))))
    x = torch.randn(*shape, generator=torch.Generator().manual_seed(35)).half()
    ro = torch.from_numpy(z["output"])
    assert torch.equal(torch_ref.channelnorm16(x), ro)
    go = torch.randn(*ro.shape, generator=torch.Generator().manual_seed(36)).half()
    assert torch.equal(torch_ref.channelnorm_backward32(x, ro, go), torch.from_numpy(z["grad_input"]))


def test_channelnorm_restatements_at_the_edges():
    """Squares that round away in the storage type, overflow, and the backward's divide by 1e-9f at a zero norm."""
    h = torch.tensor([[[[2.0 ** -13]], [[3.0]]]], dtype=torch.float16)     # (2^-13)^2 = 2^-26 < half's least subnormal
    assert torch.equal(torch_ref.channelnorm16(h), torch.tensor([[[[3.0]]]], dtype=torch.float16))
    h = torch.tensor([[[[2.0 ** -12]]]], dtype=torch.float16)               # 2^-24: the least subnormal survives
    assert float(torch_ref.channelnorm16(h)) == 2.0 ** -12
    h = torch.tensor([[[[256.0]], [[1.0]]]], dtype=torch.float16)           # 65536 overflows half
    assert float(torch_ref.channelnorm16(h)) == float("inf")
    # x != 0 with norm 0: g x / 1e-9f overflows half
    x = torch.tensor([[[[2.0 ** -13]]]], dtype=torch.float16)
    o = torch_ref.channelnorm16(x)
    assert float(o) == 0.0
    gi = torch_ref.channelnorm_backward32(x, o, torch.tensor([[[[-1.0]]]], dtype=torch.float16))
    assert float(gi) == float("-inf")
    # fp32: 2^-80 squares to 0, 1e20 to inf; 1.5 * 2^-75 squares to the least subnormal
    f = torch.tensor([[[[2.0 ** -80]], [[1.0]]]], dtype=torch.float32)
    assert float(torch_ref.channelnorm32(f)) == 1.0
    assert float(torch_ref.channelnorm32(torch.tensor([[[[1e20]]]]))) == float("inf")
    assert float(torch_ref.channelnorm32(torch.tensor([[[[1.5 * 2.0 ** -75]]]]))) == float(np.sqrt(np.float32(2.0 ** -149)))


def test_gpu_correlation_catalogue_covers_its_axes():
    """The catalogue of tests/test_gpu_corr_fp32_fp64.py reaches what its docstring claims: the tiled cases are all
    tiled-eligible (the host rule of correlation_tiled.cu) and span the listed offsets, channel counts and sizes; the
    generic ones span kernel_size, the strides, md, the pads and the channel-unroll tails."""
    import test_gpu_corr_fp32_fp64 as t
    configs = {(2, 10), (2, 4), (1, 4), (2, 2)}
    offs, Cs, Ws, oHs, Bs = set(), set(), set(), set(), set()
    for B, C, H, W, pad, k, md, s1, s2 in t.TILED:
        kr, dr, oH, oW = torch_ref.corr_geometry(H, W, pad, k, md, s1, s2)
        assert k == 1 and s1 == 1 and W % 4 == 0 and oW % 4 == 0 and (md - pad) % 4 == 0 and (s2, dr) in configs
        offs.add((s2, dr, md - pad))
        Cs.add(C)
        Ws |= {W, oW}
        oHs.add(oH if oH != s2 else "s2")
        Bs.add(B)
    assert {(s2, dr, o) for s2, dr in configs for o in (-4, 0, 4)} | {(2, 10, -8), (2, 10, 8)} <= offs
    assert {(pad, md, s2) for B, C, H, W, pad, k, md, s1, s2 in t.TILED if md % s2} == {(17, 21, 2), (13, 9, 2), (1, 5, 2)}
    assert {1, 7, 9, 16, 63, 65, 130} <= Cs and {4, 12, 124, 132, 260} <= Ws and {1, "s2", 7, 9, 17} <= oHs
    assert {1, 3} <= Bs
    G = t.GENERIC
    assert {c[5] for c in G} >= {1, 2, 3, 5} and {c[7] for c in G} >= {1, 2, 3} and {c[8] for c in G} >= {1, 2, 3}
    assert {c[6] for c in G} >= {0, 3, 5, 7} and (1, 2) in {(c[6], c[8]) for c in G}
    pads = {("0" if c[4] == 0 else "md-1" if c[4] == c[6] - 1 else "md" if c[4] == c[6] else
             "md+kr+1" if c[4] == c[6] + (c[5] - 1) // 2 + 1 else "other") for c in G}
    assert {"0", "md-1", "md", "md+kr+1"} <= pads
    assert {1, 3, 4, 5, 9} <= {c[1] for c in G}
    assert any(c[3] % 4 for c in G) and any((c[6] - c[4]) % 4 for c in G)
    for B, C, H, W, pad, k, md, s1, s2 in G:
        kr, dr, oH, oW = torch_ref.corr_geometry(H, W, pad, k, md, s1, s2)
        assert oH > 0 and oW > 0
