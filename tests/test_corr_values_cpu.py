"""The value-range models of tests/corr_values.py, pinned without a GPU: the bf16 split, the per-element tensor-core
bound on every catalogue class, the generators, and the non-finite footprint models against a brute-force dependency
scan of the fp64 restatement."""
import pytest
import torch

import corr_values as cv
import torch_ref

PRM = (4, 1, 4, 1, 2)            # pad, k, md, s1, s2: a small stand-in of FlowNetC's (20, 1, 20, 1, 2)
SHAPE = (2, 8, 6, 10)


def _gshape(shape, prm=PRM):
    kr, dr, oH, oW = torch_ref.corr_geometry(shape[2], shape[3], *prm)
    return (shape[0], (2 * dr + 1) ** 2, oH, oW)


def test_split_catalogue():
    """Every finite x splits into finite halves with |x - hi - lo| <= max(2^-16 |x|, 2^-134); +-inf splits into
    (+-max bf16, +-inf), NaN into NaN."""
    bits = cv.catalogue_bits()
    x = cv.f32_from_bits(bits)
    hi, lo = cv.split_bf16(x)
    fin = torch.isfinite(x)
    assert bool(torch.isfinite(hi[fin]).all() and torch.isfinite(lo[fin]).all())
    err = (x.double() - hi.double() - lo.double()).abs()[fin]
    lim = torch.maximum(2.0 ** -16 * x.double().abs()[fin], torch.full_like(err, 2.0 ** -134))
    assert bool((err <= lim).all()), float((err / lim).max())
    inf = torch.isinf(x)
    bmax = float(torch.tensor(0x7F7F, dtype=torch.int16).view(torch.bfloat16))
    assert bool((hi[inf].float() == torch.sign(x[inf]) * bmax).all() and (lo[inf].float() == x[inf]).all())
    nan = torch.isnan(x)
    assert bool(torch.isnan(hi[nan].float()).all())
    # the saturation changes no bit of the split of a finite value outside the window
    mag = bits & 0x7FFFFFFF
    win = (mag >= cv.WINDOW[0]) & (mag <= cv.WINDOW[1])
    h0, l0 = cv.split_bf16(x, clamp=False)
    keep = ~win & fin
    assert torch.equal(h0[keep].view(torch.int16), hi[keep].view(torch.int16))
    assert torch.equal(l0[keep].view(torch.int16), lo[keep].view(torch.int16))
    # the relative bound alone fails below about 2^-118 (lo a bf16 subnormal): the absolute term is needed
    rel = (x.double() - hi.double() - lo.double()).abs() > 2.0 ** -16 * x.double().abs()
    assert bool(rel[fin].any())
    assert float(x.double().abs()[fin & rel].max()) < 2.0 ** -117


def test_split_window_negative_control():
    """Plain rn breaks finiteness exactly on the overflow window: every pattern of [0x7F7F8000, 0x7F7FFFFF] and its
    negative, and no other finite value."""
    allw = torch.arange(cv.WINDOW[0] - 0x10000, cv.WINDOW[1] + 1, dtype=torch.int64)
    allw = torch.cat([allw, allw | (1 << 31), cv.catalogue_bits()])
    x = cv.f32_from_bits(allw)
    fin = torch.isfinite(x)
    h0, l0 = cv.split_bf16(x, clamp=False)
    broken = fin & ~(torch.isfinite(h0.float()) & torch.isfinite(l0.float()))
    mag = allw & 0x7FFFFFFF
    win = (mag >= cv.WINDOW[0]) & (mag <= cv.WINDOW[1])
    assert torch.equal(broken, win & fin)
    assert int(win.sum()) >= 2 * 0x8000
    # the emulated products of a window value and 2^-20 are NaN with plain rn, finite and close with the fix
    y = torch.full_like(x, 2.0 ** -20)
    assert bool(torch.isnan((lambda hx, lx: hx.double() * 2.0 ** -20 + lx.double() * 2.0 ** -20)(h0, l0)[win]).all())
    got = cv.tc_emulate(x[win], y[win])
    ref = x[win].double() * 2.0 ** -20
    assert bool(((got - ref).abs() <= 3 * 2.0 ** -16 * ref.abs()).all())


@pytest.mark.parametrize("cls", cv.CLASSES)
def test_tc_bound_on_emulation(cls):
    """The per-element bound holds for the emulated hh + hl + lh, summed in fp64, on every catalogue class: forward
    (out = sum_c tc(a, b) / C) and both gradients."""
    a, b, go = cv.make(cls, SHAPE, _gshape(SHAPE), 5)
    C = SHAPE[1]
    ha, la = (t.double() for t in cv.split_bf16(a))
    hb, lb = (t.double() for t in cv.split_bf16(b))
    hg, lg = (t.double() for t in cv.split_bf16(go))
    ref = torch_ref.correlation64(a.double(), b.double(), *PRM)
    emu = (torch_ref.correlation64(ha, hb, *PRM) + torch_ref.correlation64(ha, lb, *PRM) +
           torch_ref.correlation64(la, hb, *PRM))
    if cls == "overflow":
        assert bool(torch.isinf(ref.float()[ref != 0]).all()), "overflow class: every non-zero output is +-inf in fp32"
        return
    lim = cv.bound_tc_forward(a, b, PRM)
    assert bool(torch.isfinite(emu).all())
    assert bool(((emu - ref).abs() <= lim).all()), float(((emu - ref).abs() / lim).max())
    refs = torch_ref.correlation64_backward(a.double(), b.double(), go.double(), *PRM)
    emus = [x + y + z for x, y, z in zip(torch_ref.correlation64_backward(ha, hb, hg, *PRM),
                                          torch_ref.correlation64_backward(la, lb, hg, *PRM),
                                          torch_ref.correlation64_backward(ha, hb, lg, *PRM))]
    lims = cv.bound_tc_backward(a, b, go, PRM)
    for e, r, l in zip(emus, refs, lims):
        assert bool(torch.isfinite(e).all())
        assert bool(((e - r).abs() <= l).all()), float(((e - r).abs() / l).max())
    if cls == "exact":
        assert torch.equal(emu, ref) and torch.equal(emus[0], refs[0]) and torch.equal(emus[1], refs[1])
    # on ordinary data the model's bound is never looser than the closed-form kappa's split term (3 2^-16 (1 + 2^-7) S)
    if cls in ("scale", "cancel"):
        S = torch_ref.correlation64(a.double().abs(), b.double().abs(), *PRM)
        kap = (3 * 2.0 ** -16 * (1 + 2.0 ** -7) + 2 * (3 * C + 3) * 2.0 ** -24) * S + cv.eta_tc(C)
        assert bool((lim <= kap * (1 + 1e-12)).all())


def test_generators_hit_their_class():
    shp, gs = (2, 64, 8, 12), _gshape((2, 64, 8, 12))
    a, b, go = cv.make("exact", shp, gs, 1)
    for t in (a, b, go):
        assert torch.equal(cv.split_bf16(t)[1].float(), torch.zeros_like(t))
    ref = torch_ref.correlation64(a.double(), b.double(), *PRM) * 64
    assert torch.equal(ref, ref.float().double()), "exact class: every sum is exact in fp32"
    g1, g2 = torch_ref.correlation64_backward(a.double(), b.double(), go.double(), *PRM)
    assert torch.equal(g1 * 64, (g1 * 64).float().double()) and torch.equal(g2 * 64, (g2 * 64).float().double())
    a, b, go = cv.make("huge", shp, gs, 1)
    mag = cv.bits_of(a) & 0x7FFFFFFF
    assert bool(((mag >= cv.WINDOW[0]) & (mag <= cv.WINDOW[1])).float().mean() > 0.3)
    assert bool((a < 0).any() and (a > 0).any()) and float(b.abs().max()) <= 2.0 ** -30
    a, b, go = cv.make("huge_go", shp, gs, 1)
    mag = cv.bits_of(go) & 0x7FFFFFFF
    assert bool(((mag >= cv.WINDOW[0]) & (mag <= cv.WINDOW[1])).all())
    a, b, go = cv.make("subnormal", shp, gs, 1)
    assert bool(((a != 0) & (a.abs() < 2.0 ** -126)).all())
    prods = (a.double() * b.double()).abs()
    assert bool((prods < 2.0 ** -149).any()), "some products underflow fp32"
    a, b, go = cv.make("tiny", shp, gs, 1)
    assert float(a.abs().max()) < 2.0 ** -99 and float(a.abs().min()) >= 2.0 ** -126
    a, b, go = cv.make("scale", shp, gs, 1)
    e = torch.log2(a.abs().double().clamp_min(1e-300)).mean((0, 2, 3))
    assert float(e.max() - e.min()) > 60
    a, b, go = cv.make("cancel", shp, gs, 1)
    assert torch.equal(a[:, 0], a[:, 1]) and torch.equal(b[:, 0], -b[:, 1]) and float(a[:, 0].abs().max()) > 2.0 ** 16
    a, b, go = cv.make("overflow", shp, gs, 1)
    p = (a[:, :1].double() * b[:, :1].double()).abs()
    assert float(p.min()) >= 2 * 3.4028234663852886e38 and float(p.max()) < 2 ** 8 * 3.4028234663852886e38


PROBE_PRM = [PRM, (2, 1, 4, 1, 2), (3, 3, 2, 1, 1)]


@pytest.mark.parametrize("prm", PROBE_PRM, ids=["pad=md", "pad<md", "k3"])
def test_footprints_against_scan(prm):
    """The reference footprint (the fp64 restatement's non-finite mask with one inf input) equals a brute-force scan
    that perturbs the element and sees which outputs move, once the scan counts the padding taps, which the
    restatement multiplies (inf * 0 = NaN); the in-image reach is the scan without them."""
    shp = (1, 3, 7, 9)
    gs = _gshape(shp, prm)
    g = torch.Generator().manual_seed(3)
    a, b, go = (torch.randn(s, generator=g, dtype=torch.float64) for s in (shp, shp, gs))
    for which, pos in (("a", (0, 1, 3, 4)), ("b", (0, 2, 0, 8)), ("go", (0, gs[1] // 2, gs[2] - 1, 0))):
        t = {"a": a, "b": b, "go": go}
        pert = {k: v.clone() for k, v in t.items()}
        pert[which][pos] += 1.0
        moved_f = torch_ref.correlation64(pert["a"], pert["b"], *prm) != torch_ref.correlation64(a, b, *prm)
        moved_b = [x != y for x, y in zip(torch_ref.correlation64_backward(pert["a"], pert["b"], pert["go"], *prm),
                                          torch_ref.correlation64_backward(a, b, go, *prm))]
        fwd, g1, g2 = cv.inimage_reach(which, shp, gs, pos, prm)
        if fwd is not None:
            assert torch.equal(fwd, moved_f)
        assert torch.equal(g1, moved_b[0]) and torch.equal(g2, moved_b[1])
        inf = {k: v.clone() for k, v in t.items()}
        inf[which][pos] = float("inf")
        rm = cv.ref_mask_backward(inf["a"], inf["b"], inf["go"], prm)
        assert bool((g1 <= rm[0]).all() and (g2 <= rm[1]).all()), "the reference reaches at least the in-image partners"
        if which != "go":
            rf = cv.ref_mask_forward(inf["a"], inf["b"], prm)
            assert bool((fwd <= rf).all())
        if prm[0] == prm[2] and which != "go":
            tm = cv.tiled_backward_mask(inf["a"], inf["b"], inf["go"], prm)
            assert torch.equal(tm[0], rm[0]) and torch.equal(tm[1], rm[1]), "at pad = md the tiled model is the reference"


def test_tiled_model_pad_lt_md_is_wider():
    """At pad < md the tiled backward's model reaches input pixels that have no output (the reference does not)."""
    prm = (2, 1, 4, 1, 2)
    shp = (1, 2, 8, 12)
    gs = _gshape(shp, prm)
    g = torch.Generator().manual_seed(4)
    a, b, go = (torch.randn(s, generator=g, dtype=torch.float64) for s in (shp, shp, gs))
    b[0, 1, 0, 6] = float("inf")
    rm = cv.ref_mask_backward(a, b, go, prm)
    tm = cv.tiled_backward_mask(a, b, go, prm)
    assert bool((rm[0] <= tm[0]).all()) and int(tm[0].sum()) > int(rm[0].sum())


def test_tc_superset_model():
    """The tensor-core superset contains the reference footprint of an input1 / input2 element at every placement,
    and, for the dead-halo placement, leaves out the pixels of the warpgroup whose dead unit holds the element."""
    shp = (1, 64, 34, 70)
    pos = cv.probe_positions(shp)
    prm = (20, 1, 20, 1, 2)
    gs = _gshape(shp, prm)
    for name, p in pos.items():
        for which in ("a", "b"):
            _, g1, g2 = cv.inimage_reach(which, shp, gs, p, prm)
            sup = cv.tc_backward_superset(which, shp, p)
            reach = g2 if which == "a" else g1
            assert bool((reach <= sup).all()), (name, which)
    n, c, y, x = pos["dead_halo"]
    sup = cv.tc_backward_superset("b", shp, pos["dead_halo"])
    assert not bool(sup[n, c, 0:8:2, 0:32:2].any()), "warpgroup 0 of tile (0, 0) is not reached through its dead unit"
    assert bool(sup[n, c, 8:16:2, 0:32:2].all()), "warpgroup 1 of tile (0, 0) is"
    n, c, y, x = pos["out_of_band"]
    _, g1, _ = cv.inimage_reach("b", shp, gs, pos["out_of_band"], prm)
    sup = cv.tc_backward_superset("b", shp, pos["out_of_band"])
    assert bool(sup[n, c, 0, 0]) and not bool(g1[n, c, 0, 0])
