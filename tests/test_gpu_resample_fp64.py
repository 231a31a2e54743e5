"""Resample2d and the fused warp-concat kernels, element by element, against tests/resample_ref64.py's fp64 restatement,
on flows that put pixels on the edges of the tap arithmetic, at tile-boundary geometries and on strided image layouts.

Every output is a view in a NaN-poisoned, guarded allocation (tests/guarded.py) and every workspace is exactly the size
the library reports.  Each case checks, element by element, |x - ref64| <= kappa S + ETA (ETA = 2^-140 covers roundings
into the subnormal range), then max|x - ref64| / max|ref64| <= GLOBAL_TOL per tensor.

kappa, with u = 2^-24 per fp32 rounding and gamma_k = k u / (1 - k u):
- forward, bilinear: w = fl(fl(1-a) fl(1-b)) is 3 roundings from the exact weight (a, b are exact); the value is one
  __fmul_rn and three __fmaf_rn, each rounding the running sum once, so |x - ref| <= gamma_7 S, S = sum w |I|.
- forward, nearest: a copy; bit-exact (kappa = 0).
- K7: per channel, the tap differences (1), the weights 1-b (1), their products (1) and sum (1), times g (1): 5 roundings
  of the |.| expression; C terms accumulated in fp32 (C).  kappa = gamma_{C+5}, S = sum_c |g_c| [(1-b)(|I_TR|+|I_TL|) +
  b(|I_BR|+|I_BL|)] (and the y analogue).
- K6: each contribution s * g is 4 roundings (1-at, 1-bt, their product, times g); the n contributions of a target are
  added by atomics in any order (n - 1 roundings of partial sums bounded by S), and the transpose into the planar
  gradient may add once more: kappa = gamma_{n+5}, n counted per target by the helper.
- the fused chain (derived in resample_ref64.warp_concat_backward): d = img0 - v has E_d = gamma_7 S_v + u(|img0|+|v|);
  n = |d| errs by E_n = ||E_d|| + gamma_{C+2} n; g_d = g_n d / (n + 1e-9) by |g_n| (E_d + |d| E_n / n) / n +
  gamma_4 |g_d|; g_v = g_w - g_d adds u(|g_w| + |g_d|); K7 of g_v carries E_gv through |D| and adds gamma_{C+5} S_K7;
  flow / flow_div and the |flow| term add gamma_1 and gamma_6 of themselves, and adding the parts gamma_3 of their
  |sum|.  The x4 adjoint sums <= 8 columns then <= 8 rows (or 16 pixels for nearest), <= 4 tile partials and scales by
  mul: gamma_21 (gamma_17) of the 64-term absolute sum on top of the propagated pixel bounds.  Pixels whose n is 0
  must give g_d = 0 exactly, and so grad_x[:, :C] equal gcat's x channels bit for bit there.

GLOBAL_TOL comes from the first passing run of this file, on an H100 80GB HBM3 (700 W power limit, driver 580.159.03;
30 cases, about 25 s).  The largest values over all cases were:

    quantity                      max |d| / (kappa S)   max|d| / max|ref64|
    forward                       0.433                 1.2e-7
    K7                            0.271                 8.1e-8
    K6                            0.332                 3.9e-7
    fused forward                 0.800                 1.0e-7
    FusionConcat forward          0.499                 6.1e-8
    FusionConcat grad_x           0.615                 1.5e-7
    FusionConcat g_sd / g_s2      0.068 / 0.063         1.4e-7 / 1.5e-7
    warp-concat grad_x            0.958                 1.0e-6
    warp-concat grad_flow full    0.401                 1.8e-7
    ... bilinear x4 adjoint       0.028                 2.0e-7
    ... nearest x4 adjoint        0.101                 2.5e-7

GLOBAL_TOL = 1e-5 is about 10 times the largest of them.  grad_x comes closest to its bound where the diff norm n is
small and g_d = g_n d / n amplifies the forward's rounding by 1 / n, which the bound carries.

Negative controls.  Each edge of resample_ref64's catalogue has a variant of the restatement that is wrong only there,
applied to one axis; it is judged only at the pixels whose coordinate on that axis is the edge (edge_hits), and it
"fires" when the kernel's output there is outside the bound of the variant (nearest: not bit-equal).  Every edge's
control must fire in at least one Resample2d case (test_report_ratios, which runs last, asserts it).  CONTROLS:

    -1-eps, -0.5, -eps, -2^-24       forward   right tap = clamped left tap + 1 (wrong left of 0: 1 instead of 0)
    -1, -big, -(2^24+2)              K7        the same; alpha = 0 there, so only K7 sees the right tap
    0, int                           K7        the left difference at an integer coordinate instead of the right one
    n-1-eps, n-1                     forward   clamp to n-2 instead of n-1 (an off-by-one at the upper clamp)
    n-1+eps, n, n+0.5, big, 2^24+2   forward   clamp with the image's dims instead of the flow's (image larger)
    alpha_tiny, alpha_1-2^-24        forward   fractions cut to 8 bits (2^-20 -> 0; 1 - 2^-24 -> 1 - 2^-8)
    half                             nearest   round half to even (2.5 -> 2, 0.5 -> 0)
    0.49999997                       nearest   floor(fp32(xf + 0.5f)) (rounds to 1)
    k+0.5-ulp                        nearest   the coordinate rounded to fp16 first (2.4999998 -> 2.5 -> 3)

The fused backward has one more: an adjoint that drops tile (0, 0)'s partial for the cells it shares with its
neighbours must be rejected on those cells.  The catalogue also reaches the fused kernels: full-resolution edge flows in
mode 0, and through the nearest upsample in mode 2 (each cell holds its top-left pixel's edge flow / 4, exact).

Bit-for-bit invariances: the Resample2d forward is identical in both runs (one per scatter); the Resample2d flow
gradient is identical across the two scatters and need1; the warp-concat flow gradient is identical in a repeat call,
with and without the image gradient, and for a sample alone and inside a batch.  Image gradients go through atomics and are
only bounded.
"""
import ctypes

import numpy as np
import pytest
import torch

import resample_ref64 as r64
from guarded import SENTINEL, Arena

pytestmark = pytest.mark.gpu
P = ctypes.c_void_p
GLOBAL_TOL = 1e-5
# the Resample2d image-gradient scatter, chosen by the workspace the backward is handed: the queried size (vector
# reductions into the interleaved scratch) or none (planar scalar reductions)
SCATTERS = ("vector", "planar")
STATS = {}
# edge of the catalogue -> (the output that shows it, the variant of the restatement that is wrong only there)
CONTROLS = {
    "-1-eps": ("fwd", "right_of_clamped"), "-0.5": ("fwd", "right_of_clamped"), "-eps": ("fwd", "right_of_clamped"),
    "-2^-24": ("fwd", "right_of_clamped"), "-1": ("k7", "right_of_clamped"), "-big": ("k7", "right_of_clamped"),
    "-(2^24+2)": ("k7", "right_of_clamped"), "0": ("k7", "k7_left"), "int": ("k7", "k7_left"),
    "n-1-eps": ("fwd", "clamp_short"), "n-1": ("fwd", "clamp_short"), "n-1+eps": ("fwd", "clamp_image"),
    "n": ("fwd", "clamp_image"), "n+0.5": ("fwd", "clamp_image"), "big": ("fwd", "clamp_image"),
    "2^24+2": ("fwd", "clamp_image"), "alpha_tiny": ("fwd", "frac_fixed8"), "alpha_1-2^-24": ("fwd", "frac_fixed8"),
    "half": ("nearest", "half_even"), "0.49999997": ("nearest", "half_f32"), "k+0.5-ulp": ("nearest", "coord_f16"),
}
FIRED, RS_RUN = {}, []


def _f2():
    import flownet2_b200
    return flownet2_b200


def _p(t):
    return P(t.data_ptr()) if t is not None else P(0)


def _st():
    return P(torch.cuda.current_stream().cuda_stream)


def _strides(t):
    return (ctypes.c_int64 * 4)(*t.stride())


def _where_tile(i, py, extra=""):
    b, y, x = i[0], i[-2], i[-1]
    return "sample %d pixel (y %d, x %d), tile (bx %d, by %d) at PY %d%s" % (b, y, x, x // 32, y // (8 * py), py, extra)


def _check(x, ref, E, what, where, stats):
    d = (x.double() - ref).abs()
    lim = E + r64.ETA
    bad = d > lim
    if bool(bad.any()):
        i = tuple(int(v) for v in bad.nonzero()[0])
        pytest.fail("%s: %d elements beyond kappa S; the first at %s (%s): |d| = %.3e, bound %.3e, ref %.9e, got %.9e" % (
            what, int(bad.sum()), i, where(i), float(d[i]), float(lim[i]), float(ref[i]), float(x[i])))
    key = what.split(" ")[0]
    ratio = float(torch.where(E > 0, d / E.clamp_min(1e-300), torch.zeros_like(d)).max())
    glob = float(d.max() / ref.abs().max().clamp_min(1e-300))
    assert glob <= GLOBAL_TOL, "%s: max|d|/max|ref| = %.3e > %.1e" % (what, glob, GLOBAL_TOL)
    s = stats.setdefault(key, [0.0, 0.0])
    s[0], s[1] = max(s[0], ratio), max(s[1], glob)


def _rejects(x, ref, E, mask):
    """True when some element of x under `mask` is outside the bound of this (deliberately wrong) reference."""
    return bool(((x.double() - ref).abs() > E + r64.ETA)[mask].any())


# ----------------------------------------------------------------------------------------------------------------
# Resample2d: both scatters at tile-boundary geometries, edge flows, negative controls and invariances
# ----------------------------------------------------------------------------------------------------------------
# (B, C, H, W, image batch, iH, iW)
RS_SHAPES = [(1, 1, 1, 1, 2, 3, 4), (3, 2, 7, 31, 3, 7, 31), (1, 3, 9, 32, 2, 12, 40), (3, 4, 8, 33, 4, 10, 35),
             (1, 5, 33, 95, 2, 40, 100), (3, 3, 31, 17, 4, 31, 20), (1, 2, 15, 64, 1, 17, 66)]


def _rs_calls(L, img, flow, gout, scatter, arena):
    B, C, H, W = gout.shape
    iB, _, iH, iW = img.shape
    st = _strides(img)
    r = {}
    for bil in (1, 0):
        o = arena.out((B, C, H, W))
        assert L.fn2b200_resample2d_forward(_p(img), st, _p(flow), _p(o), B, C, iH, iW, H, W, 1, bil, _st()) == 0, \
            L.fn2b200_last_error()
        r["fwd", bil] = o
    nws = int(L.fn2b200_resample2d_backward_workspace(st, B, C, iH, iW, H, W)) if scatter == "vector" else 0
    ws = arena.workspace(nws)
    gi, gf = arena.out((B, C, iH, iW)), arena.out((B, 2, H, W))
    assert L.fn2b200_resample2d_backward_ws(_p(img), st, _p(flow), _p(gout), _p(gi), _p(gf), B, C, iH, iW, H, W, 1, 1, 1,
                                            _p(ws), nws, _st()) == 0, L.fn2b200_last_error()
    gf1 = arena.out((B, 2, H, W))
    assert L.fn2b200_resample2d_backward_ws(_p(img), st, _p(flow), _p(gout), P(0), _p(gf1), B, C, iH, iW, H, W, 1, 1, 1,
                                            P(0), 0, _st()) == 0, L.fn2b200_last_error()
    arena.check()
    r.update(gimg=gi, gflow=gf, gflow_only=gf1)
    return r


@pytest.mark.parametrize("B,C,H,W,iB,iH,iW", RS_SHAPES, ids=["x".join(map(str, s)) for s in RS_SHAPES])
def test_resample2d_fp64(B, C, H, W, iB, iH, iW, record_property):
    L = _f2()._lib.LIB
    g = torch.Generator().manual_seed(1000 + 7 * H + W)
    img = (torch.rand(iB, C, iH, iW, generator=g) - 0.5).cuda()
    flow, where = r64.edge_flow(B, H, W, 31 * H + W)
    flow = flow.cuda()
    gout = torch.randn(B, C, H, W, generator=g).cuda()
    fwd, Sf = r64.forward(img, flow)
    near, _ = r64.forward(img, flow, bilinear=False)
    bwd = r64.backward(img, flow, gout)
    Ef, E7, E6 = r64.gamma(7) * Sf, r64.gamma(C + 5) * bwd["S_K7"], r64.gamma(bwd["n_K6"] + 5) * bwd["S_K6"]
    first, stats = None, {}
    for sc in SCATTERS:
        r = _rs_calls(L, img, flow, gout, sc, Arena())
        wt = lambda i, sc=sc: sc + ": " + _where_tile(i, 4)                     # noqa: E731
        _check(r["fwd", 1], fwd, Ef, "forward %s" % sc, wt, stats)
        assert torch.equal(r["fwd", 0].double(), near), "%s: nearest forward differs from the restatement" % sc
        _check(r["gflow"], bwd["gflow"], E7, "K7 %s" % sc, wt, stats)
        _check(r["gimg"], bwd["gimg"], E6, "K6 %s" % sc, wt, stats)
        # pixels no contribution reaches are exactly 0
        assert bool((r["gimg"][(bwd["n_K6"] == 0).expand_as(r["gimg"])] == 0).all()), sc + ": untouched gradient != 0"
        assert torch.equal(r["gflow"], r["gflow_only"]), sc + ": the flow gradient depends on need1"
        if first is None:
            first = r
        else:
            assert torch.equal(r["fwd", 1], first["fwd", 1]) and torch.equal(r["fwd", 0], first["fwd", 0]), \
                sc + ": forward bits differ from the first run"
            assert torch.equal(r["gflow"], first["gflow"]), sc + ": flow gradient bits differ from the vector scatter's"
    # negative controls, each judged only at the pixels whose coordinate on that axis is the control's edge, with the
    # wrong variant applied to that axis alone
    hits = r64.edge_hits(flow)
    for (name, axis), m in hits.items():
        if not bool(m.any()):
            continue
        out, variant = CONTROLS[name]
        if out == "nearest":
            v = r64.forward(img, flow, False, variant, axis)[0]
            fired = bool((first["fwd", 0].double() != v)[m.unsqueeze(1).expand_as(v)].any())
        elif out == "fwd":
            v = r64.forward(img, flow, True, variant, axis)[0]
            fired = _rejects(first["fwd", 1], v, Ef, m.unsqueeze(1).expand_as(v))
        else:
            v = r64.backward(img, flow, gout, variant, axis)["gflow"]
            fired = _rejects(first["gflow"], v, E7, m.unsqueeze(1).expand_as(v))
        FIRED[name] = FIRED.get(name, 0) + int(fired)
    RS_RUN.append((B, C, H, W))
    for k, (ratio, glob) in stats.items():
        STATS.setdefault(k, [0.0, 0.0])
        STATS[k] = [max(STATS[k][0], ratio), max(STATS[k][1], glob)]
        record_property(k, "%.3e %.3e" % (ratio, glob))


# ----------------------------------------------------------------------------------------------------------------
# warp-concat: forward, and backward across the 32 x 16 tile / 8 x 4 cell grid
# ----------------------------------------------------------------------------------------------------------------
WC_SHAPES = [(1, 1, 7), (2, 3, 8), (1, 4, 9), (2, 5, 17), (1, 8, 1), (2, 9, 17)]
GRADS = {"both": (True, True), "x_only": (True, False), "flow_only": (False, True)}
MUL = {0: 1.0, 1: 20.0, 2: 4.0}


def _layouts(C):
    return {"concat": r64.layout(C, flow_div=20.0),
            "fusion": r64.layout(C, cat_channels=C + 7, ch_x=0, n_x=C, ch_warped=-1, ch_flow=C + 1, ch_flow_norm=C + 4,
                                 ch_diff_norm=C + 6)}


def _wc_bwd(L, x, flow, gcat, C, lay, mode, mul, need_x, need_flow, arena):
    B, _, fh, fw = flow.shape
    H, W = x.shape[2], x.shape[3]
    gx = arena.out((B, 2 * C, H, W)) if need_x else None
    gf = arena.out(tuple(flow.shape)) if need_flow else None
    nws = int(L.fn2b200_warp_concat_backward_up_workspace(B, C, H, W, mode, int(need_x)))
    ws = arena.workspace(nws)
    rc = L.fn2b200_warp_concat_backward_up(_p(x), _strides(x), C, _p(flow), fh, fw, mode, ctypes.c_float(mul), _p(gcat),
                                           lay["cat_channels"], lay["ch_x"], lay["n_x"], lay["ch_warped"], lay["ch_flow"],
                                           ctypes.c_float(lay["flow_div"]), lay["ch_flow_norm"], lay["ch_diff_norm"],
                                           _p(gx), _p(gf), _p(ws), nws, B, H, W, _st())
    assert rc == 0, L.fn2b200_last_error()
    arena.check()
    return gx, gf


def _wc_fwd(L, x, flow, C, lay, mode, mul, arena):
    B, _, fh, fw = flow.shape
    H, W = x.shape[2], x.shape[3]
    out = arena.out((B, lay["cat_channels"], H, W), fill=SENTINEL)
    rc = L.fn2b200_warp_concat_forward(_p(x), _strides(x), C, _p(flow), fh, fw, mode, ctypes.c_float(mul), _p(out),
                                       lay["cat_channels"], lay["ch_x"], lay["n_x"], lay["ch_warped"], lay["ch_flow"],
                                       ctypes.c_float(lay["flow_div"]), lay["ch_flow_norm"], lay["ch_diff_norm"], B, H, W,
                                       _st())
    assert rc == 0, L.fn2b200_last_error()
    arena.check()
    return out


def _wc_inputs(B, C, fh, fw, mode, seed):
    g = torch.Generator().manual_seed(seed)
    H, W = 4 * fh, 4 * fw
    x = torch.rand(B, 2 * C, H, W, generator=g) - 0.5
    # img0 == img1 where sample 0's full-resolution flow is exactly 0 (rows 0-1; 0-3 for nearest): n = 0 exactly there.
    # Elsewhere img0 is independent: where the exact d is 0 but fp32's is not, g_d = g_n d / n is a direction set by
    # rounding alone, which no bound can follow.
    R = 4 if mode == 2 else 2
    x[0, :C, :R] = x[0, C:, :R]
    if mode == 0:
        flow, _ = r64.edge_flow(B, H, W, seed)
        flow[0, :, :2] = 0
    elif mode == 2:
        # the catalogue through the nearest upsample: each cell takes the full-resolution edge flow of its top-left
        # pixel divided by MUL[2] = 4 (exact both ways), so that pixel's coordinate is the catalogue value
        flow = r64.edge_flow(B, H, W, seed)[0][:, :, ::4, ::4] / MUL[2]
        flow[0, :, 0] = 0
    else:
        flow = torch.randn(B, 2, fh, fw, generator=g) * 0.3
        flow[0, :, 0] = 0                                  # full-resolution rows 0-1 (bilinear), 0-3 (nearest): zero
    return x.cuda(), flow.cuda()


@pytest.mark.parametrize("mode", [0, 1, 2], ids=["full", "bilinear", "nearest"])
@pytest.mark.parametrize("B,fh,fw", WC_SHAPES, ids=["%dx%dx%d" % s for s in WC_SHAPES])
def test_warp_concat_fp64(B, fh, fw, mode, record_property):
    L = _f2()._lib.LIB
    H, W = 4 * fh, 4 * fw
    mul = MUL[mode]
    tiles_y, tiles_x = (H + 15) // 16, (W + 31) // 32
    stats = {}
    for C in (1, 2, 3):
        x, flow = _wc_inputs(B, C, fh, fw, mode, 100 * fh + 10 * fw + C + mode)
        f32 = r64.upsample_flow32(flow, mode, mul) if mode else flow.float()
        if mode != 1:
            assert any(bool(m.any()) for m in r64.edge_hits(f32).values()), "no catalogue coordinate reached"
        for lname, lay in _layouts(C).items():
            what = "C=%d %s" % (C, lname)
            gcat = torch.randn(B, lay["cat_channels"], H, W, generator=torch.Generator().manual_seed(C)).cuda()
            # forward; with flow_div = 1 the flow channel is the upsampled flow itself, bit for bit
            cat = _wc_fwd(L, x, flow, C, lay, mode, mul, Arena())
            ref, E = r64.warp_concat_forward(x, f32, C, lay)
            own = ~torch.isnan(ref)
            assert bool((cat[~own] == SENTINEL).all()), what + ": the forward wrote a channel its layout does not own"
            wt = lambda i: _where_tile(i, 2)                                                 # noqa: E731
            _check(torch.where(own, cat, 0.0), torch.where(own, ref, 0.0), E, "fwd_chain " + what, wt, stats)
            if mode and lname == "fusion":
                assert torch.equal(cat[:, C + 1:C + 3], f32), "the fused forward's flow is not load_flow's fp32 upsample"
            # backward, every gradient choice
            r = r64.warp_concat_backward(x, f32, gcat, C, lay, mode, mul)
            res = {}
            for gname, (nx, nf) in GRADS.items():
                res[gname] = _wc_bwd(L, x, flow, gcat, C, lay, mode, mul, nx, nf, Arena())
            gx, gf = res["both"]
            _check(gx, r["gx"], r["E_gx"], "gx " + what, wt, stats)
            cell = lambda i: "cell (%d, %d), tiles y %s x %s" % (                             # noqa: E731
                i[-2], i[-1], sorted({max(i[-2] - 1, 0) // 4, min(i[-2] + 1, fh - 1) // 4}),
                sorted({max(i[-1] - 1, 0) // 8, min(i[-1] + 1, fw - 1) // 8}))
            _check(gf, r["gflow"], r["E_gflow"], "gflow%d %s" % (mode, what), cell if mode == 1 else wt, stats)
            zero = (r["n"] == 0).expand(B, C, H, W)
            if lay["ch_x"] >= 0 and lay["n_x"] >= C:
                gx0 = gcat[:, lay["ch_x"]:lay["ch_x"] + C]
                assert bool(zero.any()) and torch.equal(gx[:, :C][zero], gx0[zero]), what + ": g_d != 0 where n = 0"
            _check(res["x_only"][0], r["gx"], r["E_gx"], "gx " + what + " x_only", wt, stats)
            assert torch.equal(res["flow_only"][1], gf), what + ": the flow gradient depends on need_x"
            again = _wc_bwd(L, x, flow, gcat, C, lay, mode, mul, True, True, Arena())[1]
            assert torch.equal(again, gf), what + ": a repeat call gave other flow-gradient bits"
            if B > 1:
                s = slice(B - 1, B)
                alone = _wc_bwd(L, x[s].contiguous(), flow[s].contiguous(), gcat[s].contiguous(), C, lay, mode, mul,
                                False, True, Arena())[1]
                assert torch.equal(alone, gf[s]), what + ": the last sample alone differs from the batch"
            # negative control: an adjoint that drops tile (0, 0)'s partial for the cells it shares with its neighbours,
            # judged on those cells only
            if mode == 1 and (tiles_x > 1 or tiles_y > 1):
                v = r64.upsample_adjoint(r["g_up"], 1, mul, drop=(0, 0))
                shared = torch.zeros_like(gf, dtype=torch.bool)
                shared[..., :5, :9] = True
                shared[..., :4, :8] = False
                assert _rejects(gf, v, r["E_gflow"], shared), what + ": dropping tile (0, 0)'s shared partials not rejected"
    for k, (ratio, glob) in stats.items():
        STATS.setdefault(k, [0.0, 0.0])
        STATS[k] = [max(STATS[k][0], ratio), max(STATS[k][1], glob)]
        record_property(k, "%.3e %.3e" % (ratio, glob))


# ----------------------------------------------------------------------------------------------------------------
# FusionConcat: two nearest warp-concat passes into one 11-channel buffer (pybind/fn2b200_ops.cc FUSION_SD, FUSION_S2)
# ----------------------------------------------------------------------------------------------------------------
DIV = 20.0
FUSION_SD = r64.layout(3, cat_channels=11, ch_x=0, n_x=3, ch_warped=-1, ch_flow=3, ch_flow_norm=7, ch_diff_norm=9)
FUSION_S2 = r64.layout(3, cat_channels=11, ch_x=-1, n_x=0, ch_warped=-1, ch_flow=5, ch_flow_norm=8, ch_diff_norm=10)
FUSION_NEEDS = [(True, True, True), (True, False, False), (False, True, False), (False, False, True)]


def _fusion_inputs(B, fh, fw, seed):
    g = torch.Generator().manual_seed(seed)
    H, W = 4 * fh, 4 * fw
    x = torch.rand(B, 6, H, W, generator=g) - 0.5
    x[0, :3, :4] = x[0, 3:, :4]                       # both flows are 0 on rows 0-3 of sample 0: n = 0 exactly there
    sd = torch.randn(B, 2, fh, fw, generator=g) * 3 * DIV          # sd_flow2 is divided by div_flow, s2_flow2 multiplied
    s2 = torch.randn(B, 2, fh, fw, generator=g) * 3 / DIV
    sd[0, :, 0] = 0
    s2[0, :, 0] = 0
    gcat = torch.randn(B, 11, H, W, generator=g)
    return x.cuda(), sd.cuda(), s2.cuda(), gcat.cuda()


@pytest.mark.parametrize("B,fh,fw", [(2, 3, 8), (1, 9, 17)], ids=["2x3x8", "1x9x17"])
def test_fusion_concat_fp64(B, fh, fw, record_property):
    """The SD pass (x | sd flow / div | norms, flow_mul = 1 / div_flow) and the S2 pass (no x channels, so its
    grad_x[:, :3] is g_d alone; flow_mul = div_flow) through the C ABI into one sentinel-filled buffer, the operator and
    the module, against two fp64 restatements; the backward for every need_* choice, its x gradient the sum of both."""
    f = _f2()
    L = f._lib.LIB
    H, W = 4 * fh, 4 * fw
    x, sd, s2, gcat = _fusion_inputs(B, fh, fw, 10 * fh + fw)
    passes = [(sd, float(torch.tensor(1.0 / DIV, dtype=torch.float32)), FUSION_SD), (s2, DIV, FUSION_S2)]
    refs = [(fl, mul, lay, r64.upsample_flow32(fl, 2, mul)) for fl, mul, lay in passes]
    stats = {}
    wt = lambda i: _where_tile(i, 2)                                                           # noqa: E731
    # forward: the C ABI, one pass after the other into one buffer
    arena = Arena()
    cat = arena.out((B, 11, H, W), fill=SENTINEL)
    for k, (fl, mul, lay, _) in enumerate(refs):
        rc = L.fn2b200_warp_concat_forward(_p(x), _strides(x), 3, _p(fl), fh, fw, 2, ctypes.c_float(mul), _p(cat), 11,
                                           lay["ch_x"], lay["n_x"], lay["ch_warped"], lay["ch_flow"],
                                           ctypes.c_float(lay["flow_div"]), lay["ch_flow_norm"], lay["ch_diff_norm"], B, H,
                                           W, _st())
        assert rc == 0, L.fn2b200_last_error()
        if k == 0:
            torch.cuda.synchronize()
            assert bool((cat[:, [5, 6, 8, 10]] == SENTINEL).all()), "the SD pass wrote the S2 pass's channels"
    arena.check()
    (rsd, esd), (rs2, es2) = (r64.warp_concat_forward(x, f32, 3, lay) for _, _, lay, f32 in refs)
    ref, E = torch.where(torch.isnan(rsd), rs2, rsd), torch.where(torch.isnan(rsd), es2, esd)
    assert not bool(torch.isnan(ref).any())
    _check(cat, ref, E, "fusion_fwd", wt, stats)
    assert torch.equal(cat[:, 3:5], refs[0][3]) and torch.equal(cat[:, 5:7], refs[1][3]), \
        "the fused forward's flows are not load_flow's fp32 upsample"
    op = torch.ops.fn2b200.fusion_concat(x, sd, s2, DIV)
    assert torch.equal(op, cat), "fusion_concat op != the two C-ABI passes"
    assert torch.equal(f.fused.FusionConcat(DIV)(x, sd, s2), cat), "FusionConcat module != the two C-ABI passes"
    # backward
    r = [r64.warp_concat_backward(x, f32, gcat, 3, lay, 2, mul) for _, mul, lay, f32 in refs]
    gx_ref = r[0]["gx"] + r[1]["gx"]
    E_gx = r[0]["E_gx"] + r[1]["E_gx"] + r64.U * (r[0]["gx"].abs() + r[1]["gx"].abs())
    got = {}
    for need in FUSION_NEEDS:
        got[need] = torch.ops.fn2b200.fusion_concat_backward(x, sd, s2, gcat, DIV, *need)
        gx, gsd, gs2 = got[need]
        if need[0]:
            _check(gx, gx_ref, E_gx, "fusion_gx %s" % (need,), wt, stats)
            zero = ((r[0]["n"] == 0) & (r[1]["n"] == 0)).expand(B, 3, H, W)
            assert bool(zero.any()) and torch.equal(gx[:, :3][zero], gcat[:, :3][zero]), "g_d != 0 where n = 0"
        for k, (g, name) in enumerate(((gsd, "sd"), (gs2, "s2"))):
            if need[k + 1]:
                _check(g, r[k]["gflow"], r[k]["E_gflow"], "fusion_g%s %s" % (name, need), wt, stats)
                assert torch.equal(g, got[FUSION_NEEDS[0]][k + 1]), "fusion g_%s depends on the other needs" % name
    # the module's autograd: the same flow gradients bit for bit, the x gradient within the bound
    xa, sda, s2a = (t.clone().requires_grad_() for t in (x, sd, s2))
    f.fused.FusionConcat(DIV)(xa, sda, s2a).backward(gcat)
    assert torch.equal(sda.grad, got[FUSION_NEEDS[0]][1]) and torch.equal(s2a.grad, got[FUSION_NEEDS[0]][2])
    _check(xa.grad, gx_ref, E_gx, "fusion_gx autograd", wt, stats)
    for k, (ratio, glob) in stats.items():
        STATS.setdefault(k, [0.0, 0.0])
        STATS[k] = [max(STATS[k][0], ratio), max(STATS[k][1], glob)]
        record_property(k, "%.3e %.3e" % (ratio, glob))


# ----------------------------------------------------------------------------------------------------------------
# layouts: strided images through the C ABI, the operators and the modules' autograd, bit for bit against .contiguous()
# ----------------------------------------------------------------------------------------------------------------
def _layout_views(base):
    """(name, view) of base [B, C, H, W]: a channel slice, channels_last, a batch expand (stride 0), a 4-byte offset."""
    B, C, H, W = base.shape
    big = torch.cat((torch.randn(B, 3, H, W, device="cuda"), base), 1)
    off = torch.empty(base.numel() + 1, device="cuda")[1:].view(base.shape).copy_(base)
    assert off.storage_offset() == 1
    return [("slice", big[:, 3:]), ("channels_last", base.contiguous(memory_format=torch.channels_last)),
            ("expand", base[:1].expand(B, C, H, W)), ("offset4", off)]


@pytest.mark.parametrize("C", [1, 3])
def test_layouts_bit_for_bit(C):
    f = _f2()
    F2 = f.functional
    B, H, W = 2, 20, 36
    g = torch.Generator(device="cuda").manual_seed(C)
    base = torch.rand(B, C, H, W, device="cuda", generator=g)
    flow = torch.randn(B, 2, H, W, device="cuda", generator=g) * 3
    go = torch.randn(B, C, H, W, device="cuda", generator=g)
    xbase = torch.rand(B, 2 * C, H, W, device="cuda", generator=g)
    gcat = torch.randn(B, 3 * C + 3, H, W, device="cuda", generator=g)
    for name, v in _layout_views(base):
        c = v.contiguous()
        assert torch.equal(F2.resample2d_forward(v, flow), F2.resample2d_forward(c, flow)), name + ": C ABI forward"
        a, b = F2.resample2d_backward(v, flow, go), F2.resample2d_backward(c, flow, go)
        assert torch.equal(a[1], b[1]), name + ": C ABI flow gradient"
        assert torch.allclose(a[0], b[0], rtol=1e-5, atol=1e-5), name + ": C ABI image gradient (atomics: bounded)"
        assert torch.equal(torch.ops.fn2b200.resample2d_forward(v, flow, 1, True),
                           torch.ops.fn2b200.resample2d_forward(c, flow, 1, True)), name + ": operator forward"
        outs = []
        for t in (v, c):
            fl = flow.clone().requires_grad_()
            o = f.Resample2d()(t, fl)
            o.backward(go)
            outs.append((o.detach(), fl.grad))
        assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1]), name + ": module autograd"
    for name, v in _layout_views(xbase):
        c = v.contiguous()
        assert torch.equal(F2.warp_concat_forward(v, flow, C=C), F2.warp_concat_forward(c, flow, C=C)), name + ": wc fwd"
        a, b = F2.warp_concat_backward(v, flow, gcat, C=C), F2.warp_concat_backward(c, flow, gcat, C=C)
        assert torch.equal(a[1], b[1]), name + ": warp-concat flow gradient"
        assert torch.allclose(a[0], b[0], rtol=1e-5, atol=1e-5), name + ": warp-concat image gradient (atomics: bounded)"
        outs = []
        for t in (v, c):
            fl = flow.clone().requires_grad_()
            o = f.fused.WarpConcat(div_flow=20.0)(t, fl)
            o.backward(gcat)
            outs.append((o.detach(), fl.grad))
        assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1]), name + ": WarpConcat autograd"
        if C == 3:
            sd, s2 = (torch.randn(B, 2, H // 4, W // 4, device="cuda", generator=g) for _ in range(2))
            assert torch.equal(torch.ops.fn2b200.fusion_concat(v, sd, s2, DIV),
                               torch.ops.fn2b200.fusion_concat(c, sd, s2, DIV)), name + ": fusion_concat forward"
            a = torch.ops.fn2b200.fusion_concat_backward(v, sd, s2, gcat[:, :11], DIV, True, True, True)
            b = torch.ops.fn2b200.fusion_concat_backward(c, sd, s2, gcat[:, :11], DIV, True, True, True)
            assert torch.equal(a[1], b[1]) and torch.equal(a[2], b[2]), name + ": fusion_concat flow gradients"


def test_report_ratios():
    """Runs last: prints the largest |d| / (kappa S) and max|d| / max|ref64| per quantity over the cases above, and
    how many (case, axis) pairs each edge's negative control rejected; when every Resample2d case ran, every edge's
    control must have rejected the kernel's output in at least one of them."""
    for k in sorted(STATS):
        print("RATIO %-14s %.3e %.3e" % (k, STATS[k][0], STATS[k][1]))
    for k in CONTROLS:
        print("CONTROL %-14s %-8s %-17s fired %d" % ((k,) + CONTROLS[k] + (FIRED.get(k, 0),)))
    if len(RS_RUN) < len(RS_SHAPES):
        pytest.skip("not every Resample2d case ran")
    assert not [k for k in CONTROLS if not FIRED.get(k)], "edges whose negative control never rejected the kernel"
