"""The tensor-core correlation's persistent tile schedule at every channel count, element by element, against an fp64
reference.

`corr_fwd_tc_kernel` and `corr_bwd_tc_kernel<C/64, CAT>` run one CTA per SM, deal the tiles out round-robin and carry
their shared-memory rings from one tile to the next; the forward deals the (tile, unit) pairs of its last, partial
round in shares that may start inside a tile and run into the next.  tests/corr_tc_schedule.py models that assignment
and picks, from this GPU's SM count, a batch for each regime of it (fewer tiles than SMs, whole rounds, shares of 1, 2,
5 and 6 units, three rounds and a partial one, multi-tile samples with ragged edges).  Every regime runs at C = 64, 128,
192 and 256 through the C ABI:

- forward (`_ws`) and `forward_cat` (cat_channels = 448, ch_offset = 5, LeakyReLU slope 0.1);
- backward with both gradients, gradInput1 only and gradInput2 only, each with the split handed over and recomputed;
- `backward_cat` with LeakyReLU's mask read from the concat (split handed over and recomputed), and the plain backward
  of the masked gradient.

Every output is a view in a NaN-poisoned, guarded allocation (tests/guarded.py), so every element must be written and
nothing outside the view touched; the concat channels the call does not own hold a sentinel that must survive.

Accuracy, element by element against tests/torch_ref.py's fp64 correlation.  Each operand is split x = hi + lo (two
bf16): |x - hi| <= 2^-8 |x|, and lo = rn(x - hi) leaves |x - hi - lo| <= 2^-16 |x|.  The kernels sum the three
products hi*hi + hi*lo + lo*hi; each is exact in fp32 (8 x 8 significand bits), and the dropped part
lo*lo + (x - hi - lo) y + x' (y - hi - lo) is at most 3 * 2^-16 (1 + 2^-7) |x y|.  The 3K products of an output
element (K = C for the forward; at most K = 441 band entries for a gradient) are accumulated in fp32 on the tensor
core, and the result is scaled by 1/C (and, for the concat, by the slope).  Round-to-nearest accumulation errs by at
most u = 2^-24 of the running sum of |products| per addition; the tensor core is not known to round like IEEE fp32
(it may truncate), so allow 2u per addition and per scaling:

    |x - ref64| <= kappa(K) * S,   kappa(K) = 3 * 2^-16 * (1 + 2^-7) + 2 * (3K + 3) * 2^-24,

S being the same sum over |a|, |b|, |gradOutput| (the fp64 reference applied to absolute values).  kappa = 6.94e-5,
9.23e-5, 1.15e-4 and 1.38e-4 for the forward at C = 64, 128, 192 and 256, and 2.04e-4 for the gradients.  An element
whose S is 0 (every product in the padding) must be exactly 0.

The bound is a worst case that random data does not approach, so a second, global statistic, max|d| / max|ref64| of a
whole tensor, must stay below GLOBAL_TOL.  Dropping one of the cross products hi*lo or lo*hi costs ~2^-9 per product,
1e-4 to 1e-3 of max|ref| (DESIGN section 4.1).  GLOBAL_TOL comes from the first run of this file, on an H100 80GB
HBM3 (132 SMs, 700 W power limit, driver 580.159.03).  The largest values over all regimes and over the forward, the
concat and every gradient were:

    C      max |d| / (kappa S)   max|d| / max|ref64|
    64     0.087                 6.6e-6
    128    0.046                 7.7e-6
    192    0.039                 7.9e-6
    256    0.037                 6.9e-6

GLOBAL_TOL = 2e-5 is 2.5 times the largest of them, and a dropped cross product exceeds it several times over.

Schedule invariance, bit for bit: the arithmetic of an element does not depend on the CTA, segment or ring slot that
runs its tile or unit, so the first and last samples and those whose tiles fall in the forward's partial round must
give the same bits computed alone (B = 1) and in a batch of another size (another dealing), and a second identical call
must repeat every bit.  The gradients of the one-gradient launches and of either split setting must equal those of
the two-gradient launch, and backward_cat the plain backward of the masked gradient.

A failing element is reported with its place in the schedule: sample, parity class, tile, unit (forward) or warpgroup
(backward), CTA and segment.
"""
import ctypes

import numpy as np
import pytest
import torch

import corr_tc_schedule as sch
import torch_ref
from guarded import SENTINEL, Arena
from oracle import cpu as orc
from util import assert_close

pytestmark = pytest.mark.gpu
P = ctypes.c_void_p
MD, S2 = 20, 2
PRM = (MD, 1, MD, 1, S2)                  # pad, kernel_size, max_displacement, stride1, stride2
D = 441
CAT_CH, CH_OFF, SLOPE = D + 7, 5, 0.1
CS = [64, 128, 192, 256]
GLOBAL_TOL = 2e-5
NEEDS = ((1, 1), (1, 0), (0, 1))


def kappa(K):
    return 3 * 2.0 ** -16 * (1 + 2.0 ** -7) + 2 * (3 * K + 3) * 2.0 ** -24


def _sms():
    """The SM count the launchers read; an H100 SXM's where there is no GPU (the cases are then only collected)."""
    if torch.cuda.is_available():
        return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count
    return 132


SMS = _sms()
CASES = [(r,) + sch.pick(r, SMS) for r in sch.REGIMES]
IDS = ["%s-%s" % (c[0], sch.describe(*c[1:], SMS)) for c in CASES]


def _f2():
    import flownet2_b200
    return flownet2_b200


def _p(t):
    return P(t.data_ptr()) if t is not None else P(0)


def _ok(L, rc):
    assert rc == 0, L.fn2b200_last_error()


def _inputs(B, C, H, W, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    a, b = (torch.randn(B, C, H, W, device="cuda", generator=g) for _ in range(2))
    go = torch.randn(B, D, H, W, device="cuda", generator=g)
    gcat = torch.randn(B, CAT_CH, H, W, device="cuda", generator=g)
    return a, b, go, gcat


def _calls(a, b, go, gcat):
    """Every call of a case, on guarded outputs and a guarded workspace of exactly the queried size."""
    L = _f2()._lib.LIB
    arena = Arena()
    B, C, H, W = a.shape
    st = P(torch.cuda.current_stream().cuda_stream)
    nws = int(L.fn2b200_correlation_forward_workspace(B, C, H, W, *PRM))
    assert nws > 0 and nws == int(L.fn2b200_correlation_backward_workspace(B, C, H, W, *PRM))
    ws = arena.workspace(nws)
    r = {"out": arena.out((B, D, H, W)), "cat": arena.out((B, CAT_CH, H, W), fill=SENTINEL)}
    _ok(L, L.fn2b200_correlation_forward_ws(_p(a), _p(b), _p(r["out"]), B, C, H, W, *PRM, 1, _p(ws), nws, st))
    _ok(L, L.fn2b200_correlation_forward_cat(_p(a), _p(b), _p(r["cat"]), CAT_CH, CH_OFF, SLOPE, B, C, H, W, *PRM, 1,
                                             _p(ws), nws, st))
    for split in (1, 0):                       # 1 first: the workspace holds the forward's split of (a, b)
        for need in NEEDS:
            g1, g2 = (arena.out((B, C, H, W)) if n else None for n in need)
            _ok(L, L.fn2b200_correlation_backward_ws(_p(a), _p(b), _p(go), _p(g1), _p(g2), B, C, H, W, *PRM, 1, _p(ws),
                                                     nws, split, st))
            r["g", split, need] = (g1, g2)
        c1, c2 = arena.out((B, C, H, W)), arena.out((B, C, H, W))
        _ok(L, L.fn2b200_correlation_backward_cat(_p(a), _p(b), _p(gcat), _p(r["cat"]), CAT_CH, CH_OFF, SLOPE, _p(c1),
                                                  _p(c2), B, C, H, W, *PRM, 1, _p(ws), nws, split, st))
        r["c", split] = (c1, c2)
    c = r["cat"][:, CH_OFF:CH_OFF + D]
    gs = gcat[:, CH_OFF:CH_OFF + D]
    r["gm"] = torch.where(c > 0, gs, gs * SLOPE).contiguous()
    m1, m2 = arena.out((B, C, H, W)), arena.out((B, C, H, W))
    _ok(L, L.fn2b200_correlation_backward_ws(_p(a), _p(b), _p(r["gm"]), _p(m1), _p(m2), B, C, H, W, *PRM, 1, _p(ws), nws,
                                             1, st))
    r["m"] = (m1, m2)
    arena.check()
    return r


def _tensors(r):
    """(name, tensor) of every output of a case."""
    yield "out", r["out"]
    yield "cat", r["cat"]
    for k, v in r.items():
        if isinstance(k, tuple) or k == "m":
            for i, t in enumerate(v):
                if t is not None:
                    yield "%s grad%d" % (k, i + 1), t


def _check(x, ref, S, K, what, where, stats):
    """|x - ref| <= kappa(K) S element by element, then max|x - ref| / max|ref| <= GLOBAL_TOL."""
    d = (x.double() - ref).abs()
    lim = kappa(K) * S
    bad = d > lim
    if bool(bad.any()):
        i = tuple(int(v) for v in bad.nonzero()[0])
        pytest.fail("%s: %d elements beyond kappa S; the first, %s = %s: |d| = %.3e, kappa S = %.3e, ref %.6e, got %.6e" % (
            what, int(bad.sum()), i, where(i), float(d[i]), float(lim[i]), float(ref[i]), float(x[i])))
    ratio = float(torch.where(lim > 0, d / lim.clamp_min(1e-300), torch.zeros_like(d)).max())
    glob = float(d.max() / ref.abs().max())
    if glob > GLOBAL_TOL:
        i = np.unravel_index(int(d.argmax()), tuple(d.shape))
        pytest.fail("%s: max|d|/max|ref| = %.3e > %.1e; the largest |d| at %s = %s" % (
            what, glob, GLOBAL_TOL, tuple(int(v) for v in i), where(i)))
    stats["ratio"] = max(stats.get("ratio", 0.0), ratio)
    stats["global"] = max(stats.get("global", 0.0), glob)


def _check_fp64(a, b, go, gcat, r, fwd, bwd, stats):
    B, C, H, W = a.shape
    a64, b64, aa, ba = a.double(), b.double(), a.double().abs(), b.double().abs()
    ref = torch_ref.correlation64(a64, b64, MD, 1, MD, 1, S2)
    S = torch_ref.correlation64(aa, ba, MD, 1, MD, 1, S2)
    wf = lambda i: sch.locate_forward(fwd, H, W, *i)                                   # noqa: E731
    _check(r["out"], ref, S, C, "forward", wf, stats)
    _check(r["cat"][:, CH_OFF:CH_OFF + D], torch.where(ref > 0, ref, ref * SLOPE), S, C, "forward_cat", wf, stats)
    others = torch.cat([r["cat"][:, :CH_OFF], r["cat"][:, CH_OFF + D:]], 1)
    assert bool((others == SENTINEL).all()), "forward_cat wrote channels outside [ch_offset, ch_offset + 441)"
    del ref, S
    for gname, gout, grads in (("backward", go, r["g", 1, (1, 1)]), ("backward_cat", r["gm"], r["c", 1])):
        g64 = gout.double()
        refs = torch_ref.correlation64_backward(a64, b64, g64, MD, 1, MD, 1, S2)
        Ss = torch_ref.correlation64_backward(aa, ba, g64.abs(), MD, 1, MD, 1, S2)
        for k in range(2):
            wb = lambda i, k=k: "channel %d: %s" % (i[1], sch.locate_backward(bwd, H, W, k, i[0], i[2], i[3]))  # noqa: E731
            _check(grads[k], refs[k], Ss[k], D, "%s grad%d" % (gname, k + 1), wb, stats)
        del refs, Ss


def _check_bits(r):
    """The variants of one call that must agree bit for bit."""
    out = r["out"]
    assert torch.equal(r["cat"][:, CH_OFF:CH_OFF + D], torch.where(out > 0, out, out * SLOPE)), "forward_cat != act(forward)"
    g1, g2 = r["g", 1, (1, 1)]
    for split in (1, 0):
        for need in NEEDS:
            x1, x2 = r["g", split, need]
            assert x1 is None or torch.equal(x1, g1), "grad1 of split=%d need=%s differs from the two-gradient call" % (
                split, need)
            assert x2 is None or torch.equal(x2, g2), "grad2 of split=%d need=%s differs from the two-gradient call" % (
                split, need)
        assert all(torch.equal(x, y) for x, y in zip(r["c", split], r["m"])), \
            "backward_cat (split=%d) != the plain backward of the masked gradient" % split


@pytest.mark.parametrize("C", CS)
@pytest.mark.parametrize("regime,B,H,W", CASES, ids=IDS)
def test_tc_schedule(regime, B, H, W, C, record_property):
    f = _f2()
    assert f._lib.LIB.fn2b200_correlation_path(C, H, W, *PRM) == 2
    nt = sch.ntiles(B, H, W)
    fwd, bwd = sch.Forward(nt, SMS), sch.Backward(nt, SMS)
    assert sch.REGIMES[regime][1](fwd)
    a, b, go, gcat = _inputs(B, C, H, W, 1000 * C + B)
    r = _calls(a, b, go, gcat)
    _check_bits(r)
    stats = {}
    _check_fp64(a, b, go, gcat, r, fwd, bwd, stats)
    record_property("max_elem_ratio", "%.3e" % stats["ratio"])
    record_property("max_global", "%.3e" % stats["global"])

    # a second identical call repeats every bit
    again = dict(_tensors(_calls(a, b, go, gcat)))
    for name, t in _tensors(r):
        assert torch.equal(t, again[name]), "%s: a second identical call gave other bits" % name
    del again

    # the first and last samples, and those of the forward's partial round, alone and in a batch of another size
    nxt, nyt = sch.tile_grid(H, W)
    part = [sch.decode(t, nxt, nyt)[0] for t in range(fwd.full, nt)]
    sel = sorted({0, B - 1} | ({min(part), max(part)} if part else set()))
    other = sel + [sel[0]] * (2 if len(sel) + 1 == B else 1)
    batches = [[n] for n in sel if B > 1] + [other]
    for idx in batches:
        s = torch.tensor(idx, device="cuda")
        sub = dict(_tensors(_calls(a[s].contiguous(), b[s].contiguous(), go[s].contiguous(), gcat[s].contiguous())))
        for name, t in _tensors(r):
            assert torch.equal(t[s], sub[name]), "%s: samples %s computed in a batch of %d differ from the batch of %d (%s)" % (
                name, idx, len(idx), B, sch.describe(len(idx), H, W, SMS))


@pytest.mark.parametrize("C", CS)
def test_tc_autograd_and_oracle(C):
    """The Correlation module's forward and backward (the forward's split handed to the backward: one launch) equal the
    functional calls bit for bit, in a regime where a CTA's share of the partial round spans two tiles.  On one small
    shape the CPU oracle ties the fp64 reference to the reference's semantics, and the kernels to the 1e-4 contract."""
    f = _f2()
    F2 = f.functional
    _, B, H, W = next(c for c in CASES if c[0] == "wper2")
    a, b, go, _ = _inputs(B, C, H, W, 7 * C)
    ad, bd = a.clone().requires_grad_(), b.clone().requires_grad_()
    n0 = F2.launch_count()
    out = f.Correlation(*PRM, 1)(ad, bd)
    n1 = F2.launch_count()
    out.backward(go)
    torch.cuda.synchronize()
    assert (n1 - n0, F2.launch_count() - n1) == (2, 1), "split + forward, then the backward alone"
    assert torch.equal(out.detach(), F2.correlation_forward(a, b, *PRM))
    r1, r2 = F2.correlation_backward(a, b, go, *PRM)
    assert torch.equal(ad.grad, r1) and torch.equal(bd.grad, r2)

    a, b, go = a[:1].cpu(), b[:1].cpu(), go[:1].cpu()
    o = orc.correlation_forward(a.numpy(), b.numpy(), *PRM)
    o1, o2 = orc.correlation_backward(a.numpy(), b.numpy(), go.numpy(), *PRM)
    a64, b64 = a.cuda().double(), b.cuda().double()
    ref = torch_ref.correlation64(a64, b64, MD, 1, MD, 1, S2)
    S = torch_ref.correlation64(a64.abs(), b64.abs(), MD, 1, MD, 1, S2)
    refs = torch_ref.correlation64_backward(a64, b64, go.cuda().double(), MD, 1, MD, 1, S2)
    Ss = torch_ref.correlation64_backward(a64.abs(), b64.abs(), go.cuda().double().abs(), MD, 1, MD, 1, S2)
    for x, rr, s, n in ((o, ref, S, C), (o1, refs[0], Ss[0], D), (o2, refs[1], Ss[1], D)):
        assert bool(((torch.from_numpy(x).cuda().double() - rr).abs() <= 2 * (n + 2) * 2.0 ** -24 * s).all())
    assert_close(out[:1].detach().cpu().numpy(), o, 1e-4, "C=%d forward vs oracle" % C)
    assert_close(ad.grad[:1].cpu().numpy(), o1, 1e-4, "C=%d grad1 vs oracle" % C)
    assert_close(bd.grad[:1].cpu().numpy(), o2, 1e-4, "C=%d grad2 vs oracle" % C)
