"""The FP32-FMA correlation kernels (`corr_fwd_tiled_kernel` / `corr_bwd_tiled_kernel`, and the generic
`corr_fwd_generic_kernel` / `corr_bwd_generic_kernel` that run every parameter set the other families refuse),
element by element, against tests/torch_ref.py's fp64 restatement, across the reference's parameter space.

Every call goes through the C ABI on guarded, NaN-poisoned outputs (tests/guarded.py); the concat channels that are not
the correlation's hold a sentinel that must survive, and the workspace is exactly the queried size (0: none of these
cases runs on tensor cores).  Each case asserts its family with fn2b200_correlation_path and checks, through the
torch.profiler kernel names, that the kernels of that family and no others ran (a case whose record lacks one of its
kernels runs once more, as the profiler can drop records of kernels that ran).  Per case: the forward, forward_cat at
ch_offset 3 with LeakyReLU slope 0.1 and 0; the backward with both gradients, gradInput1 only and gradInput2 only, and
backward_cat (slope 0.1) -- the backward only for stride1 = 1, the reference's only backward.

Accuracy, per element: |x - ref64| <= kappa(K) S, S being the restatement applied to |a|, |b| and |gradOutput| (for
backward_cat the masked gradient).  These are IEEE round-to-nearest fp32 pipes: a sum whose every term passes through at
most n roundings errs by at most gamma_n S, gamma_n = n u / (1 - n u), u = 2^-24, and gamma_n <= (n + 1) u for the n here.
kappa(K) = (K + 2) u, the +2 covering the divide by k^2 C and the LeakyReLU slope (or, backward_cat, the slope applied
to each gradOutput value, one rounding before its product):

    tiled forward     acc = fmaf(a, b, acc) over the C channels (the first is exact): C - 1 roundings   K = C
    generic forward   4 fma chains of <= ceil(C/4) products, combined in 2 adds, the k^2 tap sums added
                      into one accumulator: <= C/4 + 3 + k^2 <= k^2 C + k^2 + 3 roundings             K = k^2 C + k^2 + 3
    tiled backward    acc = fmaf(g, other, acc) over the D displacements: D - 1 roundings             K = D
    generic backward  per displacement a window sum of <= k^2 gradOutput values (k^2 - 1), times the
                      other input (1), added into the accumulator (1): <= D (k^2 + 1) roundings      K = D (k^2 + 1)

Elements whose S is 0 (every tap in the padding, or a gradient no output reads) must be exactly 0.  On top, per tensor,
max|x - ref64| / max|ref64| <= GLOBAL_TOL.

The catalogue.  Tiled: every (stride2, dr) of FN2_TILED_CONFIGS at off = md - pad in {-4, 0, +4}, and +-8 at (2, 10);
md % s2 != 0 with pad != md at (pad, md, s2) = (17, 21, 2), (13, 9, 2), (1, 5, 2); C over 1, 7, 9, 16, 63, 65, 130; W
and oW over 4, 12, 124, 132, 260 (partial last 8-pixel group and 128-pixel tile); oH over 1, s2, 7, 9, 17 (the forward's
4-row quads of one parity); B 1 and 3; C = 64, 128, 192, 256 at a ragged FlowNetC shape with FN2B200_CORR_FWD/BWD=fma;
and FlowNet2's [8, 256, 56, 128] through the workspace-less plain entry points.  Generic: kernel_size 1, 2, 3, 5; stride1
1, 2, 3 (forward only); stride2 1, 2, 3; md 0, 1 (with s2 = 2: D = 1), 3, 5, 7; pad 0, md - 1, md, md + kr + 1; C 1, 3,
4, 5, 9 around the 4-way channel unroll's tail; W % 4 != 0 and (md - pad) % 4 != 0; and a tiled configuration whose
operands start 4 bytes past a 16-byte boundary.

GLOBAL_TOL comes from the first run of this file, on an H100 80GB HBM3 (700 W power limit, driver 580.159.03; 35
cases, about 30 s together with tests/test_gpu_channelnorm_exact.py).  The largest values over all cases were:

    family    output         max |d| / (kappa S)   max|d| / max|ref64|
    tiled     forward        0.398                 7.0e-7
    tiled     forward_cat    0.341                 6.3e-7
    tiled     backward       0.150                 1.1e-6
    tiled     backward_cat   0.169                 4.6e-7
    generic   forward        0.235                 2.3e-7
    generic   forward_cat    0.180                 2.3e-7
    generic   backward       0.312                 4.0e-7
    generic   backward_cat   0.474                 2.2e-7

GLOBAL_TOL = 2.8e-6 is 2.5 times the largest of them.  Every negative control was rejected in both families and, where
it acts on both, in both directions.

Bit for bit: a one-gradient call equals the two-gradient call; backward_cat equals the plain backward of the masked
gradient; forward_cat's planes equal LeakyReLU of the forward's; the first and last samples computed alone equal the same
samples in the batch (gridDim.z carries the sample); a repeated call repeats every bit.

Negative controls.  Each variant of torch_ref.VARIANTS is compared with the kernels' output only on the elements it can
change (torch_ref.variant_edges), within its own kappa S; it is rejected when some such element lies outside.
test_zz_every_control_rejected, which runs last, asserts that each variant was rejected in at least one case, and
`replicate` at least once per family and direction, so the border taps of each kernel are reached.
"""
import ctypes

import pytest
import torch

import torch_ref
from guarded import SENTINEL, Arena
from util import cuda_profile

pytestmark = pytest.mark.gpu
P = ctypes.c_void_p
U = 2.0 ** -24
GLOBAL_TOL = 2.8e-6
CH_OFF, SLOPES = 3, (0.1, 0.0)
NEEDS = ((1, 1), (1, 0), (0, 1))
STATS, REJECTED = {}, {}

# (B, C, H, W, pad, k, md, s1, s2)
TILED = [
    (1, 16, 9, 124, 24, 1, 20, 1, 2), (3, 65, 7, 260, 20, 1, 20, 1, 2), (1, 130, 9, 132, 16, 1, 20, 1, 2),
    (1, 7, 18, 28, 12, 1, 20, 1, 2), (1, 9, 1, 4, 28, 1, 20, 1, 2),
    (1, 1, 1, 4, 12, 1, 8, 1, 2), (3, 63, 17, 124, 8, 1, 8, 1, 2), (1, 9, 15, 12, 4, 1, 8, 1, 2),
    (1, 7, 1, 252, 8, 1, 4, 1, 1), (1, 16, 1, 132, 4, 1, 4, 1, 1), (3, 65, 25, 12, 0, 1, 4, 1, 1),
    (1, 130, 1, 4, 8, 1, 4, 1, 2), (1, 1, 2, 260, 4, 1, 4, 1, 2), (3, 16, 15, 132, 0, 1, 4, 1, 2),
    (1, 9, 17, 132, 17, 1, 21, 1, 2), (1, 7, 9, 4, 13, 1, 9, 1, 2), (3, 63, 10, 12, 1, 1, 5, 1, 2),
]
GENERIC = [
    (2, 3, 9, 11, 0, 1, 3, 1, 1), (1, 5, 8, 10, 2, 3, 3, 1, 1), (1, 4, 7, 9, 5, 2, 5, 1, 2),
    (1, 9, 10, 13, 10, 5, 7, 1, 3), (2, 1, 6, 7, 2, 1, 1, 1, 2), (1, 3, 5, 6, 0, 1, 0, 1, 1),
    (1, 4, 9, 12, 8, 5, 5, 1, 2), (1, 5, 11, 9, 6, 2, 7, 1, 1), (3, 9, 8, 13, 4, 3, 3, 1, 3),
    (1, 5, 12, 13, 5, 3, 3, 2, 1), (1, 4, 13, 14, 3, 1, 3, 3, 3), (1, 9, 11, 10, 6, 2, 5, 3, 2),
]
# (name, family, case, environment switch, misalign, plain entry points only)
CASES = ([("tiled-%d" % i, "tiled", c, None, 0, False) for i, c in enumerate(TILED)] +
         [("tiled-fma-C%d" % C, "tiled", (2, C, 10, 52, 20, 1, 20, 1, 2), "fma", 0, False) for C in (64, 128, 192, 256)] +
         [("tiled-flownet2", "tiled", (8, 256, 56, 128, 20, 1, 20, 1, 2), None, 0, True)] +
         [("generic-%d" % i, "generic", c, None, 0, False) for i, c in enumerate(GENERIC)] +
         [("generic-misaligned", "generic", (1, 16, 9, 12, 20, 1, 20, 1, 2), None, 4, False)])
FAMILY_CODE = {"generic": 0, "tiled": 1}


def _f2():
    import flownet2_b200
    return flownet2_b200


def _p(t):
    return P(t.data_ptr()) if t is not None else P(0)


def _ok(L, rc):
    assert rc == 0, L.fn2b200_last_error()


def _dev(t, misalign):
    v = torch.empty(t.numel() + 4, device="cuda")[misalign // 4:misalign // 4 + t.numel()].view(t.shape)
    v.copy_(t)
    assert v.data_ptr() % 16 == misalign
    return v


def kappa(K):
    return (K + 2) * U


def _K(family, direction, C, D, k):
    if family == "tiled":
        return C if direction == "forward" else D
    return k * k * C + k * k + 3 if direction == "forward" else D * (k * k + 1)


def _calls(a, b, go, gcat, prm, misalign, plain):
    """Every call of a case, on guarded outputs; returns the outputs by name."""
    L = _f2()._lib.LIB
    arena = Arena()
    B, C, H, W = a.shape
    pad, k, md, s1, s2 = prm
    D, oH, oW = go.shape[1:]
    CAT = gcat.size(1)
    st = P(torch.cuda.current_stream().cuda_stream)
    if not plain:
        assert int(L.fn2b200_correlation_forward_workspace(B, C, H, W, *prm)) == 0
        assert int(L.fn2b200_correlation_backward_workspace(B, C, H, W, *prm)) == 0
    r = {"out": arena.out((B, D, oH, oW), misalign=misalign)}
    if plain:
        _ok(L, L.fn2b200_correlation_forward(_p(a), _p(b), _p(r["out"]), B, C, H, W, *prm, 1, st))
    else:
        _ok(L, L.fn2b200_correlation_forward_ws(_p(a), _p(b), _p(r["out"]), B, C, H, W, *prm, 1, P(0), 0, st))
        for slope in SLOPES:
            r["cat", slope] = arena.out((B, CAT, oH, oW), misalign=misalign, fill=SENTINEL)
            _ok(L, L.fn2b200_correlation_forward_cat(_p(a), _p(b), _p(r["cat", slope]), CAT, CH_OFF, slope, B, C, H, W,
                                                     *prm, 1, P(0), 0, st))
    if s1 == 1:
        for need in NEEDS[:1] if plain else NEEDS:
            g1, g2 = (arena.out((B, C, H, W), misalign=misalign) if n else None for n in need)
            if plain:
                _ok(L, L.fn2b200_correlation_backward(_p(a), _p(b), _p(go), _p(g1), _p(g2), B, C, H, W, *prm, 1, st))
            else:
                _ok(L, L.fn2b200_correlation_backward_ws(_p(a), _p(b), _p(go), _p(g1), _p(g2), B, C, H, W, *prm, 1, P(0),
                                                         0, 0, st))
            r["g", need] = (g1, g2)
        if not plain:
            c1, c2 = arena.out((B, C, H, W), misalign=misalign), arena.out((B, C, H, W), misalign=misalign)
            _ok(L, L.fn2b200_correlation_backward_cat(_p(a), _p(b), _p(gcat), _p(r["cat", 0.1]), CAT, CH_OFF, 0.1,
                                                      _p(c1), _p(c2), B, C, H, W, *prm, 1, P(0), 0, 0, st))
            r["c"] = (c1, c2)
            c = r["cat", 0.1][:, CH_OFF:CH_OFF + D]
            gs = gcat[:, CH_OFF:CH_OFF + D]
            r["gm"] = _dev(torch.where(c > 0, gs, gs * 0.1), misalign)
            m1, m2 = arena.out((B, C, H, W), misalign=misalign), arena.out((B, C, H, W), misalign=misalign)
            _ok(L, L.fn2b200_correlation_backward_ws(_p(a), _p(b), _p(r["gm"]), _p(m1), _p(m2), B, C, H, W, *prm, 1,
                                                     P(0), 0, 0, st))
            r["m"] = (m1, m2)
    arena.check()
    return r


def _tensors(r):
    for key, v in r.items():
        if key == "gm":
            continue
        if isinstance(v, tuple):
            for i, t in enumerate(v):
                if t is not None:
                    yield "%s grad%d" % (key, i + 1), t
        else:
            yield str(key), v


def _check(x, ref, S, K, what, stats):
    d = (x.double() - ref).abs()
    lim = kappa(K) * S
    bad = d > lim
    if bool(bad.any()):
        i = tuple(int(v) for v in bad.nonzero()[0])
        pytest.fail("%s: %d elements beyond kappa S; the first at %s: |d| = %.3e, kappa S = %.3e, ref %.9e, got %.9e" % (
            what, int(bad.sum()), i, float(d[i]), float(lim[i]), float(ref[i]), float(x[i])))
    ratio = float(torch.where(lim > 0, d / lim.clamp_min(1e-300), torch.zeros_like(d)).max())
    glob = float(d.max() / ref.abs().max().clamp_min(1e-300))
    assert glob <= GLOBAL_TOL, "%s: max|d|/max|ref| = %.3e > %.1e" % (what, glob, GLOBAL_TOL)
    s = stats.setdefault(what.split(" ")[0], [0.0, 0.0])
    s[0], s[1] = max(s[0], ratio), max(s[1], glob)


def _profiled(call, want):
    """call() under torch.profiler; returns its result and the names of the correlation kernels that ran.  The profiler
    has been seen to drop the records of kernels that did run (their outputs were written; see also
    tests/test_gpu_kernel_coverage.py), so when a name in `want` is missing the call runs once more under a fresh
    profiler and the kernels of both records count."""
    names = set()
    for attempt in range(2):
        with cuda_profile() as prof:
            res = call()
            torch.cuda.synchronize()
        names |= {e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and "corr" in e.name}
        if attempt == 0:
            first = res
        if all(any(w in n for n in names) for w in want):
            break
    return first, names


@pytest.mark.parametrize("name,family,case,env,misalign,plain", CASES, ids=[c[0] for c in CASES])
def test_corr_fp32_vs_fp64(name, family, case, env, misalign, plain, monkeypatch):
    f = _f2()
    L = f._lib.LIB
    B, C, H, W = case[:4]
    prm = case[4:]
    pad, k, md, s1, s2 = prm
    kr, dr, oH, oW = torch_ref.corr_geometry(H, W, *prm)
    D = (2 * dr + 1) ** 2
    if env:
        assert L.fn2b200_correlation_path(C, H, W, *prm) == 2
        monkeypatch.setenv("FN2B200_CORR_FWD", env)
        monkeypatch.setenv("FN2B200_CORR_BWD", env)
    if not misalign and not plain:
        assert L.fn2b200_correlation_path(C, H, W, *prm) == FAMILY_CODE[family]
    g = torch.Generator(device="cuda").manual_seed(sum(case) + 17 * C)
    a, b = (_dev(torch.randn(B, C, H, W, device="cuda", generator=g), misalign) for _ in range(2))
    go = _dev(torch.randn(B, D, oH, oW, device="cuda", generator=g), misalign)
    gcat = _dev(torch.randn(B, D + CH_OFF + 2, oH, oW, device="cuda", generator=g), misalign)

    want = {"corr_fwd_%s_kernel" % family} | ({"corr_bwd_%s_kernel" % family} if s1 == 1 else set())
    r, ran = _profiled(lambda: _calls(a, b, go, gcat, prm, misalign, plain), want)
    assert {w for w in want if any(w in n for n in ran)} == want, sorted(ran)
    assert all(any(w in n for w in want) for n in ran), "kernels of another family ran: %s" % sorted(ran)

    # bit-for-bit invariances
    out = r["out"]
    if not plain:
        for slope in SLOPES:
            cat = r["cat", slope]
            assert torch.equal(cat[:, CH_OFF:CH_OFF + D], torch.where(out > 0, out, out * slope)), slope
            assert bool((cat[:, :CH_OFF] == SENTINEL).all() and (cat[:, CH_OFF + D:] == SENTINEL).all()), slope
    if s1 == 1:
        g1, g2 = r["g", (1, 1)]
        for need in NEEDS[1:] if not plain else ():
            x1, x2 = r["g", need]
            assert x1 is None or torch.equal(x1, g1), need
            assert x2 is None or torch.equal(x2, g2), need
        if not plain:
            assert all(torch.equal(x, y) for x, y in zip(r["c"], r["m"])), "backward_cat != backward of the masked gradient"

    # fp64, element by element
    stats = STATS.setdefault(family, {})
    a64, b64 = a.double(), b.double()
    aa, ba = a64.abs(), b64.abs()
    ref = torch_ref.correlation64(a64, b64, *prm)
    S = torch_ref.correlation64(aa, ba, *prm)
    Kf = _K(family, "forward", C, D, k)
    _check(out, ref, S, Kf, "forward", stats)
    for slope in SLOPES if not plain else ():
        _check(r["cat", slope][:, CH_OFF:CH_OFF + D], torch.where(ref > 0, ref, ref * slope), S, Kf,
               "forward_cat slope %g" % slope, stats)
    Kb = _K(family, "backward", C, D, k)
    if s1 == 1:
        todo = [("backward", go, r["g", (1, 1)])]
        if not plain:
            c = r["cat", 0.1][:, CH_OFF:CH_OFF + D].double()
            gs = gcat[:, CH_OFF:CH_OFF + D].double()
            todo.append(("backward_cat", torch.where(c > 0, gs, gs * 0.1), r["c"]))
        for what, gout, grads in todo:
            g64 = gout.double()
            refs = torch_ref.correlation64_backward(a64, b64, g64, *prm)
            Ss = torch_ref.correlation64_backward(aa, ba, g64.abs(), *prm)
            for i in range(2):
                _check(grads[i], refs[i], Ss[i], Kb, "%s grad%d" % (what, i + 1), stats)
            del refs, Ss
    del ref, S

    # a repeated call, and the first and last samples alone
    again = dict(_tensors(_calls(a, b, go, gcat, prm, misalign, plain)))
    for key, t in _tensors(r):
        assert torch.equal(t, again[key]), "%s: a repeated call gave other bits" % key
    del again
    for n in sorted({0, B - 1}) if B > 1 else ():
        sub = dict(_tensors(_calls(*(_dev(t[n:n + 1].clone(), misalign) for t in (a, b, go, gcat)), prm, misalign, plain)))
        for key, t in _tensors(r):
            assert torch.equal(t[n:n + 1], sub[key]), "%s: sample %d alone differs from the batch of %d" % (key, n, B)

    # negative controls, on the forward and the two-gradient backward
    if plain:
        return
    for v in torch_ref.VARIANTS:
        fm, m1, m2 = torch_ref.variant_edges(v, a.shape, *prm, device="cuda")
        if bool(fm.any()):
            rv = torch_ref.correlation64(a64, b64, *prm, variant=v)
            Sv = torch_ref.correlation64(aa, ba, *prm, variant=v)
            if bool(((out.double() - rv).abs() > kappa(Kf) * Sv)[fm].any()):
                REJECTED.setdefault(v, set()).add((family, "forward"))
        if s1 == 1 and bool(m1.any() or m2.any()):
            rv = torch_ref.correlation64_backward(a64, b64, go.double(), *prm, variant=v)
            Sv = torch_ref.correlation64_backward(aa, ba, go.double().abs(), *prm, variant=v)
            for x, rr, ss, m in zip(r["g", (1, 1)], rv, Sv, (m1, m2)):
                if bool(((x.double() - rr).abs() > kappa(Kb) * ss)[m].any()):
                    REJECTED.setdefault(v, set()).add((family, "backward"))


def test_zz_every_control_rejected():
    """Runs last: every variant was rejected somewhere, `replicate` in each family and direction; prints the largest
    ratios of the run."""
    if not STATS:
        pytest.skip("no correlation case ran")
    for fam, st in sorted(STATS.items()):
        for what, (ratio, glob) in sorted(st.items()):
            print("STATS %-8s %-14s max|d|/(kappa S) %.3f  max|d|/max|ref64| %.2e" % (fam, what, ratio, glob))
    for v in torch_ref.VARIANTS:
        print("REJECTED %-12s %s" % (v, sorted(REJECTED.get(v, ()))))
    missing = [v for v in torch_ref.VARIANTS if not REJECTED.get(v)]
    assert not missing, "variants never rejected: %s" % missing
    want = {(f, d) for f in ("tiled", "generic") for d in ("forward", "backward")}
    assert want <= REJECTED["replicate"], "replicate not rejected for %s" % sorted(want - REJECTED["replicate"])
