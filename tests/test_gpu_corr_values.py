"""Every correlation kernel family across fp32's value range, element by element against fp64, and the footprint of a
single NaN or inf input element.  The value classes, bounds and footprint models are tests/corr_values.py's.

Families: the tensor-core kernels at C = 64, 192, 256 (H, W even, a ragged last tile); the TMA-tiled FP32-FMA kernels at
the same configuration under FN2B200_CORR_FWD/BWD=fma and at pad < md; the generic kernels at kernel_size 3 and on
operands 4 bytes past a 16-byte boundary.  The profiler confirms which family ran.  Calls go through the C ABI on
guarded buffers (tests/guarded.py): forward, forward_cat (LeakyReLU slopes 0.1 and 0), both gradients, and backward_cat
(slope 0.1), which must equal the plain backward of the masked gradient.  Outputs that may hold NaN or inf are poisoned
with a signalling NaN no kernel writes, so every element must still be written.

- exact class: every family bit-equal to fp32(ref64), except the tensor-core kernels at C = 192, whose scaling by
  rn(1/C) leaves them within 1 ulp.
- bound classes: |x - ref64| <= the per-element bound (corr_values.bound_tc_* / bound_fma), finite outputs.
- overflow: +-inf exactly where ref64 != 0 (every product of a sum overflows with one sign), 0 elsewhere; forward_cat's
  slope 0 gives NaN on -inf (-inf * 0), as torch does.
- probes: one NaN in input1, input2 or gradOutput at each placement of corr_values.probe_positions (+inf too at the
  interior and border ones), or a NaN in backward_cat's concat activation.  Forward: the non-finite mask is the reference's (the tensor-core and tiled
  kernels multiply the zero padding, inf * 0 = NaN, as the reference does), NaN wherever the reference is NaN; the
  generic kernels skip padding taps, so their mask is the in-image reach.  Backward: tensor cores, reference mask <=
  kernel mask <= reference mask + corr_values.tc_backward_superset; tiled, corr_values.tiled_backward_mask (the
  reference's at pad = md); generic, the in-image reach.  Every element outside the kernel's mask meets the finite
  bound against the reference with the probe set to 0.
- the split pass: the workspace's bf16 hi / lo of every fp32 exponent with boundary mantissas equal corr_values.split_bf16
  bit for bit (NaN by isnan).

The largest |d| / bound per family, direction and class is recorded (record_property) and printed by the last test.
"""
import ctypes
import zlib

import pytest
import torch

import corr_values as cv
import torch_ref
from guarded import POISON_SNAN, SENTINEL, Arena
from util import cuda_profile

pytestmark = pytest.mark.gpu
P = ctypes.c_void_p
CH_OFF, SLOPES = 3, (0.1, 0.0)
TC_PRM = (20, 1, 20, 1, 2)
# name -> (family, (B, C, H, W), (pad, k, md, s1, s2), environment switch, misalignment in bytes)
FAMILIES = {
    "tc-C64": ("tc", (1, 64, 34, 70), TC_PRM, None, 0),
    "tc-C192": ("tc", (1, 192, 34, 70), TC_PRM, None, 0),
    "tc-C256": ("tc", (1, 256, 34, 38), TC_PRM, None, 0),
    "tiled-fma": ("tiled", (1, 64, 34, 72), TC_PRM, "fma", 0),          # the tiled kernels need W % 4 == 0
    "tiled-pad16": ("tiled", (1, 16, 34, 56), (16, 1, 20, 1, 2), None, 0),
    "generic-k3": ("generic", (2, 5, 12, 13), (5, 3, 3, 1, 1), None, 0),
    "generic-misaligned": ("generic", (1, 16, 9, 12), TC_PRM, None, 4),
}
PROBE_FAMILIES = ("tc-C64", "tiled-fma", "tiled-pad16", "generic-k3")
STATS = {}


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


def _shapes(shape, prm):
    kr, dr, oH, oW = torch_ref.corr_geometry(shape[2], shape[3], *prm)
    D = (2 * dr + 1) ** 2
    return (shape[0], D, oH, oW), D, kr


def _calls(a, b, go, gcat, prm, misalign, poison):
    """Every call of a case on guarded outputs; returns the outputs by name and the workspace."""
    L = _f2()._lib.LIB
    arena = Arena(poison=poison)
    B, C, H, W = a.shape
    D, oH, oW = go.shape[1:]
    CAT = gcat.size(1)
    st = P(torch.cuda.current_stream().cuda_stream)
    nws = int(L.fn2b200_correlation_forward_workspace(B, C, H, W, *prm))
    ws = arena.workspace(nws)
    r = {"out": arena.out((B, D, oH, oW), misalign=misalign)}
    _ok(L, L.fn2b200_correlation_forward_ws(_p(a), _p(b), _p(r["out"]), B, C, H, W, *prm, 1, _p(ws), nws, st))
    for slope in SLOPES:
        r["cat", slope] = arena.out((B, CAT, oH, oW), misalign=misalign, fill=SENTINEL)
        _ok(L, L.fn2b200_correlation_forward_cat(_p(a), _p(b), _p(r["cat", slope]), CAT, CH_OFF, slope, B, C, H, W, *prm,
                                                 1, _p(ws), nws, st))
    g1, g2 = arena.out((B, C, H, W), misalign=misalign), arena.out((B, C, H, W), misalign=misalign)
    _ok(L, L.fn2b200_correlation_backward_ws(_p(a), _p(b), _p(go), _p(g1), _p(g2), B, C, H, W, *prm, 1, _p(ws), nws, 0,
                                             st))
    r["g"] = (g1, g2)
    c1, c2 = arena.out((B, C, H, W), misalign=misalign), arena.out((B, C, H, W), misalign=misalign)
    _ok(L, L.fn2b200_correlation_backward_cat(_p(a), _p(b), _p(gcat), _p(r["cat", 0.1]), CAT, CH_OFF, 0.1, _p(c1),
                                              _p(c2), B, C, H, W, *prm, 1, _p(ws), nws, 0, st))
    r["c"] = (c1, c2)
    c = r["cat", 0.1][:, CH_OFF:CH_OFF + D]
    gs = gcat[:, CH_OFF:CH_OFF + D]
    r["gm"] = _dev(torch.where(c > 0, gs, gs * 0.1), misalign)
    m1, m2 = arena.out((B, C, H, W), misalign=misalign), arena.out((B, C, H, W), misalign=misalign)
    _ok(L, L.fn2b200_correlation_backward_ws(_p(a), _p(b), _p(r["gm"]), _p(m1), _p(m2), B, C, H, W, *prm, 1, _p(ws), nws,
                                             0, st))
    r["m"] = (m1, m2)
    arena.check()
    for slope in SLOPES:
        cat = r["cat", slope]
        assert bool((cat[:, :CH_OFF] == SENTINEL).all() and (cat[:, CH_OFF + D:] == SENTINEL).all())
    return r, ws


def _same(x, y):
    """Equal, NaN matching NaN."""
    return bool(((x == y) | (torch.isnan(x) & torch.isnan(y))).all())


def _setup(name, monkeypatch):
    fam, shape, prm, env, mis = FAMILIES[name]
    gshape, D, kr = _shapes(shape, prm)
    L = _f2()._lib.LIB
    B, C, H, W = shape
    if env:
        monkeypatch.setenv("FN2B200_CORR_FWD", env)
        monkeypatch.setenv("FN2B200_CORR_BWD", env)
    elif not mis:
        assert L.fn2b200_correlation_path(C, H, W, *prm) == {"generic": 0, "tiled": 1, "tc": 2}[fam]
    return fam, shape, prm, mis, gshape, D, kr


def _inputs(a, b, go, gcat, mis):
    return tuple(_dev(t.cuda(), mis) for t in (a, b, go, gcat))


def _gcat(go, seed):
    B, D, oH, oW = go.shape
    g = torch.Generator().manual_seed(seed)
    gcat = torch.randn((B, D + CH_OFF + 2, oH, oW), generator=g)
    gcat[:, CH_OFF:CH_OFF + D] = go
    return gcat


def _K(fam, direction, C, D, k):
    if fam == "tiled":
        return C if direction == "forward" else D
    if fam == "generic":
        return k * k * C + k * k + 3 if direction == "forward" else D * (k * k + 1)
    return C if direction == "forward" else D


def _bounds(fam, a, b, go, prm, k):
    """(forward bound, (grad1 bound, grad2 bound)) in fp64 on the GPU."""
    C, D = a.size(1), go.size(1)
    a64, b64, g64 = a.double(), b.double(), go.double()
    if fam == "tc":
        return cv.bound_tc_forward(a64.float(), b64.float(), prm), cv.bound_tc_backward(a64.float(), b64.float(),
                                                                                         g64.float(), prm)
    S = torch_ref.correlation64(a64.abs(), b64.abs(), *prm)
    Ss = torch_ref.correlation64_backward(a64.abs(), b64.abs(), g64.abs(), *prm)
    return (cv.bound_fma(S, _K(fam, "forward", C, D, k)),
            tuple(cv.bound_fma(s, _K(fam, "backward", C, D, k)) for s in Ss))


def _ratio(x, ref, lim, what, mask=None):
    d = (x.double() - ref).abs()
    if mask is not None:
        d, ref, lim, x = d[mask], ref[mask], lim[mask], x[mask]
    bad = ~(d <= lim)
    if bool(bad.any()):
        i = int(bad.nonzero()[0][0]) if bad.dim() == 1 else tuple(int(v) for v in bad.nonzero()[0])
        pytest.fail("%s: %d elements beyond the bound; the first at %s: |d| = %.3e, bound %.3e, ref %.9e, got %.9e" % (
            what, int(bad.sum()), i, float(d[i]), float(lim[i]), float(ref[i]), float(x[i])))
    return float(torch.where(lim > 0, d / lim.clamp_min(1e-300), torch.zeros_like(d)).max()) if d.numel() else 0.0


def _stat(key, r):
    STATS[key] = max(STATS.get(key, 0.0), r)


def _profiled_family(call, fam):
    """call() under torch.profiler; returns its result and asserts that the family's kernels, and no others, ran."""
    want = {"corr_fwd_%s_kernel" % fam, "corr_bwd_%s_kernel" % fam}
    allowed = want | ({"corr_tc_split_kernel"} if fam == "tc" else set())
    names = set()
    for attempt in range(2):              # the profiler can drop records of kernels that ran
        with cuda_profile() as prof:
            res = call()
            torch.cuda.synchronize()
        names |= {e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and "corr" in e.name}
        if attempt == 0:
            first = res
        if all(any(w in n for n in names) for w in want):
            break
    assert all(any(w in n for n in names) for w in want), sorted(names)
    assert all(any(w in n for w in allowed) for n in names), "kernels of another family ran: %s" % sorted(names)
    return first


# ------------------------------------------------------------------------------------------------
# Value classes
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cls", cv.CLASSES)
@pytest.mark.parametrize("name", list(FAMILIES))
def test_corr_value_class(name, cls, monkeypatch, record_property):
    fam, shape, prm, mis, gshape, D, kr = _setup(name, monkeypatch)
    k = prm[1]
    B, C, H, W = shape
    if fam == "generic" and k > 1 and cls == "huge_go":
        pytest.skip("the generic backward sums each k x k window of gradOutput before multiplying, so a window of "
                    "values near FLT_MAX overflows where the reference's products do not (DESIGN section 2)")
    a, b, go = cv.make(cls, shape, gshape, zlib.crc32((name + cls).encode()) & 0xFFFF)
    a, b, go, gcat = _inputs(a, b, go, _gcat(go, 1), mis)
    poison = POISON_SNAN if cls == "overflow" else None
    call = lambda: _calls(a, b, go, gcat, prm, mis, poison)      # noqa: E731
    r, _ = _profiled_family(call, fam) if cls == "exact" else call()
    out, (g1, g2) = r["out"], r["g"]
    D_ = go.size(1)
    for slope in SLOPES:
        assert _same(r["cat", slope][:, CH_OFF:CH_OFF + D_], torch.where(out > 0, out, out * slope)), slope
    assert all(_same(x, y) for x, y in zip(r["c"], r["m"])), "backward_cat != backward of the masked gradient"

    a64, b64, g64 = a.double(), b.double(), go.double()
    ref = torch_ref.correlation64(a64, b64, *prm)
    refs = torch_ref.correlation64_backward(a64, b64, g64, *prm)
    if cls == "exact":
        exact = fam != "tc" or (C & (C - 1)) == 0
        for x, rr, what in ((out, ref, "forward"), (g1, refs[0], "grad1"), (g2, refs[1], "grad2")):
            want = rr.float()
            if exact:
                assert torch.equal(x, want), "%s: %d elements differ from fp32(ref64)" % (what, int((x != want).sum()))
            else:
                ulp = (torch.nextafter(want.abs(), torch.full_like(want, float("inf"))) - want.abs())
                assert bool(((x - want).abs() <= ulp).all()), "%s: more than 1 ulp from fp32(ref64)" % what
        return
    if cls == "overflow":
        for x, rr, what in ((out, ref, "forward"), (g1, refs[0], "grad1"), (g2, refs[1], "grad2")):
            want = torch.where(rr == 0, torch.zeros_like(rr), torch.sign(rr) * float("inf")).float()
            assert torch.equal(x, want), "%s: %d elements are not the expected +-inf / 0" % (what, int((x != want).sum()))
        return
    assert bool(torch.isfinite(out).all() and torch.isfinite(g1).all() and torch.isfinite(g2).all()), \
        "finite inputs gave non-finite outputs"
    bf, (b1, b2) = _bounds(fam, a, b, go, prm, k)
    ratios = {"forward": _ratio(out, ref, bf, "forward")}
    for slope in SLOPES:
        ratios["forward_cat"] = max(ratios.get("forward_cat", 0.0), _ratio(
            r["cat", slope][:, CH_OFF:CH_OFF + D_], torch.where(ref > 0, ref, ref * slope), bf, "forward_cat %g" % slope))
    ratios["grad1"] = _ratio(g1, refs[0], b1, "grad1")
    ratios["grad2"] = _ratio(g2, refs[1], b2, "grad2")
    mrefs = torch_ref.correlation64_backward(a64, b64, r["gm"].double(), *prm)
    mb = _bounds(fam, a, b, r["gm"], prm, k)[1]
    ratios["backward_cat"] = max(_ratio(r["c"][i], mrefs[i], mb[i], "backward_cat grad%d" % (i + 1)) for i in range(2))
    for what, v in ratios.items():
        _stat((name, what, cls), v)
        record_property("ratio_%s" % what, "%.3e" % v)


def test_tc_subnormals_exact():
    """Exact subnormal arithmetic on the tensor cores: an fp32 subnormal input (a bf16 subnormal hi, lo = 0) times 1,
    and two normal inputs whose product is an fp32 subnormal, each the only non-zero term of its sum.  The results are
    exact unless the tensor core flushes subnormal inputs or partial sums to zero; the test pins which holds."""
    L = _f2()._lib.LIB
    B, C, H, W = 1, 64, 16, 32
    a = torch.zeros(B, C, H, W, device="cuda")
    b = torch.zeros_like(a)
    a[0, 0, 4, 4], b[0, 0, 4, 4] = 2.0 ** -130, 1.0            # bf16 subnormal input, result 2^-136
    a[0, 1, 8, 8], b[0, 1, 8, 8] = 2.0 ** -70, 2.0 ** -70      # subnormal product 2^-140, result 2^-146
    r, _ = _calls(a, b, torch.zeros(B, 441, H, W, device="cuda"), torch.zeros(B, 441 + CH_OFF + 2, H, W, device="cuda"),
                  TC_PRM, 0, None)
    d0 = 10 * 21 + 10                                          # displacement (0, 0)
    got_in, got_prod = float(r["out"][0, d0, 4, 4]), float(r["out"][0, d0, 8, 8])
    print("TC_SUBNORMAL input %.6e (exact %.6e)  product %.6e (exact %.6e)" % (got_in, 2.0 ** -136, got_prod, 2.0 ** -146))
    assert L.fn2b200_correlation_path(C, H, W, *TC_PRM) == 2
    assert got_in == 2.0 ** -136, "the tensor core flushed a bf16 subnormal input"
    assert got_prod == 2.0 ** -146, "the tensor core flushed a subnormal product"


# ------------------------------------------------------------------------------------------------
# Split pass
# ------------------------------------------------------------------------------------------------
def test_tc_split_pass_bits():
    """The split pass's workspace, [hi(in1) | lo(in1) | hi(in2) | lo(in2)], each [n][class][yc][xc][c] bf16, equals
    split_bf16 bit for bit on every fp32 exponent with boundary mantissas and on the specials (NaN by isnan)."""
    bits = cv.catalogue_bits()
    B, C, H, W = 1, 64, 12, 16
    n = B * C * H * W
    vals = cv.f32_from_bits(bits.repeat((n + len(bits) - 1) // len(bits))[:n])
    g = torch.Generator().manual_seed(2)
    a = vals.view(B, C, H, W)
    b = vals[torch.randperm(n, generator=g)].view(B, C, H, W)
    gshape, D, _ = _shapes((B, C, H, W), TC_PRM)
    a, b = a.cuda(), b.cuda()
    L = _f2()._lib.LIB
    st = P(torch.cuda.current_stream().cuda_stream)
    arena = Arena(poison=POISON_SNAN)
    nws = int(L.fn2b200_correlation_forward_workspace(B, C, H, W, *TC_PRM))
    ws = arena.workspace(nws)
    out = arena.out(gshape)
    _ok(L, L.fn2b200_correlation_forward_ws(_p(a), _p(b), _p(out), B, C, H, W, *TC_PRM, 1, _p(ws), nws, st))
    arena.check()
    w = ws.view(torch.int16).view(4, B, 4, H // 2, W // 2, C).cpu()
    for i, x in enumerate((a, b)):
        cls = x.cpu().view(B, C, H // 2, 2, W // 2, 2).permute(0, 3, 5, 2, 4, 1).reshape(B, 4, H // 2, W // 2, C)
        hi, lo = cv.split_bf16(cls)
        for got, want, what in ((w[2 * i], hi, "hi"), (w[2 * i + 1], lo, "lo")):
            gf, wf = got.view(torch.bfloat16).float(), want.float()
            nan = torch.isnan(wf)
            assert torch.equal(torch.isnan(gf), nan), "input%d %s: NaN placement differs" % (i + 1, what)
            diff = (got != want.view(torch.int16)) & ~nan
            if bool(diff.any()):
                j = tuple(int(v) for v in diff.nonzero()[0])
                pytest.fail("input%d %s: %d values differ; x = %r (0x%08X): got 0x%04X, model 0x%04X" % (
                    i + 1, what, int(diff.sum()), float(cls[j]), int(cv.bits_of(cls[j].reshape(1))[0]),
                    int(got[j]) & 0xFFFF, int(want.view(torch.int16)[j]) & 0xFFFF))


# ------------------------------------------------------------------------------------------------
# Non-finite probes
# ------------------------------------------------------------------------------------------------
def _probes(name):
    fam, shape, prm = FAMILIES[name][:3]
    pos = cv.probe_positions(shape) if shape[2] >= 30 else {
        "interior": (shape[0] - 1, shape[1] // 2, shape[2] // 2, shape[3] // 2), "border": (0, 0, 0, shape[3] - 1),
        "last_channel": (0, shape[1] - 1, shape[2] - 1, 1)}
    gshape, D, _ = _shapes(shape, prm)
    out = []
    for which in ("a", "b", "go"):
        for pname, p in pos.items():
            if which == "go":
                p = (p[0], min(p[1] * 7, D - 1), min(p[2], gshape[2] - 1), min(p[3], gshape[3] - 1))
            for val in ("nan", "inf") if pname in ("interior", "border") else ("nan",):
                out.append((name, which, pname, p, val))
    out.append((name, "act", "interior", (0, D // 3, gshape[2] // 2, gshape[3] // 2), "nan"))
    return out


PROBES = [p for n in PROBE_FAMILIES for p in _probes(n)]


@pytest.mark.parametrize("name,which,pname,pos,val", PROBES, ids=["%s-%s-%s-%s" % (p[0], p[1], p[2], p[4]) for p in PROBES])
def test_corr_probe(name, which, pname, pos, val, monkeypatch):
    fam, shape, prm, mis, gshape, D, kr = _setup(name, monkeypatch)
    k = prm[1]
    g = torch.Generator().manual_seed(11)
    a, b, go = (torch.randn(s, generator=g) for s in (shape, shape, gshape))
    gcat = _gcat(go, 12)
    v = float("nan") if val == "nan" else float("inf")
    t = {"a": a, "b": b, "go": go}
    if which == "act":
        # a NaN in the concat activation that backward_cat reads: NaN > 0 is false, so its gradient takes the slope
        a, b, go, gcat = _inputs(a, b, go, gcat, mis)
        r, _ = _calls(a, b, go, gcat, prm, mis, None)
        cat = r["cat", 0.1]
        cat[pos[0], CH_OFF + pos[1], pos[2], pos[3]] = v
        L = _f2()._lib.LIB
        st = P(torch.cuda.current_stream().cuda_stream)
        B, C, H, W = shape
        nws = int(L.fn2b200_correlation_forward_workspace(B, C, H, W, *prm))
        arena = Arena()
        ws = arena.workspace(nws)
        c1, c2 = arena.out(shape, misalign=mis), arena.out(shape, misalign=mis)
        _ok(L, L.fn2b200_correlation_backward_cat(_p(a), _p(b), _p(gcat), _p(cat), gcat.size(1), CH_OFF, 0.1, _p(c1),
                                                  _p(c2), B, C, H, W, *prm, 1, _p(ws), nws, 0, st))
        arena.check()
        cs = cat[:, CH_OFF:CH_OFF + D]
        gs = gcat[:, CH_OFF:CH_OFF + D]
        gm = _dev(torch.where(cs > 0, gs, gs * 0.1), mis)
        m1, m2 = torch.empty_like(c1), torch.empty_like(c2)
        _ok(L, L.fn2b200_correlation_backward_ws(_p(a), _p(b), _p(gm), _p(m1), _p(m2), B, C, H, W, *prm, 1, _p(ws), nws,
                                                 0, st))
        torch.cuda.synchronize()
        assert torch.equal(c1, m1) and torch.equal(c2, m2)
        return
    t[which][pos] = v
    a, b, go = t["a"], t["b"], t["go"]
    gcat[:, CH_OFF:CH_OFF + D] = go
    a, b, go, gcat = _inputs(a, b, go, gcat, mis)
    r, _ = _calls(a, b, go, gcat, prm, mis, POISON_SNAN)
    out, grads = r["out"], r["g"]
    for slope in SLOPES:
        assert _same(r["cat", slope][:, CH_OFF:CH_OFF + D], torch.where(out > 0, out, out * slope)), slope
    assert all(_same(x, y) for x, y in zip(r["c"], r["m"])), "backward_cat != backward of the masked gradient"

    a64, b64, g64 = a.double(), b.double(), go.double()
    what = "%s %s probe %s at %s" % (val, which, pname, pos)
    km = ~torch.isfinite(out)
    if which != "go":
        ref = torch_ref.correlation64(a64, b64, *prm)
        rm = ~torch.isfinite(ref)
        if fam == "generic":
            want = cv.inimage_reach(which, shape, gshape, pos, prm, device="cuda")[0]
        else:
            want = rm
            nan = torch.isnan(ref)
            assert bool(torch.isnan(out[nan]).all()), "%s: forward not NaN where the reference is" % what
            inf = torch.isinf(ref)
            if fam != "tc":
                assert torch.equal(out[inf], ref[inf].float()), "%s: forward not the reference's inf" % what
        assert torch.equal(km, want), "%s: forward mask %d elements, model %d, %d differ" % (
            what, int(km.sum()), int(want.sum()), int((km != want).sum()))
    else:
        assert not bool(km.any())
    rms = cv.ref_mask_backward(a64, b64, g64, prm)
    kms = tuple(~torch.isfinite(x) for x in grads)
    for i in range(2):
        gw = "%s: gradInput%d" % (what, i + 1)
        if fam == "tc":
            sup = rms[i].clone()
            if (which, i) in (("a", 1), ("b", 0)):
                sup |= cv.tc_backward_superset(which, shape, pos, device="cuda")
            assert bool((rms[i] <= kms[i]).all()), "%s: the reference reaches %d elements the kernel leaves finite" % (
                gw, int((rms[i] & ~kms[i]).sum()))
            assert bool((kms[i] <= sup).all()), "%s: %d non-finite elements outside the modelled footprint" % (
                gw, int((kms[i] & ~sup).sum()))
            if pname == "out_of_band" and (which, i) in (("a", 1), ("b", 0)):
                assert int(kms[i].sum()) > int(rms[i].sum()), "%s: a live unit's out-of-band column reaches" % gw
        else:
            if fam == "tiled":
                want = cv.tiled_backward_mask(a64, b64, g64, prm)[i]
            else:
                want = cv.inimage_reach(which, shape, gshape, pos, prm, device="cuda")[i + 1]
            assert torch.equal(kms[i], want), "%s: mask of %d elements, model %d (reference %d), %d differ" % (
                gw, int(kms[i].sum()), int(want.sum()), int(rms[i].sum()), int((kms[i] != want).sum()))
    # every element outside the kernel's footprint meets the finite bound of the same call with the probe at 0
    z = {"a": a64.clone(), "b": b64.clone(), "go": g64.clone()}
    z[which][pos] = 0
    ref0 = torch_ref.correlation64(z["a"], z["b"], *prm)
    refs0 = torch_ref.correlation64_backward(z["a"], z["b"], z["go"], *prm)
    bf, bb = _bounds(fam, z["a"].float(), z["b"].float(), z["go"].float(), prm, k)
    _stat((name, "forward", "probe"), _ratio(out, ref0, bf, what + " forward", ~km))
    for i in range(2):
        _stat((name, "grad%d" % (i + 1), "probe"), _ratio(grads[i], refs0[i], bb[i], what + " grad", ~kms[i]))


def test_zz_report():
    """Runs last: prints the largest |d| / bound per family, direction and class."""
    if not STATS:
        pytest.skip("no case ran")
    for (name, what, cls), v in sorted(STATS.items()):
        print("RATIO %-20s %-13s %-10s %.3e" % (name, what, cls, v))
