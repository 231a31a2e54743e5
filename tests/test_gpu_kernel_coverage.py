"""Every compiled kernel instantiation, launched and checked against the CPU oracle on poisoned, guarded buffers.

tests/kernel_manifest.py maps each `__global__` instantiation of libfn2b200.so to the case below that launches it
(tests/test_kernel_manifest_cpu.py keeps the map equal to the library's symbol table).  Every case runs under
torch.profiler and fails if an instantiation the manifest gives it was not among the kernels it launched, so a dispatch
change that silently stops reaching a variant fails here.

Buffers (DESIGN section 9):
- every output, gradient and workspace is a view inside a larger allocation filled with one NaN bit pattern; after the
  call the bytes around each view must still hold it (no write outside the buffer), and every element of an output
  view must be finite (no element left unwritten) and match the reference;
- workspaces are exactly the size the library's query returns;
- views start 256 bytes into their allocation (16- and 128-byte aligned); the `misaligned` cases start 4 bytes later.
"""
import ctypes

import numpy as np
import pytest
import torch

import torch_ref
import upsample_ref as ur
from guarded import SENTINEL, Arena
from kernel_manifest import KERNELS
from oracle import cpu as orc
from util import assert_close, cuda_profile

pytestmark = pytest.mark.gpu
P = ctypes.c_void_p
TOL = 1e-4


def _f2():
    import flownet2_b200
    return flownet2_b200


def _stream():
    return P(torch.cuda.current_stream().cuda_stream)


def _p(t):
    return P(t.data_ptr()) if t is not None else P(0)


def _kernel_names(prof):
    """Launched kernels, named as c++filt prints the symbol without its argument list."""
    return {e.name.split("(")[0] for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA}


@pytest.fixture(autouse=True)
def launched_kernels(request, monkeypatch):
    """Profiles the case (util.cuda_profile); afterwards every instantiation the manifest assigns to it must have run.
    A case that already failed is not reported twice.  The profiler has been seen to lose the record of the first
    kernel the library launches in a profiling session (a case's forward missing while its backward was recorded), so
    a case whose record is missing runs twice more in one fresh session before it fails: every kernel of the second
    run follows one already recorded.  (Requesting monkeypatch keeps the environment the case set until those runs are
    over.)"""
    want = {k for k, v in KERNELS.items() if v == request.node.name}
    failed_before = request.session.testsfailed
    with cuda_profile() as prof:
        yield
        torch.cuda.synchronize()
    if request.session.testsfailed != failed_before or not (want - _kernel_names(prof)):
        return
    with cuda_profile() as prof:
        for _ in range(2):
            request.node.runtest()
            torch.cuda.synchronize()
    missing = want - _kernel_names(prof)
    assert not missing, "%s did not launch %s; recorded %s" % (request.node.name, sorted(missing),
                                                              sorted(_kernel_names(prof)))


@pytest.fixture
def arena():
    return Arena()


def _rand(shape, seed, scale=1.0, shift=0.0):
    return (torch.rand(*shape, generator=torch.Generator().manual_seed(seed)) - shift) * scale


def _randn(shape, seed, scale=1.0):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed)) * scale


def _dev(t, misalign=0):
    """t on the GPU; misalign=4 puts it 4 bytes past a 16-byte boundary."""
    if not misalign:
        return t.cuda()
    v = torch.empty(t.numel() + 4, device="cuda")[misalign // 4:misalign // 4 + t.numel()].view(t.shape)
    v.copy_(t)
    assert v.data_ptr() % 16 == misalign
    return v


# ------------------------------------------------------------------------------------------------
# ChannelNorm
# ------------------------------------------------------------------------------------------------
def _channelnorm_case(arena, x, dtype, misalign):
    F2 = _f2().functional
    B, C, H, W = x.shape
    xd = _dev(x, misalign) if dtype == torch.float32 else _dev(x).to(dtype)
    if misalign and dtype != torch.float32:
        xd = torch.empty(xd.numel() + 2, dtype=dtype, device="cuda")[2:].view(xd.shape).copy_(xd)
        assert xd.data_ptr() % 16 == misalign
    g = _randn((B, 1, H, W), 2)
    gd = g.cuda().to(dtype) if dtype != torch.float32 else _dev(g, misalign)
    out = F2.channelnorm_forward(xd, out=arena.out((B, 1, H, W), dtype, misalign))
    gin = F2.channelnorm_backward(xd, out, gd, out=arena.out((B, C, H, W), dtype, misalign))
    arena.check()
    x32, o32, g32 = (t.float().cpu().numpy() for t in (xd, out, gd))
    return x32, o32, g32, out.float().cpu().numpy(), gin.float().cpu().numpy()


@pytest.mark.parametrize("C", [1, 2, 3, 4, 5])
def test_channelnorm_fp32(arena, C):
    x = _rand((2, C, 6, 10), C, 2.0, 0.5)                 # hw = 60: the 4-wide kernels
    x[0, :, 0, :4] = 0.0                                   # |x| = 0 pixels: output and gradient exactly 0
    xn, on, gn, out, gin = _channelnorm_case(arena, x, torch.float32, 0)
    assert_close(out, orc.channelnorm_forward(xn), TOL, "channelnorm C=%d forward" % C)
    assert_close(gin, orc.channelnorm_backward(xn, on, gn), TOL, "channelnorm C=%d backward" % C)
    # fp64 second opinion: sqrt(sum x^2) and its autograd gradient (x / n vs the kernels' x / (n + 1e-9))
    x64 = torch.from_numpy(xn).double().requires_grad_()
    n64 = torch_ref.channelnorm(x64)
    n64.backward(torch.from_numpy(gn).double())
    assert_close(out, n64.detach().numpy(), TOL, "channelnorm C=%d forward vs fp64" % C)
    g64 = torch.nan_to_num(x64.grad, 0.0).numpy()
    assert_close(gin, g64, TOL, "channelnorm C=%d backward vs fp64" % C)


def test_channelnorm_fp32_misaligned(arena):
    """hw % 4 == 0 but 4-byte aligned buffers: the scalar kernels."""
    x = _rand((2, 3, 6, 10), 7, 2.0, 0.5)
    xn, on, gn, out, gin = _channelnorm_case(arena, x, torch.float32, 4)
    assert_close(out, orc.channelnorm_forward(xn), TOL, "misaligned channelnorm forward")
    assert_close(gin, orc.channelnorm_backward(xn, on, gn), TOL, "misaligned channelnorm backward")


DT16 = {"fp16": (torch.float16, 2e-3), "bf16": (torch.bfloat16, 1.6e-2)}


@pytest.mark.parametrize("dt", list(DT16))
@pytest.mark.parametrize("misalign", [0, 4], ids=["aligned", "misaligned"])
def test_channelnorm_16bit(arena, dt, misalign):
    """hw % 8 == 0: 8-wide kernels when 16-byte aligned, the 1-wide ones 4 bytes off.  The reference is the fp32
    oracle on the same 16-bit inputs; the tolerance is two roundings of the 16-bit type."""
    dtype, tol = DT16[dt]
    x = _rand((2, 3, 8, 10), 8, 2.0, 0.5)
    xn, on, gn, out, gin = _channelnorm_case(arena, x, dtype, misalign)
    assert_close(out, orc.channelnorm_forward(xn), tol, "%s channelnorm forward" % dt)
    assert_close(gin, orc.channelnorm_backward(xn, on, gn), tol, "%s channelnorm backward" % dt)


# ------------------------------------------------------------------------------------------------
# Correlation
# ------------------------------------------------------------------------------------------------
def _corr_call(L, arena, a, b, prm, cat_channels, ch_offset, slope, misalign=0, tc=False):
    """forward_cat, then backward_cat (with LeakyReLU's mask) and the plain backward of the masked gradient, all
    through the C ABI on guarded buffers.  Returns (cat, grad_cat, (g1, g2) of backward_cat, (g1, g2) of the plain
    backward)."""
    B, C, H, W = a.shape
    D, oH, oW = _f2().functional.correlation_out_shape(C, H, W, *prm)
    ad, bd = _dev(a, misalign), _dev(b, misalign)
    st = _stream()
    ws = arena.workspace(int(L.fn2b200_correlation_forward_workspace(B, C, H, W, *prm)))
    nws = ws.numel() if ws is not None else 0
    assert (nws > 0) == tc
    cat = arena.out((B, cat_channels, oH, oW), misalign=misalign, fill=SENTINEL)
    assert L.fn2b200_correlation_forward_cat(_p(ad), _p(bd), _p(cat), cat_channels, ch_offset, slope, B, C, H, W, *prm, 1,
                                             _p(ws), nws, st) == 0, L.fn2b200_last_error()
    gcat = _dev(_randn((B, cat_channels, oH, oW), 11), misalign)
    g1, g2 = arena.out((B, C, H, W), misalign=misalign), arena.out((B, C, H, W), misalign=misalign)
    assert L.fn2b200_correlation_backward_cat(_p(ad), _p(bd), _p(gcat), _p(cat), cat_channels, ch_offset, slope, _p(g1),
                                              _p(g2), B, C, H, W, *prm, 1, _p(ws), nws, int(tc), st) == 0, L.fn2b200_last_error()
    # the plain backward of the masked gradient gives the same bits (fn2b200_correlation_backward_cat's contract)
    c = cat[:, ch_offset:ch_offset + D]
    gm = gcat[:, ch_offset:ch_offset + D]
    gm = _dev(torch.where(c > 0, gm, gm * slope).cpu(), misalign) if slope != 1.0 else _dev(gm.contiguous().cpu(), misalign)
    p1, p2 = arena.out((B, C, H, W), misalign=misalign), arena.out((B, C, H, W), misalign=misalign)
    assert L.fn2b200_correlation_backward_ws(_p(ad), _p(bd), _p(gm), _p(p1), _p(p2), B, C, H, W, *prm, 1, _p(ws), nws,
                                             int(tc), st) == 0, L.fn2b200_last_error()
    arena.check()
    return cat, gcat, gm, (g1, g2), (p1, p2)


def _corr_check(a, b, prm, cat, gm, grads, plain, ch_offset, slope, what):
    D = orc.correlation_out_shape(a.shape[1], a.shape[2], a.shape[3], *prm)[0]
    ref = orc.correlation_forward(a.numpy(), b.numpy(), *prm)
    act = np.where(ref > 0, ref, ref * np.float32(slope))
    c = cat.cpu().numpy()
    assert_close(c[:, ch_offset:ch_offset + D], act, TOL, "%s forward" % what)
    others = np.delete(c, np.s_[ch_offset:ch_offset + D], axis=1)
    assert (others == SENTINEL).all(), "%s: channels outside [ch_offset, ch_offset + D) were written" % what
    r1, r2 = orc.correlation_backward(a.numpy(), b.numpy(), gm.cpu().numpy(), *prm)
    assert_close(grads[0].cpu().numpy(), r1, TOL, "%s grad1" % what)
    assert_close(grads[1].cpu().numpy(), r2, TOL, "%s grad2" % what)
    assert torch.equal(grads[0], plain[0]) and torch.equal(grads[1], plain[1]), "%s: backward_cat != masked plain" % what
    return ref


@pytest.mark.parametrize("slope", [0.1, 0.0])
@pytest.mark.parametrize("C", [64, 128, 192, 256])
def test_corr_tensor_cores(arena, C, slope):
    """FlowNetC's configuration at every tensor-core channel count; H, W not multiples of the 8 x 16 class tile."""
    f = _f2()
    prm = (20, 1, 20, 1, 2)
    a, b = _randn((2, C, 10, 22), C), _randn((2, C, 10, 22), C + 1)
    assert f._lib.LIB.fn2b200_correlation_path(C, 10, 22, *prm) == 2
    cat, gcat, gm, grads, plain = _corr_call(f._lib.LIB, arena, a, b, prm, 441 + 5, 3, slope, tc=True)
    ref = _corr_check(a, b, prm, cat, gm, grads, plain, 3, slope, "tc C=%d" % C)
    if C == 64 and slope:
        # fp64 second opinion of the forward
        r64 = torch_ref.correlation(a.double(), b.double(), *prm).numpy()
        assert_close(ref, r64, TOL, "oracle vs fp64")
        act = np.where(r64 > 0, r64, r64 * slope)
        assert_close(cat[:, 3:444].cpu().numpy(), act, TOL, "tc forward vs fp64")


TILED = [(2, 10), (2, 4), (1, 4), (2, 2)]


@pytest.mark.parametrize("slope", [1.0, 0.1, 0.0])
@pytest.mark.parametrize("s2,dr", TILED, ids=["s2_%d-dr%d" % c for c in TILED])
def test_corr_tiled(arena, s2, dr, slope):
    """Every tiled (stride2, radius); C = 72 spans a full and a partial 64-channel block, W = 136 a full and a partial
    128-pixel tile, H = 13 is odd.  slope 1 is the plain correlation (no activation instantiations)."""
    f = _f2()
    md = s2 * dr
    prm = (md, 1, md, 1, s2)
    shape = (2, 72, 13, 136)
    a, b = _randn(shape, 20 + md), _randn(shape, 21 + md)
    assert f._lib.LIB.fn2b200_correlation_path(*shape[1:], *prm) == 1
    D = (2 * dr + 1) ** 2
    cat, gcat, gm, grads, plain = _corr_call(f._lib.LIB, arena, a, b, prm, D + 4, 1, slope)
    _corr_check(a, b, prm, cat, gm, grads, plain, 1, slope, "tiled s2=%d dr=%d slope %g" % (s2, dr, slope))


def test_corr_generic_misaligned(arena):
    """A tiled-family shape with every buffer 4 bytes past a 16-byte boundary: the generic kernels."""
    f = _f2()
    prm = (8, 1, 8, 1, 2)
    shape = (2, 20, 9, 24)
    a, b = _randn(shape, 30), _randn(shape, 31)
    assert f._lib.LIB.fn2b200_correlation_path(*shape[1:], *prm) == 1
    cat, gcat, gm, grads, plain = _corr_call(f._lib.LIB, arena, a, b, prm, 81 + 2, 2, 0.1, misalign=4)
    _corr_check(a, b, prm, cat, gm, grads, plain, 2, 0.1, "generic")
    # fp64 second opinion, forward and both gradients
    a64, b64 = a.double().requires_grad_(), b.double().requires_grad_()
    r64 = torch_ref.correlation(a64, b64, *prm)
    r64.backward(torch.from_numpy(gm.cpu().numpy()).double())
    act = torch.where(r64 > 0, r64, r64 * 0.1).detach().numpy()
    assert_close(cat[:, 2:83].cpu().numpy(), act, TOL, "generic forward vs fp64")
    assert_close(grads[0].cpu().numpy(), a64.grad.numpy(), TOL, "generic grad1 vs fp64")
    assert_close(grads[1].cpu().numpy(), b64.grad.numpy(), TOL, "generic grad2 vs fp64")


def _assert_close_gpu(a, ref, tol, what):
    """max|a - ref| / max|ref| <= tol for tensors too large to copy to the host comfortably."""
    assert a.shape == ref.shape and bool(torch.isfinite(a).all()), what
    e = float((a.double() - ref.double()).abs().max() / ref.double().abs().max())
    assert e <= tol, "%s: max|d|/max|ref| = %.3e > %.1e" % (what, e, tol)


def _launches(call):
    F2 = _f2().functional
    n0 = F2.launch_count()
    r = call()
    return r, F2.launch_count() - n0


@pytest.mark.parametrize("B", [65535, 2 * 65535 + 3])
def test_corr_tiled_batch_grid_limit(B):
    """gridDim.z carries the sample: more than 65535 samples run as several launches.  Samples on both sides of each
    chunk edge against the oracle, the whole tensor against the generic kernels (inputs 4 bytes off alignment)."""
    f = _f2()
    F2 = f.functional
    prm = (4, 1, 4, 1, 2)
    shape = (B, 4, 4, 8)
    assert f._lib.LIB.fn2b200_correlation_path(*shape[1:], *prm) == 1
    g = torch.Generator(device="cuda").manual_seed(40)
    a, b = torch.randn(*shape, device="cuda", generator=g), torch.randn(*shape, device="cuda", generator=g)
    chunks = (B + 65534) // 65535
    out, n = _launches(lambda: F2.correlation_forward(a, b, *prm))
    assert n == chunks
    go = torch.randn(out.shape, device="cuda", generator=g)
    (g1, g2), n = _launches(lambda: F2.correlation_backward(a, b, go, *prm))
    assert n == 2 * chunks
    cat = torch.full((B, 27, 4, 8), SENTINEL, device="cuda")
    F2.correlation_forward_cat(a, b, cat, 1, 0.1, *prm)
    gcat = torch.randn(cat.shape, device="cuda", generator=g)
    (c1, c2), n = _launches(lambda: F2.correlation_backward_cat(a, b, gcat, cat, 1, 0.1, *prm))
    assert n == 2 * chunks
    gm = gcat[:, 1:26]
    gm = torch.where(cat[:, 1:26] > 0, gm, gm * 0.1)
    for n in sorted({0, 65534, 65535, 65536, B - 1} & set(range(B))):
        s = slice(n, n + 1)
        an, bn = a[s].cpu().numpy(), b[s].cpu().numpy()
        ref = orc.correlation_forward(an, bn, *prm)
        assert_close(out[s].cpu().numpy(), ref, TOL, "sample %d forward" % n)
        assert_close(cat[s, 1:26].cpu().numpy(), np.where(ref > 0, ref, ref * np.float32(0.1)), TOL, "sample %d cat" % n)
        r1, r2 = orc.correlation_backward(an, bn, go[s].cpu().numpy(), *prm)
        assert_close(g1[s].cpu().numpy(), r1, TOL, "sample %d grad1" % n)
        assert_close(g2[s].cpu().numpy(), r2, TOL, "sample %d grad2" % n)
        r1, r2 = orc.correlation_backward(an, bn, gm[s].cpu().numpy(), *prm)
        assert_close(c1[s].cpu().numpy(), r1, TOL, "sample %d cat grad1" % n)
        assert_close(c2[s].cpu().numpy(), r2, TOL, "sample %d cat grad2" % n)
    # the whole batch against the generic kernels
    am, bm = _dev(a.cpu(), 4), _dev(b.cpu(), 4)
    (gen, n) = _launches(lambda: F2.correlation_forward(am, bm, *prm))
    assert n == 1
    _assert_close_gpu(out, gen, 1e-5, "forward vs generic")
    _assert_close_gpu(cat[:, 1:26], torch.where(gen > 0, gen, gen * 0.1), 1e-5, "cat vs generic")
    assert bool((cat[:, 0] == SENTINEL).all() and (cat[:, 26] == SENTINEL).all())
    for gout, (x1, x2) in ((go, (g1, g2)), (gm.contiguous(), (c1, c2))):
        (r1, r2), n = _launches(lambda: F2.correlation_backward(am, bm, _dev(gout.cpu(), 4), *prm))
        assert n == 2
        _assert_close_gpu(x1, r1, 1e-5, "grad1 vs generic")
        _assert_close_gpu(x2, r2, 1e-5, "grad2 vs generic")


@pytest.mark.parametrize("H,path", [(65532, 1), (65540, 0)])
def test_corr_tiled_height_grid_limit(H, path):
    """The tiled backward's gridDim.y is H: taller inputs run on the generic kernels."""
    f = _f2()
    F2 = f.functional
    prm = (4, 1, 4, 1, 2)
    shape = (1, 4, H, 8)
    assert f._lib.LIB.fn2b200_correlation_path(*shape[1:], *prm) == path
    a, b = _randn(shape, 50), _randn(shape, 51)
    out = F2.correlation_forward(a.cuda(), b.cuda(), *prm)
    go = _randn(tuple(out.shape), 52)
    g1, g2 = F2.correlation_backward(a.cuda(), b.cuda(), go.cuda(), *prm)
    assert_close(out.cpu().numpy(), orc.correlation_forward(a.numpy(), b.numpy(), *prm), TOL, "H=%d forward" % H)
    r1, r2 = orc.correlation_backward(a.numpy(), b.numpy(), go.numpy(), *prm)
    assert_close(g1.cpu().numpy(), r1, TOL, "H=%d grad1" % H)
    assert_close(g2.cpu().numpy(), r2, TOL, "H=%d grad2" % H)


def test_corr_tc_backward_more_than_65535_rows(monkeypatch):
    """Tensor-core backward with B * H = 67200 (sample, row) pairs against the FP32-FMA kernels, and the last sample
    against the oracle."""
    f = _f2()
    F2 = f.functional
    prm = (20, 1, 20, 1, 2)
    shape = (2100, 64, 32, 16)
    assert f._lib.LIB.fn2b200_correlation_path(*shape[1:], *prm) == 2
    g = torch.Generator(device="cuda").manual_seed(60)
    a, b = torch.randn(*shape, device="cuda", generator=g), torch.randn(*shape, device="cuda", generator=g)
    go = torch.randn((shape[0], 441, 32, 16), device="cuda", generator=g)
    g1, g2 = F2.correlation_backward(a, b, go, *prm)
    monkeypatch.setenv("FN2B200_CORR_BWD", "fma")
    r1, r2 = F2.correlation_backward(a, b, go, *prm)
    monkeypatch.delenv("FN2B200_CORR_BWD")
    _assert_close_gpu(g1, r1, 5e-5, "tc grad1 vs fma")
    _assert_close_gpu(g2, r2, 5e-5, "tc grad2 vs fma")
    n = shape[0] - 1
    o1, o2 = orc.correlation_backward(a[n:].cpu().numpy(), b[n:].cpu().numpy(), go[n:].cpu().numpy(), *prm)
    assert_close(g1[n:].cpu().numpy(), o1, TOL, "last sample grad1")
    assert_close(g2[n:].cpu().numpy(), o2, TOL, "last sample grad2")


# ------------------------------------------------------------------------------------------------
# Resample2d
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("C", [1, 2, 3, 5])
@pytest.mark.parametrize("scatter", ["vector", "planar"])
def test_resample2d(arena, scatter, C):
    """An image larger than the flow (iH > H, iW > W) with more samples than the flow (3 > 2), sigma = 6 px so that
    many taps clamp: K7 (forward, flow gradient) clamps with the flow's dims, K6 (image-gradient scatter) with the
    image's.  The forward, both gradients and the flow gradient alone, against the oracle.  The C ABI backward runs
    the scatter under test: `vector` hands it the queried workspace (the interleaved scratch when C <= 3), `planar` a
    NULL workspace of 0 bytes (scalar reductions straight into the gradient)."""
    f = _f2()
    F2, L = f.functional, f._lib.LIB
    B, H, W, iH, iW = 2, 21, 37, 26, 45
    img = _rand((3, C, iH, iW), C, 1.0, 0.5)
    flow = _randn((B, 2, H, W), 70 + C, 6.0)
    flow[0, :, 0, :8] = 0.0                              # zero flow: the taps are the pixels themselves
    gout = _randn((B, C, H, W), 71)
    imd, fld, gd = img.cuda(), flow.cuda(), gout.cuda()
    out = F2.resample2d_forward(imd, fld, out=arena.out((B, C, H, W)))
    gi, gf = F2.resample2d_backward(imd, fld, gd, out1=arena.out((3, C, iH, iW)), out2=arena.out((B, 2, H, W)))
    none, gf_only = F2.resample2d_backward(imd, fld, gd, need1=False, out2=arena.out((B, 2, H, W)))
    assert none is None
    # the C ABI with the scatter's workspace: exactly the queried size (0 for C > 3), or none
    st = F2._img_strides(imd)
    nws = int(L.fn2b200_resample2d_backward_workspace(st, B, C, iH, iW, H, W))
    assert (nws > 0) == (C <= 3)
    if scatter == "planar":
        nws = 0
    ws = arena.workspace(nws)
    gi_ws, gf_ws = arena.out((B, C, iH, iW)), arena.out((B, 2, H, W))
    assert L.fn2b200_resample2d_backward_ws(_p(imd), st, _p(fld), _p(gd), _p(gi_ws), _p(gf_ws), B, C, iH, iW, H, W, 1, 1, 1,
                                            _p(ws), nws, _stream()) == 0, L.fn2b200_last_error()
    arena.check()
    ref = orc.resample2d_forward(img.numpy(), flow.numpy())
    rgi, rgf = orc.resample2d_backward(img.numpy(), flow.numpy(), gout.numpy())
    assert_close(out.cpu().numpy(), ref, TOL, "%s C=%d forward" % (scatter, C))
    gi_n = gi.cpu().numpy()
    assert_close(gi_n, rgi, TOL, "%s C=%d image gradient" % (scatter, C))
    assert_close(gf.cpu().numpy(), rgf, TOL, "%s C=%d flow gradient" % (scatter, C))
    gi_ws_n = gi_ws.cpu().numpy()
    assert_close(gi_ws_n, rgi[:B], TOL, "%s C=%d image gradient (C ABI)" % (scatter, C))
    assert (gi_n[B:] == 0).all(), "image-gradient rows beyond the flow batch must be exactly 0"
    for g_n in (gi_n, gi_ws_n):
        beyond = np.concatenate([g_n[:B, :, H:].ravel(), g_n[:B, :, :, W:].ravel()])
        assert (beyond != 0).any(), "no image-gradient tap beyond the flow's (H, W): the case does not test K6's clamp"
    # the flow gradient does not depend on whether the image gradient is computed, nor on the scatter
    assert torch.equal(gf, gf_only) and torch.equal(gf, gf_ws)
    # fp64 second opinion of the forward where the semantics coincide (image and flow of one size: grid_sample)
    sub = torch.from_numpy(img.numpy()[:B, :, :H, :W]).double()
    r64 = torch_ref.resample2d(sub, flow.double()).numpy()
    same = F2.resample2d_forward(sub.float().cuda(), fld).cpu().numpy()
    assert_close(same, r64, TOL, "%s C=%d forward vs fp64" % (scatter, C))


# ------------------------------------------------------------------------------------------------
# Fused warp concat (forward and backward)
# ------------------------------------------------------------------------------------------------
def _layouts(C):
    """The 3C + 3 channel concat of models.py:138 and a fusion-style layout (x[:, :C], flow, norms) of concat3."""
    return {
        "concat": dict(flow_div=20.0),
        "fusion": dict(flow_div=1.0, cat_channels=C + 7, ch_x=0, n_x=C, ch_warped=-1, ch_flow=C + 1, ch_flow_norm=C + 4,
                       ch_diff_norm=C + 6),
    }


def _cat_channels(C, layout):
    return layout.get("cat_channels", 3 * C + 3)


def _bwd_kw(layout):
    return {k: v for k, v in layout.items() if k != "cat_channels"}


def _warp_backward_abi(arena, C, x, flow, gcat, mode, mul, layout, need_x, need_flow):
    """fn2b200_warp_concat_backward_up on guarded outputs and an exactly-sized guarded workspace."""
    L = _f2()._lib.LIB
    kw = dict(dict(ch_x=0, n_x=2 * C, ch_warped=2 * C, ch_flow=3 * C, flow_div=1.0, ch_flow_norm=-1, ch_diff_norm=3 * C + 2),
              **_bwd_kw(layout))
    B, _, fh, fw = flow.shape
    H, W = x.shape[2], x.shape[3]
    gx = arena.out((B, 2 * C, H, W)) if need_x else None
    gf = arena.out(tuple(flow.shape)) if need_flow else None
    nws = int(L.fn2b200_warp_concat_backward_up_workspace(B, C, H, W, mode, int(need_x)))
    ws = arena.workspace(nws)
    rc = L.fn2b200_warp_concat_backward_up(_p(x), (ctypes.c_int64 * 4)(*x.stride()), C, _p(flow), fh, fw, mode, mul,
                                           _p(gcat), gcat.size(1), kw["ch_x"], kw["n_x"], kw["ch_warped"], kw["ch_flow"],
                                           kw["flow_div"], kw["ch_flow_norm"], kw["ch_diff_norm"], _p(gx), _p(gf), _p(ws),
                                           nws, B, H, W, _stream())
    assert rc == 0, L.fn2b200_last_error()
    arena.check()
    return gx, gf


WARP_GRADS = {"both": (True, True), "x_only": (True, False), "flow_only": (False, True)}
# (B, fh, fw): full resolution 20 x 36 -- neither a multiple of the 16 x 32 tile -- and a flow row / column of one cell
WARP_SHAPES = {"ragged": (2, 5, 9), "fh1": (1, 1, 9), "fw1": (2, 5, 1)}


def _warp_case(arena, C, mode, grads, layout_name, shape, seed):
    F2 = _f2().functional
    B, fh, fw = WARP_SHAPES[shape]
    H, W = 4 * fh, 4 * fw
    mul = 20.0 if mode else 1.0
    layout = _layouts(C)[layout_name]
    x = _rand((B, 2 * C, H, W), seed, 1.0, 0.5)
    lr = _randn((B, 2, fh, fw) if mode else (B, 2, H, W), seed + 1, 6.0 / mul)   # sigma = 6 full-resolution pixels
    gcat = _randn((B, _cat_channels(C, layout), H, W), seed + 2)
    xd, ld, gd = x.cuda(), lr.cuda(), gcat.cuda()
    need_x, need_flow = WARP_GRADS[grads]
    gx, gf = _warp_backward_abi(arena, C, xd, ld, gd, mode, mul, layout, need_x, need_flow)
    rx, rf = ur.warp_concat_backward(x.numpy(), lr.numpy(), gcat.numpy(), C=C, upsample_mode=mode, flow_mul=mul,
                                     **_bwd_kw(layout))
    what = "C=%d mode %d %s %s %s" % (C, mode, grads, layout_name, shape)
    if need_x:
        assert_close(gx.cpu().numpy(), rx, TOL, what + " grad_x")
    if need_flow:
        assert_close(gf.cpu().numpy(), rf, TOL, what + " grad_flow")
        # bit-identical with and without the image gradient
        _, gf_both = _warp_backward_abi(Arena(), C, xd, ld, gd, mode, mul, layout, True, True)
        assert torch.equal(gf, gf_both), what + ": flow gradient depends on need_x"
    if mode == 0 and need_x and need_flow:
        # the Python entry point on the same call: the same flow gradient bit for bit
        px, pf = F2.warp_concat_backward(xd, ld, gd, C=C, **_bwd_kw(layout))
        assert torch.equal(pf, gf)
        assert_close(px.cpu().numpy(), gx.cpu().numpy(), 1e-6, what + " functional grad_x")


@pytest.mark.parametrize("layout", ["concat", "fusion"])
@pytest.mark.parametrize("grads", list(WARP_GRADS))
@pytest.mark.parametrize("mode", [0, 1, 2], ids=["full", "bilinear", "nearest"])
@pytest.mark.parametrize("C", [1, 2, 3])
def test_warp_concat_backward(arena, C, mode, grads, layout):
    """warp_concat_backward at C = 1, 2 and 3 (x has 2C channels) for every upsample mode, gradient choice and layout."""
    _warp_case(arena, C, mode, grads, layout, "ragged", 100 * C + 10 * mode)


@pytest.mark.parametrize("shape", ["fh1", "fw1"])
@pytest.mark.parametrize("mode", [1, 2], ids=["bilinear", "nearest"])
@pytest.mark.parametrize("C", [1, 2, 3])
def test_warp_concat_backward_one_cell_flow(arena, C, mode, shape):
    """A quarter-resolution flow one cell high or wide: every bilinear tap of that axis clamps."""
    _warp_case(arena, C, mode, "both", "concat", shape, 300 + 10 * C + mode)


@pytest.mark.parametrize("C", [1, 2, 3, 4, 5])
def test_warp_concat_forward(arena, C):
    """The fused forward for C = 1..5 (C >= 4: the runtime-C kernel), through the bilinear upsample; one output channel
    that no product owns must keep its sentinel."""
    F2 = _f2().functional
    B, fh, fw = 2, 5, 9
    H, W = 4 * fh, 4 * fw
    x = _rand((B, 2 * C, H, W), 400 + C, 1.0, 0.5)
    lr = _randn((B, 2, fh, fw), 401 + C, 0.3)
    layout = dict(ch_x=0, n_x=2 * C, ch_warped=2 * C, ch_flow=3 * C, flow_div=20.0, ch_diff_norm=3 * C + 2,
                  ch_flow_norm=3 * C + 4)
    nch = 3 * C + 5                                     # channel 3C + 3 belongs to no product
    out = F2.warp_concat_forward(x.cuda(), lr.cuda(), C=C, upsample="bilinear", flow_mul=20.0,
                                 out=arena.out((B, nch, H, W), fill=SENTINEL), **layout)
    arena.check()
    ref = orc.warp_concat_forward(x.numpy(), lr.numpy(), C=C, upsample_mode=1, flow_mul=20.0, cat_channels=nch, **layout)
    got = out.cpu().numpy()
    assert (got[:, 3 * C + 3] == SENTINEL).all(), "the unowned channel was written"
    ref[:, 3 * C + 3] = SENTINEL
    assert_close(got, ref, TOL, "fused forward C=%d" % C)
    if C > 3:
        with pytest.raises(RuntimeError, match="C=%d > 3" % C):
            F2.warp_concat_backward(x.cuda(), lr.cuda(), torch.zeros(B, nch, H, W, device="cuda"), C=C, upsample="bilinear",
                                    flow_mul=20.0, **layout)
