"""The ChannelNorm kernels, element by element: fp32 against fp64 within derived bounds and bit for bit against the fp32
restatement on the edges, fp16 and bf16 bit for bit against the fp32-arithmetic restatement (tests/torch_ref.py,
pinned on the CPU against the reference's own half kernels).

Every output is a view in a NaN-poisoned, guarded allocation (tests/guarded.py); each case checks through the
torch.profiler kernel names that the instantiation it targets ran (once more if the record lacks it: the profiler can drop
the records of kernels that ran).  Inputs are random with a catalogue of edge pixels
written over the first ones (EDGES32 / EDGES16): a zero pixel; squares that underflow to 0 or round to a subnormal in
the storage type; squares that overflow it (fp16 |x| >= 256); x != 0 with norm 0, where the backward divides by 1e-9f
(fp16: +-inf for large enough |g x|); and squares far apart in size.

fp32.  The forward is acc = fma(x_c, x_c, acc) in channel order (nvcc contracts `acc += v * v`; the first fma is exact)
then sqrtf: C - 1 roundings of a sum of positive terms, so the sum errs by at most gamma_{C-1} of itself, the square root
halves that and rounds once: |o - ref64| <= ((C - 1)/2 + 2) u ref64, u = 2^-24.  The backward g x / (o + 1e-9f), taking
the kernel's own o, rounds the product, the constant 1e-9, the sum and the quotient: |gi - ref64| <= 5 u |ref64|, against
fp64 g x / (o + 1e-9).  Zero pixels give exact zeros, and on the edge pixels both directions equal torch_ref's fp32
restatement bit for bit.  The backward equals it bit for bit everywhere.

16-bit.  Forward and backward equal torch_ref.channelnorm16 / channelnorm_backward32 bit for bit at every element.
"""
import ctypes

import pytest
import torch

import torch_ref
from guarded import Arena
from util import cuda_profile

pytestmark = pytest.mark.gpu
P = ctypes.c_void_p
U = 2.0 ** -24

# per-pixel channel patterns; a pattern shorter than C is padded with zeros, a longer one cut
EDGES32 = [
    [0.0], [2.0 ** -80] * 5, [1.5 * 2.0 ** -75], [1.0, 2.0 ** -80, 2.0 ** -80], [1e20], [1.5e19, 1.5e19],
    [1e19, 1.0], [2.0 ** -70, 2.0 ** -63], [3.0, -4.0],
]
EDGES16 = {
    torch.float16: [[0.0], [2.0 ** -13] * 4, [2.0 ** -10, 2.0 ** -12], [256.0], [-300.0, 1.0], [2.0 ** -13, -2.0 ** -13],
                    [180.0, 180.0], [3.0, -4.0], [2.0 ** -7, 2.0 ** -14]],
    torch.bfloat16: [[0.0], [2.0 ** -80] * 4, [2.0 ** -64, 2.0 ** -66], [2.0 ** 64], [-2.0 ** 70, 1.0],
                     [2.0 ** -70, -2.0 ** -75], [1e19, 1e19], [3.0, -4.0]],
}


def _f2():
    import flownet2_b200
    return flownet2_b200


def _p(t):
    return P(t.data_ptr())


def _st():
    return P(torch.cuda.current_stream().cuda_stream)


def _dev(t, misalign):
    es = t.element_size()
    v = torch.empty(t.numel() + 16 // es, dtype=t.dtype, device="cuda")[misalign // es:misalign // es + t.numel()]
    v = v.view(t.shape)
    v.copy_(t)
    assert v.data_ptr() % 16 == misalign
    return v


def _inputs(shape, dtype, edges, seed):
    """Random x and gradOutput with the edge patterns on the first pixels of every sample (and, for the norm-0 pixels,
    gradOutput values large enough that g x / 1e-9 overflows fp16)."""
    B, C, H, W = shape
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, C, H * W, generator=g, dtype=torch.float64)
    go = torch.randn(B, 1, H * W, generator=g, dtype=torch.float64)
    for i, pat in enumerate(edges[:H * W]):
        col = (pat + [0.0] * C)[:C]
        x[:, :, i] = torch.tensor(col, dtype=torch.float64)
        go[:, :, i] = 4.0 if i % 2 else -4.0
    return x.view(shape).to(dtype), go.view(B, 1, H, W).to(dtype), min(len(edges), H * W)


def _kernels(prof):
    return {e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and "channelnorm" in e.name}


def _run(x, go, misalign, want):
    """Forward and backward through the C ABI on guarded outputs; returns (o, gi) and checks the kernels that ran."""
    L = _f2()._lib.LIB
    arena = Arena()
    B, C, H, W = x.shape
    xd, gd = _dev(x, misalign), _dev(go, misalign)
    o = arena.out((B, 1, H, W), dtype=x.dtype, misalign=misalign)
    gi = arena.out((B, C, H, W), dtype=x.dtype, misalign=misalign)

    def launch():
        if x.dtype == torch.float32:
            assert L.fn2b200_channelnorm_forward(_p(xd), _p(o), B, C, H, W, 2, _st()) == 0, L.fn2b200_last_error()
            assert L.fn2b200_channelnorm_backward(_p(xd), _p(o), _p(gd), _p(gi), B, C, H, W, 2, _st()) == 0, \
                L.fn2b200_last_error()
        else:
            dt = 1 if x.dtype == torch.float16 else 2
            assert L.fn2b200_channelnorm_forward_16(_p(xd), _p(o), B, C, H, W, 2, dt, _st()) == 0, L.fn2b200_last_error()
            assert L.fn2b200_channelnorm_backward_16(_p(xd), _p(o), _p(gd), _p(gi), B, C, H, W, 2, dt, _st()) == 0, \
                L.fn2b200_last_error()
    # the profiler can drop the record of a kernel that ran: a missing name runs the (deterministic) calls once more
    ran = set()
    for _ in range(2):
        with cuda_profile() as prof:
            launch()
            torch.cuda.synchronize()
        ran |= _kernels(prof)
        if all(any(w in n for n in ran) for w in want):
            break
    for w in want:
        assert any(w in n for n in ran), "%s did not run: %s" % (w, sorted(ran))
    # the edge values make some outputs infinite; the guards must hold and no element may keep the NaN poison
    for raw, orig, start, nbytes, view, what in arena.items:
        b, ob = raw.view(torch.uint8), orig.view(torch.uint8)
        assert torch.equal(b[:start], ob[:start]) and torch.equal(b[start + nbytes:], ob[start + nbytes:]), what
        assert not bool(torch.isnan(view).any()), "%s: NaN (never written?)" % what
    return o.cpu(), gi.cpu()


def _bits_equal(x, ref, what, n_edge=None):
    x, ref = x.reshape(x.shape[0], x.shape[1], -1), ref.reshape(ref.shape[0], ref.shape[1], -1)
    if n_edge is not None:
        x, ref = x[..., :n_edge], ref[..., :n_edge]
    same = (x == ref) | (torch.isnan(x) & torch.isnan(ref))
    if not bool(same.all()):
        i = tuple(int(v) for v in (~same).nonzero()[0])
        pytest.fail("%s: %d elements differ from the restatement; the first at %s: got %r, want %r" % (
            what, int((~same).sum()), i, float(x[i]), float(ref[i])))


# (C, H, W, misalign, the kernels that must run)
FP32_CASES = [
    (1, 8, 12, 0, ("channelnorm_fwd_v4<1>", "channelnorm_bwd_v4<1>")),
    (2, 8, 12, 0, ("channelnorm_fwd_v4<2>", "channelnorm_bwd_v4<2>")),
    (3, 8, 12, 0, ("channelnorm_fwd_v4<3>", "channelnorm_bwd_v4<3>")),
    (4, 8, 12, 0, ("channelnorm_fwd_v4<4>", "channelnorm_bwd_v4<4>")),
    (5, 8, 12, 0, ("channelnorm_fwd_v4<0>", "channelnorm_bwd_v4<0>")),
    (64, 8, 12, 0, ("channelnorm_fwd_v4<0>", "channelnorm_bwd_v4<0>")),
    (3, 7, 9, 0, ("channelnorm_fwd_scalar", "channelnorm_bwd_scalar")),
    (5, 8, 12, 4, ("channelnorm_fwd_scalar", "channelnorm_bwd_scalar")),
]


@pytest.mark.parametrize("C,H,W,misalign,want", FP32_CASES, ids=["C%d-%dx%d-off%d" % c[:4] for c in FP32_CASES])
def test_channelnorm_fp32(C, H, W, misalign, want):
    x, go, ne = _inputs((2, C, H, W), torch.float32, EDGES32, 100 + C + H)
    o, gi = _run(x, go, misalign, want)
    x64 = x.double()
    ref = torch_ref.channelnorm(x64)
    fin = (ref > 2.0 ** -60) & (ref < 1.8e19)            # every square normal in fp32; the rest are edge pixels
    assert bool(((o.double() - ref).abs() <= ((C - 1) / 2 + 2) * U * ref)[fin].all()), "forward beyond its bound"
    assert bool((o[ref == 0] == 0).all()), "zero pixels"
    _bits_equal(o, torch_ref.channelnorm32(x), "forward, edge pixels", ne)
    gref = go.double() * x64 / (o.double() + 1e-9)
    ok = torch.isfinite(gref) & (gref.abs() < 1e38) & (gref.abs() > 2.0 ** -100)
    assert bool(((gi.double() - gref).abs() <= 5 * U * gref.abs())[ok].all()), "backward beyond its bound"
    assert bool((gi[x == 0] == 0).all()), "x = 0 gives an exact 0 gradient"
    _bits_equal(gi, torch_ref.channelnorm_backward32(x, o, go), "backward")


CASES16 = [(dt, C, H, W, mis) for dt in (torch.float16, torch.bfloat16)
           for C, H, W, mis in ((3, 8, 16, 0), (5, 7, 9, 0), (2, 8, 16, 4))]


@pytest.mark.parametrize("dtype,C,H,W,misalign", CASES16,
                         ids=["%s-C%d-%dx%d-off%d" % ((str(c[0])[6:],) + c[1:]) for c in CASES16])
def test_channelnorm_16bit(dtype, C, H, W, misalign):
    h8 = (H * W) % 8 == 0 and not misalign
    want = ("channelnorm_fwd_h8", "channelnorm_bwd_h8") if h8 else ("channelnorm_fwd_h1", "channelnorm_bwd_h1")
    x, go, ne = _inputs((2, C, H, W), dtype, EDGES16[dtype], 200 + C + H)
    o, gi = _run(x, go, misalign, want)
    _bits_equal(o, torch_ref.channelnorm16(x), "forward")
    _bits_equal(gi, torch_ref.channelnorm_backward32(x, o, go), "backward")
    if dtype == torch.float16:
        # the pixel of four 2^-13 channels: norm 0, so g x / 1e-9f = +-4 * 2^-13 / 1e-9 overflows to +-inf
        assert float(o[0, 0].reshape(-1)[1]) == 0.0
        assert bool(torch.isinf(gi[0].reshape(C, -1)[:min(C, 4), 1]).all())
    assert bool((o.reshape(2, -1)[:, 0] == 0).all()) and bool((gi.reshape(2, C, -1)[:, :, 0] == 0).all())
