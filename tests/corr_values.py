"""Value-range catalogue and models for the correlation kernels' accuracy tests (tests/test_corr_values_cpu.py,
tests/test_gpu_corr_values.py).  Test helper only.

- `split_bf16`: the tensor-core path's split x = hi + lo (correlation_tc.cu, tc_split_hi): hi = rn_bf16(x) saturated
  to the largest finite bf16 (cvt.rn.satfinite), so a finite x in the bf16 overflow window (|x| in [0x7F7F8000,
  0x7F7FFFFF]) and +-inf take +-max; lo = rn_bf16(x - hi).  torch's bf16 conversion rounds to nearest-even like __float2bfloat16_rn.
- `bound_tc` / `bound_fma`: per-element error bounds.  With a = ha + la + ea (and b likewise, ea exact in fp64) the
  tensor-core kernels form ha hb + ha lb + la hb, i.e. they drop exactly la lb + ea b + (ha + la) eb.  So

      |x - ref64| <= C64(|la|, |lb|) + C64(|ea|, |b|) + C64(|ha + la|, |eb|) + 2 (3K + 3) u S + eta,

  C64 being the fp64 restatement (tests/torch_ref.py) of the operation, S = C64(|a|, |b|), u = 2^-24.  Where both
  halves are normal bf16 numbers, |ea| <= 2^-16 |a| and the first three terms are the old closed-form 3 2^-16 S; below
  about 2^-118 lo is a bf16 subnormal and ea is an absolute error of up to 2^-134.  eta covers fp32 partial sums
  and products in the subnormal range: each of the 3K + 3 roundings errs by at most 2^-149 there (twice that allowed,
  as for u).  The FP32-FMA kernels: (K + 2) u S + (K + 1) 2^-149.
- Catalogue generators, one per value class (CLASSES), seeded and shape-agnostic.
- Non-finite footprints: which output elements one NaN / inf input element may reach, per family and direction.
"""
import torch

import corr_tc_schedule as sch
import torch_ref

U = 2.0 ** -24
SUB = 2.0 ** -149                     # fp32 subnormal spacing
WINDOW = (0x7F7F8000, 0x7F7FFFFF)     # finite fp32 bit patterns (and their negatives) that rn_bf16 rounds to infinity
MANTISSAS = (0x0000, 0x7FFF, 0x8000, 0x8001, 0xFFFF)   # low 16 bits at the bf16 rounding boundary


# ------------------------------------------------------------------------------------------------
# The split
# ------------------------------------------------------------------------------------------------
def f32_from_bits(bits):
    """fp32 tensor from an int64 tensor (or list) of 32-bit patterns."""
    b = torch.as_tensor(bits, dtype=torch.int64)
    return torch.where(b >= 2 ** 31, b - 2 ** 32, b).to(torch.int32).view(torch.float32)


def bits_of(x):
    return x.contiguous().view(torch.int32).to(torch.int64) & 0xFFFFFFFF


def split_bf16(x, clamp=True):
    """(hi, lo) bf16 tensors of the fp32 tensor x, as the kernels split it; clamp=False is plain rn (the unfixed split,
    a negative control)."""
    x = x.float()
    hi = x.to(torch.bfloat16)
    if clamp:
        h = hi.view(torch.int16)
        hi = torch.where((h & 0x7FFF) == 0x7F80, h - 1, h).view(torch.bfloat16)     # +-inf -> +-max finite
    lo = (x - hi.float()).to(torch.bfloat16)
    return hi, lo


def split_parts(x):
    """(ha, la, ea) in fp64: x = ha + la + ea exactly."""
    hi, lo = split_bf16(x)
    h, l = hi.double(), lo.double()
    return h, l, x.double() - h - l


def tc_emulate(x, y):
    """hh + hl + lh of two fp32 tensors, in fp64 (the tensor core's three products, exactly)."""
    hx, lx = (t.double() for t in split_bf16(x))
    hy, ly = (t.double() for t in split_bf16(y))
    return hx * hy + hx * ly + lx * hy


# ------------------------------------------------------------------------------------------------
# Bounds
# ------------------------------------------------------------------------------------------------
def eta_tc(K):
    return 2 * (3 * K + 3) * SUB


def eta_fma(K):
    return (K + 1) * SUB


def bound_tc_forward(a, b, prm):
    """Per-element bound of the tensor-core forward (K = C) against correlation64(a, b)."""
    C = a.size(1)
    ha, la, ea = split_parts(a)
    hb, lb, eb = split_parts(b)
    c = lambda x, y: torch_ref.correlation64(x.abs(), y.abs(), *prm)      # noqa: E731
    S = c(a.double(), b.double())
    return c(la, lb) + c(ea, b.double()) + c(ha + la, eb) + 2 * (3 * C + 3) * U * S + eta_tc(C)


def bound_tc_backward(a, b, go, prm):
    """(bound of gradInput1, bound of gradInput2) of the tensor-core backward (K = D) against correlation64_backward:
    gradInput1 is go x b with both split, gradInput2 go x a."""
    D = go.size(1)
    h1, l1, e1 = split_parts(a)
    h2, l2, e2 = split_parts(b)
    hg, lg, eg = split_parts(go)
    c = lambda x, y, g: torch_ref.correlation64_backward(x.abs(), y.abs(), g.abs(), *prm)   # noqa: E731
    S = c(a.double(), b.double(), go.double())
    t1 = c(l1, l2, lg)
    t2 = c(a.double(), b.double(), eg)
    t3 = c(e1, e2, hg + lg)
    return tuple(t1[i] + t2[i] + t3[i] + 2 * (3 * D + 3) * U * S[i] + eta_tc(D) for i in range(2))


def bound_fma(S, K):
    return (K + 2) * U * S + eta_fma(K)


# ------------------------------------------------------------------------------------------------
# Catalogue
# ------------------------------------------------------------------------------------------------
def _rand_exp(g, shape, lo, hi):
    return torch.randint(lo, hi + 1, shape, generator=g).double()


def _sign(g, shape):
    return torch.randint(0, 2, shape, generator=g).double() * 2 - 1


def _window(g, shape):
    bits = torch.randint(WINDOW[0], WINDOW[1] + 1, shape, generator=g) | (torch.randint(0, 2, shape, generator=g) << 31)
    return f32_from_bits(bits)


def _subnormal(g, shape):
    bits = torch.randint(1, 0x800000, shape, generator=g) | (torch.randint(0, 2, shape, generator=g) << 31)
    return f32_from_bits(bits)


def make(cls, shape, gshape, seed):
    """(a, b, go) fp32 CPU tensors of value class `cls`: a and b of `shape` (B, C, H, W), go of `gshape`."""
    g = torch.Generator().manual_seed(seed)
    B, C, H, W = shape
    rn = lambda s: torch.randn(s, generator=g, dtype=torch.float64)    # noqa: E731
    if cls == "exact":
        # integers in [-8, 8] times 2^[-2, 2]: bf16-representable (lo = 0), and with K <= 441 terms every partial sum
        # lies on the 2^-4 grid below 2^19, so every sum is exact in fp32
        m = lambda s: torch.randint(-8, 9, s, generator=g).double() * 2.0 ** _rand_exp(g, s, -2, 2)   # noqa: E731
        a, b, go = m(shape), m(shape), m(gshape)
    elif cls == "scale":
        a = rn(shape) * 2.0 ** _rand_exp(g, (1, C, 1, 1), -60, 60)
        b = rn(shape) * 2.0 ** _rand_exp(g, (1, C, 1, 1), -60, 60)
        go = rn(gshape) * 2.0 ** _rand_exp(g, (1, gshape[1], 1, 1), -30, 30)
    elif cls == "cancel":
        # channel pairs (2i, 2i + 1): a equal, b opposite, 2^20 larger than the residual channels (the last quarter),
        # so every product of the pair cancels exactly against its partner
        a, b = rn(shape), rn(shape)
        npair = (3 * C // 4) // 2
        big_a, big_b = rn((B, npair, H, W)) * 2.0 ** 20, rn((B, npair, H, W)) * 2.0 ** 20
        a[:, 0:2 * npair:2], a[:, 1:2 * npair:2] = big_a, big_a
        b[:, 0:2 * npair:2], b[:, 1:2 * npair:2] = big_b, -big_b
        go = rn(gshape)
    elif cls == "tiny":
        a = _sign(g, shape) * (1 + torch.rand(shape, generator=g, dtype=torch.float64)) * 2.0 ** _rand_exp(g, shape, -126, -100)
        b, go = rn(shape), rn(gshape)
    elif cls == "subnormal":
        # a: fp32 subnormals; b: ~1 on even channels, ~2^-20 on odd ones (products that underflow); go ~1
        a = _subnormal(g, shape).double()
        b = rn(shape)
        b[:, 1::2] *= 2.0 ** -20
        go = rn(gshape)
    elif cls == "huge":
        # a: the overflow window on half the elements, 2^100..2^127 on the rest; b and go <= 2^-30
        a = torch.where(torch.rand(shape, generator=g) < 0.5, _window(g, shape).double(),
                        _sign(g, shape) * (1 + torch.rand(shape, generator=g, dtype=torch.float64)) *
                        2.0 ** _rand_exp(g, shape, 100, 126))
        b = (rn(shape) * 2.0 ** -34).clamp(-2.0 ** -30, 2.0 ** -30)
        go = (rn(gshape) * 2.0 ** -34).clamp(-2.0 ** -30, 2.0 ** -30)
    elif cls == "huge_go":
        # go in the window, the inputs <= 2^-30
        a = (rn(shape) * 2.0 ** -34).clamp(-2.0 ** -30, 2.0 ** -30)
        b = (rn(shape) * 2.0 ** -34).clamp(-2.0 ** -30, 2.0 ** -30)
        go = _window(g, gshape).double()
    elif cls == "overflow":
        # every product of every sum overflows with one sign: |x|, |y| in [2^64.5, 2^66), so |xy| in [2^129, 2^132);
        # sample n of a has the sign (-1)^n, b and go are positive
        m = lambda s: 2.0 ** (64.5 + 1.5 * torch.rand(s, generator=g, dtype=torch.float64))   # noqa: E731
        sg = torch.tensor([(-1.0) ** n for n in range(B)], dtype=torch.float64).view(B, 1, 1, 1)
        a, b, go = m(shape) * sg, m(shape), m(gshape)
    else:
        raise ValueError(cls)
    return a.float(), b.float(), go.float()


CLASSES = ("exact", "scale", "cancel", "tiny", "subnormal", "huge", "huge_go", "overflow")
BOUND_CLASSES = ("scale", "cancel", "tiny", "subnormal", "huge", "huge_go")


def catalogue_bits(seed=0):
    """fp32 values of every exponent with boundary and random low-16-bit mantissas, both signs, and the specials."""
    g = torch.Generator().manual_seed(seed)
    bits = []
    for e in range(256):
        for hi7 in (0, 0x7F):
            for lo16 in MANTISSAS + tuple(torch.randint(0, 0x10000, (3,), generator=g).tolist()):
                for s in (0, 1):
                    bits.append((s << 31) | (e << 23) | (hi7 << 16) | lo16)
    bits += [WINDOW[0], WINDOW[1], 0x7F7F7FFF, 0x7F800000, 0xFF800000, 0x7FC00000, 0x7F800001, 0, 1 << 31]
    return torch.tensor(sorted(set(bits)), dtype=torch.int64)


# ------------------------------------------------------------------------------------------------
# Non-finite footprints
# ------------------------------------------------------------------------------------------------
def indicator(shape, pos, device="cpu"):
    t = torch.zeros(shape, dtype=torch.float64, device=device)
    t[pos] = 1.0
    return t


def ref_mask_forward(a, b, prm):
    """Non-finite mask of the fp64 forward (the reference footprint: zero padding is multiplied, inf * 0 = NaN)."""
    return ~torch.isfinite(torch_ref.correlation64(a.double(), b.double(), *prm))


def ref_mask_backward(a, b, go, prm):
    return tuple(~torch.isfinite(t) for t in torch_ref.correlation64_backward(a.double(), b.double(), go.double(), *prm))


def inimage_reach(which, shape, gshape, pos, prm, device="cpu"):
    """Outputs reached by the element `pos` of input `which` ('a', 'b' or 'go') through products whose partner lies in
    the image (padding taps not multiplied): (forward mask, gradInput1 mask, gradInput2 mask).  A dependency scan:
    the restatement on the element's indicator and all-ones partners."""
    one = torch.ones(shape, dtype=torch.float64, device=device)
    gone = torch.ones(gshape, dtype=torch.float64, device=device)
    ind = indicator(shape if which != "go" else gshape, pos, device)
    a, b, go = (ind if which == "a" else one), (ind if which == "b" else one), (ind if which == "go" else gone)
    fwd = torch_ref.correlation64(a, b, *prm) != 0 if which != "go" else None
    g1, g2 = torch_ref.correlation64_backward(a, b, go, *prm)
    # gradInput1 depends on (go, input2) only, gradInput2 on (go, input1)
    return fwd, (g1 != 0) & (which != "a"), (g2 != 0) & (which != "b")


def tiled_backward_mask(a, b, go, prm):
    """Non-finite masks of the TMA-tiled backward: gradOutput is read through a box whose rows and columns outside the
    output are zero-filled, and those zeros are multiplied by the other input, so every input pixel is reached as if
    it had an output.  Restated as the backward at pad = md of gradOutput embedded at offset md - pad (>= 0)."""
    pad, k, md, s1, s2 = prm
    off = md - pad
    assert off >= 0
    B, D, oH, oW = go.shape
    H, W = a.shape[2:]
    ge = go.new_zeros((B, D, H, W)).double()
    ge[:, :, off:off + oH, off:off + oW] = go.double()
    return ref_mask_backward(a, b, ge, (md, k, md, s1, s2))


def tc_backward_superset(which, shape, pos, device="cpu"):
    """The tensor-core backward's extra reach for one non-finite element of input1 (which = 'a', reaching gradInput2)
    or input2 ('b', reaching gradInput1): each gradient tile's warpgroup wg multiplies all 144 halo columns of its live
    units wg .. wg + 5 (4 halo rows each) against the banded gradOutput, so the element reaches, in its own channel,
    every in-image pixel of each warpgroup (4 tile rows x 16 class pixels) whose live units hold its halo row.  Returns
    the mask of the gradient it reaches (gradInput1 for 'b', gradInput2 for 'a')."""
    B, C, H, W = shape
    n, c, y, x = pos
    m = torch.zeros(shape, dtype=torch.bool, device=device)
    py, px, yc, xc = y & 1, x & 1, y >> 1, x >> 1
    Hc, Wc = H // 2, W // 2
    nxt, nyt = sch.tile_grid(H, W)
    for ty in range(nyt):
        yc0 = ty * sch.TH
        r = yc - yc0 + sch.DR                          # halo row
        if not 0 <= r < sch.TH + 2 * sch.DR:
            continue
        u = r // sch.UR
        for tx in range(nxt):
            xc0 = tx * sch.TW
            if not 0 <= xc - xc0 + sch.DR < sch.TW + 2 * sch.DR:
                continue
            for wg in (0, 1):
                if not wg <= u <= wg + sch.NU - 2:
                    continue
                ys = [2 * v + py for v in range(yc0 + 4 * wg, min(yc0 + 4 * wg + 4, Hc))]
                xs = [2 * v + px for v in range(xc0, min(xc0 + sch.TW, Wc))]
                for yy in ys:
                    m[n, c, yy, xs] = True
    return m


def probe_positions(shape):
    """name -> (n, c, y, x) of the probe placements for a tensor of `shape` (H >= 30, W >= 52): the interior; a border
    row and column; the last channel; class row 14, halo row 24 of the first tile row, in its unit 6, which is dead for
    warpgroup 0 (whose pixels, class rows 0-3, the reference does not reach from there); class column 25, halo column
    35 of the first tile column, outside the band of that tile's pixels in class columns 0-4."""
    B, C, H, W = shape
    return {"interior": (B - 1, C // 2, H // 2 + 1, W // 2 - 1), "border": (0, 1, 0, W - 1),
            "last_channel": (0, C - 1, H - 2, 3), "dead_halo": (0, 2, 2 * (sch.TH + 6), 6),
            "out_of_band": (0, 3, 4, 2 * 25)}
