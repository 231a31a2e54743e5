"""fp64 restatement of the reference Resample2d kernels (resample2d_kernel.cu:15-198) and of the fused upsample -> warp
-> diff -> channel-norm -> concat chain, with error scales (test helper; torch, CPU or CUDA, no autograd graph).

Semantics restated exactly, quirks included (the kernels reproduce all of them):
- coordinates: xf = fp32(x + dx), yf = fp32(y + dy), rounded in fp32 as the reference computes them; everything after
  that is fp64.  alpha = xf - floor(xf) is exact in fp32.
- forward, bilinear: floor-based taps clamped with the FLOW (output) dims H, W, not the image's; value
  sum_k w_k I_k with w = (1-a)(1-b), a(1-b), (1-a)b, ab in fp64.
- forward, nearest: floor(double(xf) + 0.5), clamped with the output dims.
- K6 (image gradient): floor-based taps clamped with the IMAGE dims iH, iW; fractions from int() truncation,
  xf - trunc(xf); a scatter.
- K7 (flow gradient): taps clamped with the flow dims;
      gx = sum_c g_c [(1-b)(I_TR - I_TL) + b(I_BR - I_BL)],   gy = sum_c g_c [(1-a)(I_BL - I_TL) + a(I_BR - I_TR)].
- the fused chain: d = img0 - warped, n = sqrt(sum d^2), g_d = g_n d / (n + 1e-9), flow / flow_div, |flow|, and the x4
  upsample and its adjoint through upsample_ref.upsample4_matrix in fp64.
- the upsampled flow the kernels warp with is fp32: upsample_flow32 restates load_flow's operation order bit for bit.

Every function also returns error scales: the same expression evaluated on absolute values (S), and for the K6 scatter
the number of contributions to each target (the atomics add them in any order).  For the chain, whose g_d is divided by
n, the helper returns an error bound E built from those scales; tests/test_gpu_resample_fp64.py derives it.
"""
import torch

import upsample_ref

U = 2.0 ** -24
ETA = 2.0 ** -140          # absolute allowance for up to 512 fp32 roundings into the subnormal range (2^-149 each)


def gamma(k):
    """gamma_k = k u / (1 - k u): the relative bound of k fp32 roundings (k may be a tensor)."""
    return k * U / (1 - k * U)


# ----------------------------------------------------------------------------------------------------------------
# coordinates and taps
# ----------------------------------------------------------------------------------------------------------------
def coords(flow):
    """(xf, yf) [B, H, W] fp32: x + dx and y + dy rounded in fp32, as every kernel and the reference compute them."""
    f = flow.float()
    B, _, H, W = f.shape
    xs = torch.arange(W, dtype=torch.float32, device=f.device).view(1, 1, W)
    ys = torch.arange(H, dtype=torch.float32, device=f.device).view(1, H, 1)
    return xs + f[:, 0], ys + f[:, 1]


def _on(variant, axis, ax):
    """The variant for axis `ax` (0: x, 1: y) when it is applied to `axis` (None: both)."""
    return variant if axis is None or axis == ax else None


def _axis_taps(f, n, kind=None):
    """int(floor(f)) and int(floor(f) + 1) (the + 1 in fp32, as the reference) clamped to [0, n-1].  Wrong variants:
    "right_of_clamped" takes the right tap from the clamped left one, "clamp_short" clamps to [0, n-2]."""
    fl = torch.floor(f)
    if kind == "right_of_clamped":
        lo = fl.clamp(0, n - 1).long()
        return lo, (lo + 1).clamp(max=n - 1)
    hi = max(n - 2, 0) if kind == "clamp_short" else n - 1
    return fl.clamp(0, hi).long(), (fl + 1).clamp(0, hi).long()


def floor_taps(xf, yf, W, H, variant=None, axis=None):
    """(xL, xR, yT, yB) int64, clamped to [0, W-1] / [0, H-1]; `variant` (see _axis_taps) on `axis` only."""
    xL, xR = _axis_taps(xf, W, _on(variant, axis, 0))
    yT, yB = _axis_taps(yf, H, _on(variant, axis, 1))
    return xL, xR, yT, yB


def floor_fracs(xf, yf):
    """(alpha, beta) fp64: xf - floor(xf), exact in fp32."""
    return (xf - torch.floor(xf)).double(), (yf - torch.floor(yf)).double()


def trunc_fracs(xf, yf):
    """K6's fractions: xf - int(xf) (truncation toward 0; negative for negative non-integer xf)."""
    return (xf - torch.trunc(xf)).double(), (yf - torch.trunc(yf)).double()


def _next(v, toward):
    return torch.nextafter(torch.tensor(v, dtype=torch.float32), torch.tensor(toward, dtype=torch.float32)).item()


def edge_values(n):
    """Named target coordinates of one axis of n pixels: the clamp edges, ties and fractions where the tap arithmetic
    changes.  Values are fp32 (a target that x + dx cannot reach exactly at a pixel is not placed there)."""
    return {
        "-1-eps": _next(-1.0, -2.0), "-1": -1.0, "-0.5": -0.5, "-eps": -2.0 ** -23, "0": 0.0,
        "n-1-eps": _next(n - 1.0, 0.0), "n-1": n - 1.0, "n-1+eps": _next(n - 1.0, 2.0 * n), "n": float(n),
        "n+0.5": n + 0.5,
        "half": 2.5 if n > 3 else 0.5, "0.49999997": _next(0.5, 0.0), "k+0.5-ulp": _next(min(n - 1, 2) + 0.5, 0.0),
        "alpha_tiny": min(n - 1, 3) + 2.0 ** -20, "alpha_1-2^-24": 1.0 - 2.0 ** -24, "-2^-24": -2.0 ** -24,
        "int": float(min(n - 1, 1)), "big": 1e4, "-big": -1e4, "2^24+2": 2.0 ** 24 + 2, "-(2^24+2)": -(2.0 ** 24 + 2),
    }


EDGE_NAMES = list(edge_values(8))


@torch.no_grad()
def edge_flow(B, H, W, seed, sigma=3.0, frac=0.5):
    """A random flow [B, 2, H, W] (sigma px) with about `frac` of its pixels given a catalogue coordinate on x, on y
    or both.  Returns (flow, where): where[name, axis] = bool mask [B, H, W] of the pixels whose fp32 x + dx (axis 0)
    or y + dy (axis 1) equals edge_values(n)[name] exactly."""
    g = torch.Generator().manual_seed(seed)
    flow = torch.randn(B, 2, H, W, generator=g) * sigma
    where = {}
    for axis, n in ((0, W), (1, H)):
        pos = torch.arange(n, dtype=torch.float32)
        pos = pos.view(1, 1, n) if axis == 0 else pos.view(1, n, 1)
        pos = pos.expand(B, H, W)
        pick = torch.randint(0, 2 * len(EDGE_NAMES), (B, H, W), generator=g)
        pick = torch.where(torch.rand(B, H, W, generator=g) < frac, pick % len(EDGE_NAMES), torch.full_like(pick, -1))
        for k, (name, t) in enumerate(edge_values(n).items()):
            tt = torch.tensor(t, dtype=torch.float32)
            d = tt - pos
            hit = (pick == k) & ((pos + d) == tt)
            flow[:, axis] = torch.where(hit, d, flow[:, axis])
            where[name, axis] = hit
    return flow, where


def edge_hits(flow):
    """where[name, axis]: bool [B, H, W] masks of the pixels whose fp32 coordinate equals edge_values(n)[name]."""
    xf, yf = coords(flow)
    W, H = flow.shape[3], flow.shape[2]
    return {(name, axis): (c == t) for axis, (c, n) in enumerate(((xf, W), (yf, H)))
            for name, t in edge_values(n).items()}


def _gather(img, idx):
    """img [B, C, h, w], idx [B, H, W] flat indices into h * w -> [B, C, H, W]."""
    B, C = img.shape[:2]
    flat = img.reshape(B, C, -1)
    return flat.gather(2, idx.reshape(B, 1, -1).expand(B, C, -1)).view(B, C, *idx.shape[1:])


def _taps4(img, taps, w):
    """(I_TL, I_TR, I_BL, I_BR) of img at taps (xL, xR, yT, yB) of an image of width w."""
    xL, xR, yT, yB = taps
    return [_gather(img, y * w + x) for y, x in ((yT, xL), (yT, xR), (yB, xL), (yB, xR))]


# ----------------------------------------------------------------------------------------------------------------
# Resample2d
# ----------------------------------------------------------------------------------------------------------------
def _fracs(xf, yf, variant=None, axis=None):
    """floor_fracs, or with "frac_fixed8" on `axis` the fraction cut to 8 bits (as a texture unit's filter weights)."""
    a, b = floor_fracs(xf, yf)
    q = lambda t: torch.floor(t * 256) / 256                                              # noqa: E731
    return (q(a) if _on(variant, axis, 0) == "frac_fixed8" else a), (q(b) if _on(variant, axis, 1) == "frac_fixed8" else b)


def _nearest(f, n, kind):
    if kind == "half_even":
        r = torch.round(f.double())
    elif kind == "half_f32":
        r = torch.floor(f + 0.5).double()
    elif kind == "coord_f16":
        r = torch.floor(f.half().double() + 0.5)
    else:
        r = torch.floor(f.double() + 0.5)
    return r.clamp(0, n - 1).long()


@torch.no_grad()
def forward(img, flow, bilinear=True, variant=None, axis=None):
    """(out, S) [B, C, H, W] fp64.  img [Bi >= B, C, iH >= H, iW >= W] (any strides), flow [B, 2, H, W].
    `variant` names a deliberately wrong restatement for the negative controls, applied to `axis` (0: x, 1: y; None:
    both):  "clamp_image" taps clamped with the image dims;  "right_of_clamped", "clamp_short" (see _axis_taps);
    "frac_fixed8" 8-bit fractions;  for nearest, "half_even" rounds half to even, "half_f32" computes
    floor(fp32(xf + 0.5f)), "coord_f16" rounds the coordinate to fp16 first."""
    B, _, H, W = flow.shape
    im = img[:B].double()
    iW = img.shape[3]
    xf, yf = coords(flow)
    cw = iW if _on(variant, axis, 0) == "clamp_image" else W
    ch = img.shape[2] if _on(variant, axis, 1) == "clamp_image" else H
    if not bilinear:
        xN, yN = _nearest(xf, cw, _on(variant, axis, 0)), _nearest(yf, ch, _on(variant, axis, 1))
        out = _gather(im, yN * iW + xN)
        return out, out.abs()
    taps = floor_taps(xf, yf, cw, ch, variant, axis)
    a, b = _fracs(xf, yf, variant, axis)
    a, b = a.unsqueeze(1), b.unsqueeze(1)
    ws = ((1 - a) * (1 - b), a * (1 - b), (1 - a) * b, a * b)
    Is = _taps4(im, taps, iW)
    out = sum(w * i for w, i in zip(ws, Is))
    S = sum(w * i.abs() for w, i in zip(ws, Is))
    return out, S


def _k7(im, taps, a, b, g, iW):
    """(gx, gy, S_x, S_y) [B, H, W]: K7 of gradient g [B, C, H, W] (fp64) on image taps."""
    TL, TR, BL, BR = _taps4(im, taps, iW)
    a, b = a.unsqueeze(1), b.unsqueeze(1)
    dx = (1 - b) * (TR - TL) + b * (BR - BL)
    dy = (1 - a) * (BL - TL) + a * (BR - TR)
    ax = (1 - b) * (TR.abs() + TL.abs()) + b * (BR.abs() + BL.abs())
    ay = (1 - a) * (BL.abs() + TL.abs()) + a * (BR.abs() + TR.abs())
    return (g * dx).sum(1), (g * dy).sum(1), (g.abs() * ax).sum(1), (g.abs() * ay).sum(1), ax, ay


def _k6(g, taps, at, bt, iH, iW):
    """(gimg, S, count) [B, C, iH, iW]: the K6 scatter of g [B, C, H, W] (fp64) with truncation fractions."""
    B, C = g.shape[:2]
    xL, xR, yT, yB = taps
    at, bt = at.unsqueeze(1), bt.unsqueeze(1)
    ss = ((1 - at) * (1 - bt), at * (1 - bt), (1 - at) * bt, at * bt)
    out = g.new_zeros(B, C, iH * iW)
    S = g.new_zeros(B, C, iH * iW)
    cnt = g.new_zeros(B, 1, iH * iW)
    for s, (y, x) in zip(ss, ((yT, xL), (yT, xR), (yB, xL), (yB, xR))):
        idx = (y * iW + x).reshape(B, 1, -1)
        for bb in range(B):
            out[bb].index_add_(1, idx[bb, 0], (s * g)[bb].reshape(C, -1))
            S[bb].index_add_(1, idx[bb, 0], (s.abs() * g.abs())[bb].reshape(C, -1))
            cnt[bb].index_add_(1, idx[bb, 0], torch.ones_like(idx[bb], dtype=g.dtype))
    return out.view(B, C, iH, iW), S.view(B, C, iH, iW), cnt.view(B, 1, iH, iW)


@torch.no_grad()
def backward(img, flow, gout, variant=None, axis=None):
    """The reference's two backward kernels in fp64: dict with
      gimg, S_K6, n_K6 [B, C, iH, iW]   (the image gradient of the first B samples; n_K6 = contributions per target)
      gflow, S_K7 [B, 2, H, W]
    `variant` (on `axis`, as in forward()): "clamp_image" clamps K7's taps with the image dims; "k7_left" takes the
    left / top difference at an integer coordinate (alpha = 0) instead of the right / bottom one; "right_of_clamped",
    "clamp_short" as in forward(); "k6_floor" uses floor-based K6 fractions (the same scatter: see
    tests/test_resample_ref64_cpu.py)."""
    B, C, H, W = gout.shape
    iH, iW = img.shape[2], img.shape[3]
    im = img[:B].double()
    g = gout.double()
    xf, yf = coords(flow)
    a, b = floor_fracs(xf, yf)
    cw = iW if _on(variant, axis, 0) == "clamp_image" else W
    ch = iH if _on(variant, axis, 1) == "clamp_image" else H
    kx, ky = _on(variant, axis, 0) == "k7_left", _on(variant, axis, 1) == "k7_left"
    x7 = torch.where(a == 0, xf - 1, xf) if kx else xf
    y7 = torch.where(b == 0, yf - 1, yf) if ky else yf
    a7 = torch.where(a == 0, torch.ones_like(a), a) if kx else a
    b7 = torch.where(b == 0, torch.ones_like(b), b) if ky else b
    gx, gy, sx, sy, _, _ = _k7(im, floor_taps(x7, y7, cw, ch, variant, axis), a7, b7, g, iW)
    at, bt = (a, b) if variant == "k6_floor" else trunc_fracs(xf, yf)
    gimg, S6, n6 = _k6(g, floor_taps(xf, yf, iW, iH), at, bt, iH, iW)
    return dict(gimg=gimg, S_K6=S6, n_K6=n6, gflow=torch.stack((gx, gy), 1), S_K7=torch.stack((sx, sy), 1))


# ----------------------------------------------------------------------------------------------------------------
# the x4 flow upsample (fp32, load_flow's order) and its adjoint (fp64)
# ----------------------------------------------------------------------------------------------------------------
def _fma32(a, b, c):
    """fp32 fma(a, b, c), correctly rounded: a * b is exact in fp64 here (a has <= 4 significant bits), the fp64 sum is
    rounded to odd (TwoSum residual), and rounding-to-odd at 53 bits then to nearest at 24 bits is a correct rounding."""
    p, c = a.double() * b.double(), c.double()
    s = p + c
    bp = s - c
    e = (p - bp) + (c - (s - bp))
    bits = s.view(torch.int64)
    fix = (e != 0) & ((bits & 1) == 0)
    step = torch.where((e > 0) == (s > 0), 1, -1)
    return torch.where(fix, bits + step, bits).view(torch.float64).float()


def _axis32(n_out, n, device):
    """load_flow's per-axis source index i0, neighbour offset (0 or 1) and lambdas (l0, l1), fp32."""
    p = torch.arange(n_out, dtype=torch.float32, device=device)
    s = torch.clamp(0.25 * (p + 0.5) - 0.5, min=0.0)
    i0 = s.long()
    l1 = s - i0.float()
    step = (i0 < n - 1).long()
    return i0, step, 1.0 - l1, l1


@torch.no_grad()
def upsample_flow32(flow_lr, mode, mul):
    """[B, 2, 4h, 4w] fp32: the full-resolution flow exactly as load_flow computes it.
    nearest: fp32(v * mul) of cell (y >> 2, x >> 2);  bilinear:
        fma(l0h, fma(l0w, A00, l1w * A01), l1h * fma(l0w, A10, l1w * A11)),  A = fp32(v * mul)."""
    f = flow_lr.float() * torch.tensor(mul, dtype=torch.float32)
    B, _, h, w = f.shape
    dev = f.device
    if mode == 2:
        iy = torch.arange(4 * h, device=dev) // 4
        ix = torch.arange(4 * w, device=dev) // 4
        return f[:, :, iy][:, :, :, ix].contiguous()
    if mode != 1:
        raise ValueError("upsample_flow32: mode 1 (bilinear) or 2 (nearest)")
    h0, hs, l0h, l1h = _axis32(4 * h, h, dev)
    w0, ws, l0w, l1w = _axis32(4 * w, w, dev)
    r0, r1 = f[:, :, h0], f[:, :, h0 + hs]

    def row(r):
        a, b = r[:, :, :, w0], r[:, :, :, w0 + ws]
        return _fma32(l0w.expand_as(a), a, l1w * b)

    top, bot = row(r0), row(r1)
    return _fma32(l0h.view(-1, 1).expand_as(top), top, l1h.view(-1, 1) * bot)


def upsample_adjoint(g_up, mode, mul, drop=None):
    """mul * A_h^T g_up A_w in fp64: [B, 2, 4h, 4w] -> [B, 2, h, w].  `drop` = (ty, tx) removes the partial that tile
    (ty, tx) of the 16 x 32 pixel tile grid gives the cells outside its own 4 x 8 (the cells it shares with its
    neighbours): a negative control of the per-tile partial sums."""
    h, w = g_up.shape[-2] // 4, g_up.shape[-1] // 4
    Ah = torch.from_numpy(upsample_ref.upsample4_matrix(h, mode)).to(g_up.device)
    Aw = torch.from_numpy(upsample_ref.upsample4_matrix(w, mode)).to(g_up.device)
    out = float(mul) * torch.einsum("yi,bcyx,xj->bcij", Ah, g_up.double(), Aw)
    if drop is not None:
        ty, tx = drop
        gt = torch.zeros_like(g_up, dtype=torch.float64)
        sl = (Ellipsis, slice(16 * ty, 16 * ty + 16), slice(32 * tx, 32 * tx + 32))
        gt[sl] = g_up[sl].double()
        part = float(mul) * torch.einsum("yi,bcyx,xj->bcij", Ah, gt, Aw)
        part[..., 4 * ty:4 * ty + 4, 8 * tx:8 * tx + 8] = 0
        out = out - part
    return out


# ----------------------------------------------------------------------------------------------------------------
# the fused warp-concat chain
# ----------------------------------------------------------------------------------------------------------------
def layout(C, cat_channels=None, ch_x=0, n_x=None, ch_warped=None, ch_flow=None, flow_div=1.0, ch_flow_norm=-1,
           ch_diff_norm=None):
    """The warp-concat layout with the library's defaults filled in (models.py:138's 3C + 3 channels)."""
    return dict(cat_channels=3 * C + 3 if cat_channels is None else cat_channels, ch_x=ch_x,
                n_x=2 * C if n_x is None else n_x, ch_warped=2 * C if ch_warped is None else ch_warped,
                ch_flow=3 * C if ch_flow is None else ch_flow, flow_div=flow_div, ch_flow_norm=ch_flow_norm,
                ch_diff_norm=3 * C + 2 if ch_diff_norm is None else ch_diff_norm)


@torch.no_grad()
def warp_concat_forward(x, flow32, C, lay):
    """(cat, E) [B, cat_channels, H, W] fp64: the fused forward on the full-resolution fp32 flow and its per-element
    error bound (0 where the kernel must be exact: the copied x channels; unowned channels are NaN in both)."""
    B, _, H, W = flow32.shape
    img0, img1 = x[:, :C].double(), x[:, C:2 * C]
    v, Sv = forward(img1, flow32)
    Ev = gamma(7) * Sv
    d = img0 - v
    Ed = Ev + U * (img0.abs() + v.abs())
    n = d.pow(2).sum(1, keepdim=True).sqrt()
    En = Ed.pow(2).sum(1, keepdim=True).sqrt() + gamma(C + 2) * n
    fl = flow32.double()
    cat = torch.full((B, lay["cat_channels"], H, W), float("nan"), dtype=torch.float64, device=x.device)
    E = torch.zeros_like(cat)
    if lay["ch_x"] >= 0:
        cat[:, lay["ch_x"]:lay["ch_x"] + lay["n_x"]] = x[:, :lay["n_x"]].double()
    if lay["ch_warped"] >= 0:
        cat[:, lay["ch_warped"]:lay["ch_warped"] + C] = v
        E[:, lay["ch_warped"]:lay["ch_warped"] + C] = Ev
    if lay["ch_flow"] >= 0:
        cat[:, lay["ch_flow"]:lay["ch_flow"] + 2] = fl / float(torch.tensor(lay["flow_div"], dtype=torch.float32))
        E[:, lay["ch_flow"]:lay["ch_flow"] + 2] = U * fl.abs() / abs(lay["flow_div"])
    if lay["ch_flow_norm"] >= 0:
        f = fl.pow(2).sum(1, keepdim=True).sqrt()
        cat[:, lay["ch_flow_norm"]:lay["ch_flow_norm"] + 1] = f
        E[:, lay["ch_flow_norm"]:lay["ch_flow_norm"] + 1] = gamma(3) * f
    if lay["ch_diff_norm"] >= 0:
        cat[:, lay["ch_diff_norm"]:lay["ch_diff_norm"] + 1] = n
        E[:, lay["ch_diff_norm"]:lay["ch_diff_norm"] + 1] = En
    return cat, E


@torch.no_grad()
def warp_concat_backward(x, flow32, gcat, C, lay, mode=0, mul=1.0, drop=None):
    """The fused backward in fp64 on the full-resolution fp32 flow: dict with
      gx, E_gx [B, 2C, H, W];  gflow, E_gflow (quarter resolution for mode 1 / 2, else [B, 2, H, W]);
      n [B, 1, H, W] (the diff norm; g_d is exactly 0 where it is 0);  g_up (the full-resolution flow gradient)."""
    B, _, H, W = flow32.shape
    g = gcat.double()
    img0, img1 = x[:, :C].double(), x[:, C:2 * C]
    im1 = img1.double()
    xf, yf = coords(flow32)
    taps = floor_taps(xf, yf, W, H)
    a, b = floor_fracs(xf, yf)
    v, Sv = forward(img1, flow32)
    d = img0 - v
    Ed = gamma(7) * Sv + U * (img0.abs() + v.abs())
    n = d.pow(2).sum(1, keepdim=True).sqrt()
    En = Ed.pow(2).sum(1, keepdim=True).sqrt() + gamma(C + 2) * n
    zero = torch.zeros_like(d)

    def ch(k, m=1):
        return g[:, lay[k]:lay[k] + m] if lay[k] >= 0 else None

    gn = ch("ch_diff_norm")
    if gn is not None:
        den = n + 1e-9
        gd = gn * d / den
        safe = torch.where(n > 0, n, torch.ones_like(n))
        Egd = torch.where(n > 0, gn.abs() * (Ed + d.abs() * En / safe) / safe + gamma(4) * gd.abs(), zero)
    else:
        gd, Egd = zero, zero
    gw = ch("ch_warped", C)
    gv = (gw if gw is not None else zero) - gd
    Egv = Egd + U * ((gw.abs() if gw is not None else zero) + gd.abs())
    # image gradient: [gcat_x0 + g_d | gcat_x1 + K6(g_v)], the second half summed by the atomics then added
    nx = lay["n_x"] if lay["ch_x"] >= 0 else 0
    gxc = torch.zeros(B, 2 * C, H, W, dtype=torch.float64, device=x.device)
    if nx:
        gxc[:, :nx] = g[:, lay["ch_x"]:lay["ch_x"] + nx]
    at, bt = trunc_fracs(xf, yf)
    sc, Ssc, cnt = _k6(gv, taps, at, bt, H, W)
    Esc = _k6(Egv, taps, at, bt, H, W)[1]                             # sum |s| E_gv
    gx = torch.cat((gxc[:, :C] + gd, gxc[:, C:] + sc), 1)
    E_gx = torch.cat((Egd + U * (gxc[:, :C].abs() + gd.abs()),
                      Esc + gamma(cnt + 6) * (Ssc + gxc[:, C:].abs())), 1)
    # flow gradient at full resolution
    gfx, gfy, sx, sy, ax, ay = _k7(im1[:B], taps, a, b, gv, im1.shape[3])
    gup = torch.stack((gfx, gfy), 1)
    Eup = torch.stack(((Egv * ax).sum(1) + gamma(C + 5) * sx, (Egv * ay).sum(1) + gamma(C + 5) * sy), 1)
    Sup = torch.stack((sx, sy), 1)
    fl = flow32.double()
    gf = ch("ch_flow", 2)
    if gf is not None:
        t = gf / float(torch.tensor(lay["flow_div"], dtype=torch.float32))
        gup, Eup, Sup = gup + t, Eup + gamma(1) * t.abs(), Sup + t.abs()
    gfn = ch("ch_flow_norm")
    if gfn is not None:
        f = fl.pow(2).sum(1, keepdim=True).sqrt()
        t = gfn * fl / (f + 1e-9)
        gup, Eup, Sup = gup + t, Eup + gamma(6) * t.abs(), Sup + t.abs()
    Eup = Eup + gamma(3) * Sup                                         # the two or three partial sums added
    out = dict(gx=gx, E_gx=E_gx, n=n, g_up=gup)
    if mode == 0:
        out.update(gflow=gup, E_gflow=Eup)
        return out
    out["gflow"] = upsample_adjoint(gup, mode, mul, drop)
    # per cell: <= 8 + 8 (bilinear rows, then columns) or 16 (nearest) sums, <= 4 tile partials, x mul
    out["E_gflow"] = upsample_adjoint(Eup + gamma(21 if mode == 1 else 17) * Sup, mode, abs(mul))
    return out
