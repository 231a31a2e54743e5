"""Stock-PyTorch formulations of the three layers ("oracle C" in SURVEY.md section 4).

Independent third opinion used to pin the CPU restatement: autograd through these gives the
gradients.  fp64-capable, CPU or CUDA.  Test helper only.
"""
import math

import numpy as np
import torch
import torch.nn.functional as F


def correlation(f1, f2, pad_size, kernel_size, max_displacement, stride1, stride2):
    """out[n,tc,oy,ox] = 1/(k*k*C) * sum_{j,i,c} P1[oy*s1+md+j, ox*s1+md+i] * P2[.. + tj*s2, .. + ti*s2]
    (correlation_cuda_kernel.cu:73-147)."""
    B, C, H, W = f1.shape
    kr = (kernel_size - 1) // 2
    br = kr + max_displacement
    pH, pW = H + 2 * pad_size, W + 2 * pad_size
    dr = max_displacement // stride2
    oH = int(math.ceil((pH - 2 * br) / stride1))
    oW = int(math.ceil((pW - 2 * br) / stride1))
    # extra zero margin so the kernel_size > 1 border taps (row/col -1 and pH/pW of the padded buffer,
    # which the reference reads out of bounds) are explicit zeros instead of wrapped indices
    ex = kr + 1
    p1 = F.pad(f1, (pad_size + ex,) * 4)
    p2 = F.pad(f2, (pad_size + ex,) * 4)
    outs = []
    ys = torch.arange(oH, device=f1.device) * stride1 + max_displacement + ex
    xs = torch.arange(oW, device=f1.device) * stride1 + max_displacement + ex
    for tj in range(-dr, dr + 1):
        for ti in range(-dr, dr + 1):
            acc = 0
            for j in range(-kr, kr + 1):
                for i in range(-kr, kr + 1):
                    a = p1[:, :, (ys + j)][:, :, :, (xs + i)]
                    b = p2[:, :, (ys + j + tj * stride2)][:, :, :, (xs + i + ti * stride2)]
                    acc = acc + (a * b).sum(1)
            outs.append(acc / (kernel_size * kernel_size * C))
    return torch.stack(outs, 1)


def corr_geometry(H, W, pad_size, kernel_size, max_displacement, stride1, stride2):
    """(kr, dr, oH, oW) as the reference computes them: dr = md // s2, and each output dim the float ceil of a float
    division (correlation_cuda.cc:33-34), of the padded extent less the border md + kr on each side."""
    kr, dr = (kernel_size - 1) // 2, max_displacement // stride2
    br = kr + max_displacement
    oH = int(math.ceil(np.float32(H + 2 * pad_size - 2 * br) / np.float32(stride1)))
    oW = int(math.ceil(np.float32(W + 2 * pad_size - 2 * br) / np.float32(stride1)))
    return kr, dr, oH, oW


# Deliberately wrong restatements, each of which flips exactly one thing; the GPU tests show that the kernels are told
# apart from each of them on the elements where it differs.
VARIANTS = {
    "replicate": "replicate padding instead of zero padding",
    "centre_br": "the patch centre at oy*s1 + md + kr instead of oy*s1 + md",
    "norm_odd": "the sum divided by (2kr+1)^2 C instead of k^2 C (differs for even k)",
    "drop_tail8": "the forward sums only the first 8 floor(C/8) channels (the tiled forward's channel chunk)",
    "drop_tail64": "gradients of channels >= 64 floor(C/64) are 0 (the tiled backward's channel block)",
    "swap_planes": "displacement (tj, ti) in plane ti*ds + tj instead of tj*ds + ti",
    "mirror2": "gradInput2 shifted by +(tj, ti) s2 instead of -(tj, ti) s2 (gradInput1's displacement sign)",
}


def _corr_setup(a, pad_size, kernel_size, max_displacement, stride1, stride2, variant):
    assert variant is None or variant in VARIANTS, variant
    B, C, H, W = a.shape
    kr, dr, oH, oW = corr_geometry(H, W, pad_size, kernel_size, max_displacement, stride1, stride2)
    # margin around the input large enough that every tap of every variant is an index inside the buffer: taps
    # outside the reference's padded extent (the kernel_size > 1 border taps, which the reference reads out of bounds)
    # then read explicit zeros (SURVEY C-3) rather than wrapped indices
    e = pad_size + 2 * kr + max_displacement + dr * stride2 + 1
    # buffer index of output (0, 0)'s patch centre: padded coordinate md (not md + kr)
    c0 = e - pad_size + max_displacement + (kr if variant == "centre_br" else 0)
    ds = 2 * dr + 1
    disp = [(d, tj, ti) for d, (tj, ti) in enumerate((tj, ti) for tj in range(-dr, dr + 1) for ti in range(-dr, dr + 1))]
    if variant == "swap_planes":
        disp = [((ti + dr) * ds + tj + dr, tj, ti) for _, tj, ti in disp]
    norm = ((2 * kr + 1) if variant == "norm_odd" else kernel_size) ** 2 * C
    return e, c0, kr, oH, oW, disp, norm


def _corr_pad(t, e, variant):
    return F.pad(t, (e,) * 4, mode="replicate" if variant == "replicate" else "constant")


def correlation64(f1, f2, pad_size, kernel_size, max_displacement, stride1, stride2, variant=None):
    """The forward as an explicit sum of shifted products of the zero-padded inputs, batched, in the inputs' dtype
    (fp64 for a reference) on their device, without an autograd graph:

        out[n, tc, oy, ox] = 1/(k*k*C) sum_{c, j, i} P1[n, c, y + j, x + i] * P2[n, c, y + j + tj s2, x + i + ti s2],
        y = oy s1 + md, x = ox s1 + md (padded coordinates), tc = (tj + dr) (2 dr + 1) + ti + dr, |j|, |i| <= kr

    (correlation_cuda_kernel.cu:73-147).  `variant` names one of VARIANTS."""
    B, C, H, W = f1.shape
    e, c0, kr, oH, oW, disp, norm = _corr_setup(f1, pad_size, kernel_size, max_displacement, stride1, stride2, variant)
    s1, s2 = stride1, stride2
    nc = 8 * (C // 8) if variant == "drop_tail8" else C
    with torch.no_grad():
        p1, p2 = _corr_pad(f1[:, :nc], e, variant), _corr_pad(f2[:, :nc], e, variant)
        out = f1.new_zeros((B, len(disp), oH, oW))

        def win(p, y, x):
            return p[:, :, y:y + s1 * (oH - 1) + 1:s1, x:x + s1 * (oW - 1) + 1:s1]
        for d, tj, ti in disp:
            for j in range(-kr, kr + 1):
                for i in range(-kr, kr + 1):
                    y, x = c0 + j, c0 + i
                    out[:, d].add_((win(p1, y, x) * win(p2, y + tj * s2, x + ti * s2)).sum(1))
        return out.div_(norm)


def correlation64_backward(f1, f2, grad_output, pad_size, kernel_size, max_displacement, stride1, stride2,
                           variant=None):
    """(grad_input1, grad_input2) of correlation64 (stride1 = 1, as the reference's backward): each displacement plane
    of grad_output times the shifted other input, accumulated for every tap into zero-padded gradients that are then
    cropped, and divided by k*k*C."""
    assert stride1 == 1, "the reference's backward indexes out of bounds for stride1 != 1"
    B, C, H, W = f1.shape
    e, c0, kr, oH, oW, disp, norm = _corr_setup(f1, pad_size, kernel_size, max_displacement, 1, stride2, variant)
    s2, sg2 = stride2, (-1 if variant == "mirror2" else 1)
    with torch.no_grad():
        p1, p2 = _corr_pad(f1, e, variant), _corr_pad(f2, e, variant)
        g1, g2 = torch.zeros_like(p1), torch.zeros_like(p2)

        def win(p, y, x):
            return p[:, :, y:y + oH, x:x + oW]
        for d, tj, ti in disp:
            g = grad_output[:, d:d + 1]
            for j in range(-kr, kr + 1):
                for i in range(-kr, kr + 1):
                    y, x = c0 + j, c0 + i
                    win(g1, y, x).addcmul_(g, win(p2, y + tj * s2, x + ti * s2))
                    win(g2, y + sg2 * tj * s2, x + sg2 * ti * s2).addcmul_(g, win(p1, y, x))
        crop = (slice(None), slice(None), slice(e, e + H), slice(e, e + W))
        g1, g2 = g1[crop].div_(norm), g2[crop].div_(norm)
        if variant == "drop_tail64":
            g1[:, 64 * (C // 64):] = 0
            g2[:, 64 * (C // 64):] = 0
        return g1, g2


def variant_edges(variant, shape, pad_size, kernel_size, max_displacement, stride1, stride2, device="cpu"):
    """(forward mask, grad_input1 mask, grad_input2 mask): the elements on which `variant` can differ from the
    restatement.  replicate: the elements with a tap (forward) or a partner (gradients) in the padding, found by
    filling the padding with 1 instead of 0 on all-ones inputs; the others by their definitions in VARIANTS."""
    B, C, H, W = shape
    prm = (pad_size, kernel_size, max_displacement, stride1, stride2)
    kr, dr, oH, oW = corr_geometry(H, W, *prm)
    ds = 2 * dr + 1
    fwd = torch.zeros((B, ds * ds, oH, oW), dtype=torch.bool, device=device)
    g1 = torch.zeros(shape, dtype=torch.bool, device=device)
    g2 = torch.zeros_like(g1)
    if variant == "replicate":
        one = torch.ones(shape, dtype=torch.float64, device=device)
        fwd = correlation64(one, one, *prm, variant="replicate") != correlation64(one, one, *prm)
        if stride1 == 1:
            go = torch.ones(fwd.shape, dtype=torch.float64, device=device)
            r = correlation64_backward(one, one, go, *prm, variant="replicate")
            z = correlation64_backward(one, one, go, *prm)
            g1, g2 = r[0] != z[0], r[1] != z[1]
    elif variant in ("centre_br", "norm_odd"):
        on = kr > 0 if variant == "centre_br" else kernel_size % 2 == 0
        fwd[:], g1[:], g2[:] = on, on, on
    elif variant == "drop_tail8":
        fwd[:] = C % 8 != 0
    elif variant == "drop_tail64":
        g1[:, 64 * (C // 64):] = True
        g2[:, 64 * (C // 64):] = True
    elif variant == "swap_planes":
        tj, ti = torch.arange(ds * ds, device=device).div(ds, rounding_mode="floor"), torch.arange(ds * ds, device=device) % ds
        fwd[:, tj != ti] = True
        g1[:], g2[:] = ds > 1, ds > 1
    elif variant == "mirror2":
        g2[:] = ds > 1
    else:
        raise ValueError(variant)
    return fwd, g1, g2


def channelnorm32(x):
    """The fp32 ChannelNorm forward as the kernels compute it: acc = fma(x_c, x_c, acc) in channel order (nvcc contracts
    `acc += v * v`), then sqrtf.  Each fma is restated as the exact fp64 product plus acc, rounded to fp64 and then to
    fp32; that equals the single fp32 rounding unless the fp64 sum lands within 2^-53 of an fp32 rounding midpoint."""
    x = x.double()
    acc = torch.zeros_like(x[:, :1]).float()
    for c in range(x.size(1)):
        acc = (x[:, c:c + 1] * x[:, c:c + 1] + acc.double()).float()
    return acc.sqrt()


def channelnorm16(x):
    """The 16-bit ChannelNorm forward (channelnorm_kernel.cu:55-56 on half): each square is computed in fp32 and
    rounded to the storage type, the squares are summed in fp32 in channel order, then sqrtf and one rounding."""
    xf = x.float()
    acc = torch.zeros_like(xf[:, :1])
    for c in range(x.size(1)):
        acc = acc + (xf[:, c:c + 1] * xf[:, c:c + 1]).to(x.dtype).float()
    return acc.sqrt().to(x.dtype)


def channelnorm_backward32(x, o, g):
    """g * x / (o + 1e-9f) in fp32, rounded once to x's dtype (the kernels' 16-bit and fp32 backward)."""
    return (g.float() * x.float() / (o.float() + np.float32(1e-9))).to(x.dtype)


def resample2d(img, flow):
    """grid_sample(border, align_corners=True) restatement of resample2d_kernel.cu:15-72 (k=1)."""
    B, _, H, W = flow.shape
    ys, xs = torch.meshgrid(torch.arange(H, dtype=flow.dtype, device=flow.device),
                            torch.arange(W, dtype=flow.dtype, device=flow.device), indexing="ij")
    gx = 2 * (xs + flow[:, 0]) / max(W - 1, 1) - 1
    gy = 2 * (ys + flow[:, 1]) / max(H - 1, 1) - 1
    return F.grid_sample(img, torch.stack((gx, gy), -1), mode="bilinear", padding_mode="border",
                         align_corners=True)


def channelnorm(x):
    return x.pow(2).sum(1, keepdim=True).sqrt()
