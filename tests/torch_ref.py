"""Stock-PyTorch formulations of the three layers ("oracle C" in SURVEY.md section 4).

Independent third opinion used to pin the CPU restatement: autograd through these gives the
gradients.  fp64-capable, CPU or CUDA.  Test helper only.
"""
import math

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


def _corr_geometry(f, pad_size, max_displacement, stride2):
    B, C, H, W = f.shape
    dr = max_displacement // stride2
    oH, oW = H + 2 * pad_size - 2 * max_displacement, W + 2 * pad_size - 2 * max_displacement
    shifts = [(max_displacement + tj * stride2, max_displacement + ti * stride2)
              for tj in range(-dr, dr + 1) for ti in range(-dr, dr + 1)]
    return C, oH, oW, shifts


def correlation_k1(f1, f2, pad_size, max_displacement, stride2):
    """The kernel_size = 1, stride1 = 1 forward as an explicit sum over the (2 dr + 1)^2 displacements of shifted
    products of the zero-padded inputs, in the inputs' dtype (fp64 for a reference), without an autograd graph:
    out[n, d, y, x] = 1/C sum_c P1[n, c, y + md, x + md] * P2[n, c, y + md + tj s2, x + md + ti s2]."""
    C, oH, oW, shifts = _corr_geometry(f1, pad_size, max_displacement, stride2)
    with torch.no_grad():
        p1, p2 = F.pad(f1, (pad_size,) * 4), F.pad(f2, (pad_size,) * 4)
        md = max_displacement
        a = p1[:, :, md:md + oH, md:md + oW]
        out = f1.new_empty((f1.size(0), len(shifts), oH, oW))
        for d, (sy, sx) in enumerate(shifts):
            torch.sum(a * p2[:, :, sy:sy + oH, sx:sx + oW], 1, out=out[:, d])
        return out.div_(C)


def correlation_k1_backward(f1, f2, grad_output, pad_size, max_displacement, stride2):
    """(grad_input1, grad_input2) of correlation_k1: each displacement plane of grad_output times the shifted other
    input, accumulated into zero-padded gradients that are then cropped."""
    C, oH, oW, shifts = _corr_geometry(f1, pad_size, max_displacement, stride2)
    B, _, H, W = f1.shape
    with torch.no_grad():
        p1, p2 = F.pad(f1, (pad_size,) * 4), F.pad(f2, (pad_size,) * 4)
        g1, g2 = torch.zeros_like(p1), torch.zeros_like(p2)
        md = max_displacement
        a, ga = p1[:, :, md:md + oH, md:md + oW], g1[:, :, md:md + oH, md:md + oW]
        for d, (sy, sx) in enumerate(shifts):
            g = grad_output[:, d:d + 1]
            ga.addcmul_(g, p2[:, :, sy:sy + oH, sx:sx + oW])
            g2[:, :, sy:sy + oH, sx:sx + oW].addcmul_(g, a)
        crop = (slice(None), slice(None), slice(pad_size, pad_size + H), slice(pad_size, pad_size + W))
        return g1[crop].div_(C), g2[crop].div_(C)


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
