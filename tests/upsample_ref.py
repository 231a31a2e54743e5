"""CPU reference for the backward of the x4 flow upsample and of the fused warp-concat op through it (test support).

nn.Upsample(scale_factor=4) is separable: out = mul * A_h @ in @ A_w^T with one [4n, n] interpolation matrix per axis,
built here from the same formulas orc_upsample4 (oracle/oracle.c) and the kernels' load_flow use:
  bilinear (align_corners=False): src = max(0.25 (y + 0.5) - 0.5, 0), i0 = int(src), i1 = i0 + (i0 < n - 1),
                                  weights 1 - (src - i0) and src - i0 (multiples of 1/8: exact in any precision)
  nearest:                        src = min(y // 4, n - 1)
so the adjoint is mul * A_h^T @ grad @ A_w, evaluated in fp64.  Pinned against torch autograd through
F.interpolate in tests/test_warp_concat_train_cpu.py.
"""
import numpy as np

from oracle import cpu as orc


def upsample4_matrix(n, mode):
    """[4n, n] interpolation matrix of one axis; mode 1 = bilinear, 2 = nearest."""
    A = np.zeros((4 * n, n))
    for y in range(4 * n):
        if mode == 2:
            A[y, min(y // 4, n - 1)] = 1.0
            continue
        if mode != 1:
            raise ValueError("upsample4_matrix: mode must be 1 (bilinear) or 2 (nearest)")
        s = max(0.25 * (y + 0.5) - 0.5, 0.0)
        i0 = int(s)
        i1 = i0 + (1 if i0 < n - 1 else 0)
        A[y, i0] += 1.0 - (s - i0)
        A[y, i1] += s - i0
    return A


def upsample4_backward(grad, mode, mul=1.0):
    """Adjoint of orc.upsample4(planes, mode, mul): grad [B, C, 4h, 4w] -> [B, C, h, w] (fp64)."""
    g = np.asarray(grad, np.float64)
    h, w = g.shape[-2] // 4, g.shape[-1] // 4
    return float(mul) * np.einsum("yi,bcyx,xj->bcij", upsample4_matrix(h, mode), g, upsample4_matrix(w, mode))


def warp_concat_backward(x, flow, grad_cat, C=3, upsample_mode=0, flow_mul=1.0, **layout):
    """Backward of orc.warp_concat_forward(x, flow, C, upsample_mode, flow_mul, ...) -> (grad_x [B,2C,H,W], grad_flow
    shaped like flow): upsample the flow, run the oracle's full-resolution backward composition, apply the adjoint."""
    if not upsample_mode:
        return orc.warp_concat_backward(x, flow, grad_cat, C=C, **layout)
    flow_up = orc.upsample4(flow, upsample_mode, flow_mul)
    gx, g_up = orc.warp_concat_backward(x, flow_up, grad_cat, C=C, **layout)
    return gx, upsample4_backward(g_up, upsample_mode, flow_mul).astype(np.float32)
