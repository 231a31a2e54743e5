"""CPU tests of the warp-concat backward through the x4 flow upsample (fn2b200_warp_concat_backward_up and the Python
layers on it): the CPU reference for the upsample's adjoint and the composed backward against fp64 torch autograd,
argument errors reported before anything touches the device, and the Python surface."""
import ctypes
import inspect

import numpy as np
import pytest
import torch
import torch.nn.functional as TF

import upsample_ref as ur
from oracle import cpu as orc

P, I64 = ctypes.c_void_p, ctypes.c_int64 * 4
MODES = [(1, "bilinear"), (2, "nearest")]


@pytest.mark.parametrize("mode,name", MODES)
@pytest.mark.parametrize("h,w", [(1, 1), (3, 5), (10, 18)])
def test_upsample4_backward_equals_fp64_autograd(mode, name, h, w):
    g = torch.Generator().manual_seed(h * 100 + w)
    lr = torch.randn(2, 2, h, w, generator=g, dtype=torch.float64, requires_grad=True)
    up = TF.interpolate(lr * 20.0, scale_factor=4, mode=name, **({"align_corners": False} if mode == 1 else {}))
    # the matrices are the forward of orc.upsample4 too
    fwd = 20.0 * np.einsum("yi,bcij,xj->bcyx", ur.upsample4_matrix(h, mode), lr.detach().numpy(), ur.upsample4_matrix(w, mode))
    assert np.abs(fwd - up.detach().numpy()).max() <= 1e-12 * max(1.0, np.abs(fwd).max())
    assert np.abs(orc.upsample4(lr.detach().numpy(), mode, 20.0) - fwd).max() <= 1e-5 * max(1.0, np.abs(fwd).max())
    gu = torch.randn(up.shape, generator=g, dtype=torch.float64)
    up.backward(gu)
    got = ur.upsample4_backward(gu.numpy(), mode, 20.0)
    assert got.shape == (2, 2, h, w)
    assert np.abs(got - lr.grad.numpy()).max() <= 1e-12 * np.abs(lr.grad.numpy()).max()


def _resample_fp64(img, flow_up):
    """Resample2d's bilinear warp in fp64 (grid_sample, border, align_corners=True: see test_oracle_cpu)."""
    H, W = flow_up.shape[-2:]
    yy, xx = torch.meshgrid(torch.arange(H).double(), torch.arange(W).double(), indexing="ij")
    grid = torch.stack(((xx + flow_up[:, 0]) / (W - 1) * 2 - 1, (yy + flow_up[:, 1]) / (H - 1) * 2 - 1), -1)
    return TF.grid_sample(img, grid, mode="bilinear", padding_mode="border", align_corners=True)


@pytest.mark.parametrize("mode,name", MODES)
def test_warp_concat_backward_up_composition_against_fp64_autograd(mode, name):
    g = torch.Generator().manual_seed(5 + mode)
    x = torch.rand(1, 6, 12, 16, generator=g) - 0.5
    lr = torch.randn(1, 2, 3, 4, generator=g) * 0.1
    norm = lambda t: t.pow(2).sum(1, keepdim=True).sqrt()
    for layout, mul in ((dict(flow_div=20.0), 20.0),                                     # concat1 / concat2
                        (dict(flow_div=1.0, cat_channels=11, ch_x=0, n_x=3, ch_warped=-1, ch_flow=3,
                              ch_flow_norm=7, ch_diff_norm=9), 0.05)):                   # concat3, FlowNetSD half
        fwd_layout = {k: v for k, v in layout.items()}
        cat = orc.warp_concat_forward(x.numpy(), lr.numpy(), upsample_mode=mode, flow_mul=mul, **fwd_layout)
        gc = torch.randn(cat.shape, generator=g)
        bwd_layout = {k: v for k, v in layout.items() if k != "cat_channels"}
        rx, rf = ur.warp_concat_backward(x.numpy(), lr.numpy(), gc.numpy(), upsample_mode=mode, flow_mul=mul, **bwd_layout)
        assert rf.shape == (1, 2, 3, 4) and rx.shape == (1, 6, 12, 16)
        xd, fd = x.double().requires_grad_(), lr.double().requires_grad_()
        up = TF.interpolate(fd * mul, scale_factor=4, mode=name, **({"align_corners": False} if mode == 1 else {}))
        warped = _resample_fp64(xd[:, 3:], up)
        dn = norm(xd[:, :3] - warped)
        if "cat_channels" in layout:
            ref = torch.cat((xd[:, :3], up, torch.zeros_like(up), norm(up), torch.zeros_like(dn), dn, torch.zeros_like(dn)), 1)
        else:
            ref = torch.cat((xd, warped, up / 20.0, dn), 1)
        assert np.abs(cat - ref.detach().numpy()).max() < 1e-5
        ref.backward(gc.double())
        assert np.abs(rx - xd.grad.numpy()).max() < 1e-5 * max(1.0, np.abs(rx).max())
        assert np.abs(rf - fd.grad.numpy()).max() < 1e-5 * max(1.0, np.abs(rf).max())


def _bwd_up(C=3, fh=2, fw=2, mode=1, cat_channels=12, layout=(0, 6, 6, 9, 20.0, -1, 11), gx=P(16), gf=P(16),
            ws=P(0), ws_bytes=0, B=1, H=8, W=8, x=P(16)):
    from flownet2_b200._lib import LIB
    one = P(16)                  # never dereferenced: validation fails (or a no-op returns) first
    st = I64(6 * H * W, H * W, W, 1)
    ch_x, n_x, ch_warped, ch_flow, flow_div, ch_flow_norm, ch_diff_norm = layout
    return LIB.fn2b200_warp_concat_backward_up(x, st, C, one, fh, fw, mode, 20.0, one, cat_channels, ch_x, n_x, ch_warped,
                                               ch_flow, flow_div, ch_flow_norm, ch_diff_norm, gx, gf, ws, ws_bytes, B, H,
                                               W, P(0))


def test_backward_up_argument_validation():
    from flownet2_b200._lib import LIB
    err = lambda: LIB.fn2b200_last_error()
    need = int(LIB.fn2b200_warp_concat_backward_up_workspace(1, 3, 8, 8, 1, 1))
    assert _bwd_up(mode=3, ws=P(16), ws_bytes=need) == -1 and b"upsample_mode 3" in err()
    assert _bwd_up(fh=2, fw=3, ws=P(16), ws_bytes=need) == -1 and b"does not match" in err()
    assert _bwd_up(mode=0, ws=P(16), ws_bytes=need) == -1 and b"does not match" in err()       # mode 0 wants fh = H
    assert _bwd_up(C=4, ws=P(16), ws_bytes=need) == -2 and b"C=4 > 3" in err()
    assert _bwd_up(layout=(0, 6, 4, 9, 20.0, -1, 11), ws=P(16), ws_bytes=need) == -1 and b"overlap" in err()
    assert _bwd_up(ws=P(16), ws_bytes=need - 16) == -1 and b"workspace" in err()
    assert _bwd_up(ws=P(0), ws_bytes=need) == -1 and b"workspace" in err()
    assert _bwd_up(ws=P(24), ws_bytes=need) == -1 and b"16-byte aligned" in err()
    # the 2^31-element guard on the concat gradient
    assert _bwd_up(B=4096, H=256, W=256, fh=64, fw=64, ws=P(16), ws_bytes=1 << 40) == -1
    assert b"warp_concat_backward_up: tensor exceeds 2^31" in err()
    # a NULL x with a gradient wanted
    assert _bwd_up(x=P(0), ws=P(16), ws_bytes=need) == -3 and b"null pointer" in err()
    # no gradient wanted, and B == 0: successful no-ops
    assert _bwd_up(gx=P(0), gf=P(0)) == 0
    assert _bwd_up(B=0, x=P(0), gx=P(0)) == 0


def test_backward_up_workspace_query():
    from flownet2_b200._lib import LIB
    q = LIB.fn2b200_warp_concat_backward_up_workspace
    scratch = 2 * 448 * 1024 * 16                                 # the image-gradient scatter scratch, B = 2
    partials = 2 * (1024 // 32) * (448 // 16) * 2 * 6 * 10 * 4     # 2 x 6 x 10 floats per 32 x 16 tile
    assert q(2, 3, 448, 1024, 2, 0) == 0
    assert q(2, 3, 448, 1024, 2, 1) == scratch
    assert q(2, 3, 448, 1024, 1, 0) == partials
    assert q(2, 3, 448, 1024, 1, 1) == scratch + partials
    assert q(2, 3, 448, 1024, 0, 1) == LIB.fn2b200_warp_concat_backward_workspace(2, 3, 448, 1024) == scratch
    assert q(2, 3, 448, 1024, 0, 0) == 0
    assert q(2, 4, 448, 1024, 1, 1) == 0 and q(2, 3, 448, 1024, 3, 1) == 0 and q(0, 3, 448, 1024, 1, 1) == 0


def test_python_surface_and_no_cpu_fallback():
    import flownet2_b200 as f
    sig = inspect.signature(f.functional.warp_concat_backward)
    assert list(sig.parameters)[-4:] == ["upsample", "flow_mul", "need_x", "need_flow"]
    assert [sig.parameters[k].default for k in ("upsample", "flow_mul", "need_x", "need_flow")] == [None, 1.0, True, True]
    assert list(inspect.signature(f.fused.WarpConcat.__init__).parameters)[1:] == ["div_flow", "upsample"]
    assert inspect.signature(f.fused.WarpConcat).parameters["upsample"].default is None
    assert list(inspect.signature(f.fused.FusionConcat.__init__).parameters)[1:] == ["div_flow"]
    assert list(inspect.signature(f.fused.flownet2_train_forward).parameters) == ["net", "inputs"]
    x, lr = torch.zeros(1, 6, 8, 8), torch.zeros(1, 2, 2, 2)
    with pytest.raises(RuntimeError, match="CUDA tensors only"):
        f.functional.warp_concat_backward(x, lr, torch.zeros(1, 12, 8, 8), upsample="bilinear", flow_mul=20.0)
    with pytest.raises(RuntimeError, match="CUDA tensors only"):
        f.fused.WarpConcat(20.0, upsample="bilinear")(x, lr)
    with pytest.raises(RuntimeError, match="CUDA tensors only"):
        f.fused.FusionConcat(20.0)(x, lr, lr)
