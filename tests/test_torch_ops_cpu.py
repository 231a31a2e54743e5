"""torch.ops.fn2b200 without a GPU: the operator library loads and registers every schema, and the fake kernels give
the C ABI's shapes and workspace sizes (meta tensors run the fake kernels)."""
import itertools
import subprocess
import sys

import pytest
import torch

import flownet2_b200 as f
from flownet2_b200 import ops
from flownet2_b200._lib import LIB

fn = torch.ops.fn2b200


def _meta(*shape, dtype=torch.float32):
    return torch.empty(*shape, dtype=dtype, device="meta")


def test_library_loads_without_gpu_and_registers_every_schema():
    code = ("import torch, sys; torch.ops.load_library(sys.argv[1]); "
            "print(' '.join(sorted(s.name.split('::')[1] for s in torch._C._jit_get_all_schemas() "
            "if s.name.startswith('fn2b200::'))))")
    r = subprocess.run([sys.executable, "-c", code, ops.LIBRARY_PATH], capture_output=True, text=True, timeout=300,
                       env={"CUDA_VISIBLE_DEVICES": "", "PATH": "/usr/bin:/bin"})
    assert r.returncode == 0, r.stderr[-2000:]
    assert r.stdout.split() == sorted(ops.OPS)
    for name in ops.OPS:
        assert getattr(fn, name).default._schema.name == "fn2b200::" + name


def test_modules_refuse_cpu_tensors():
    x = torch.zeros(1, 6, 8, 8)
    with pytest.raises(RuntimeError, match="CUDA tensors only"):
        f.CorrelationFunction.apply(x, x, 0, 1, 0, 1, 1)
    with pytest.raises(RuntimeError, match="CUDA tensors only"):
        f.fused.CorrelationCat(0, 1, 0, 1, 1)(x, x, x)
    with pytest.raises(RuntimeError, match="not implemented for 'CPU'|CPU"):
        fn.channelnorm_forward(x, 2)


GRID = list(itertools.product([(1, 64, 8, 16), (2, 256, 48, 64), (2, 20, 13, 36), (1, 128, 7, 9)],
                              [(20, 1, 20, 1, 2), (4, 1, 4, 1, 1), (3, 3, 3, 1, 1), (0, 1, 0, 1, 1), (2, 1, 4, 2, 2),
                               (5, 3, 6, 3, 2)]))


@pytest.mark.parametrize("env", [None, "fma"])
def test_fake_correlation_shapes_and_workspace_follow_the_c_abi(env, monkeypatch):
    if env:
        monkeypatch.setenv("FN2B200_CORR_FWD", env)
    checked = 0
    for (B, C, H, W), prm in GRID:
        D, oH, oW = f.functional.correlation_out_shape(C, H, W, *prm)
        if oH <= 0 or oW <= 0:
            continue
        ws = int(LIB.fn2b200_correlation_forward_workspace(B, C, H, W, *prm))
        if env:
            assert ws == 0
        a = _meta(B, C, H, W)
        out, w = fn.correlation_forward(a, a, *prm, 1)
        assert tuple(out.shape) == (B, D, oH, oW) and out.dtype == torch.float32
        assert tuple(w.shape) == (ws,) and w.dtype == torch.uint8
        cat, w2 = fn.correlation_forward_cat(_meta(B, 32, oH, oW), a, a, *prm, 1, 0.1)
        assert tuple(cat.shape) == (B, 32 + D, oH, oW) and tuple(w2.shape) == (ws,)
        g1, g2 = fn.correlation_backward(a, a, out, w, *prm, 1, True, False)
        assert tuple(g1.shape) == (B, C, H, W) and g2.numel() == 0
        g1, g2 = fn.correlation_backward_cat(a, a, cat, cat, w2, 32, 0.1, *prm, 1, False, True)
        assert g1.numel() == 0 and tuple(g2.shape) == (B, C, H, W)
        checked += 1
    assert checked >= 20
    # the tensor-core configuration of FlowNetC has a workspace unless FN2B200_CORR_FWD=fma
    assert (int(LIB.fn2b200_correlation_forward_workspace(2, 256, 48, 64, 20, 1, 20, 1, 2)) > 0) == (env is None)


def test_fake_float_ceil_output_shape():
    """oH = ceil((H + 2 pad - 2 (kr + md)) / s1) in float: s1 = 3 on 11 + 2*5 - 2*(1 + 6) = 7 rows -> 3."""
    out, _ = fn.correlation_forward(_meta(1, 8, 11, 12), _meta(1, 8, 11, 12), 5, 3, 6, 3, 2, 1)
    assert tuple(out.shape) == (1, 49, 3, 3)


def test_fake_layer_and_fused_shapes():
    img, flow = _meta(2, 3, 16, 24), _meta(2, 2, 16, 24)
    assert tuple(fn.resample2d_forward(img, flow, 1, True).shape) == (2, 3, 16, 24)
    g1, g2 = fn.resample2d_backward(_meta(3, 3, 16, 24), flow, img, 1, True, True, True)
    assert tuple(g1.shape) == (3, 3, 16, 24) and tuple(g2.shape) == (2, 2, 16, 24)
    for dt, out_dt in ((torch.float32, torch.float32), (torch.float16, torch.float16), (torch.bfloat16, torch.bfloat16),
                       (torch.float64, torch.float32)):
        x = _meta(2, 3, 16, 24, dtype=dt)
        o = fn.channelnorm_forward(x, 2)
        assert tuple(o.shape) == (2, 1, 16, 24) and o.dtype == out_dt
        assert fn.channelnorm_backward(x, o, o, 2).dtype == out_dt
    x, lr = _meta(2, 6, 16, 24), _meta(2, 2, 4, 6)
    assert tuple(fn.warp_concat_forward(x, lr, 3, 1, 20.0, 20.0, 12, 0, 6, 6, 9, -1, 11).shape) == (2, 12, 16, 24)
    gx, gf = fn.warp_concat_backward(x, lr, _meta(2, 12, 16, 24), 3, 1, 20.0, 20.0, 0, 6, 6, 9, -1, 11, False, True)
    assert gx.numel() == 0 and tuple(gf.shape) == (2, 2, 4, 6)
    c3 = fn.fusion_concat(x, lr, lr, 20.0)
    assert tuple(c3.shape) == (2, 11, 16, 24)
    gx, gs, g2 = fn.fusion_concat_backward(x, lr, lr, c3, 20.0, True, False, True)
    assert tuple(gx.shape) == (2, 6, 16, 24) and gs.numel() == 0 and tuple(g2.shape) == (2, 2, 4, 6)
