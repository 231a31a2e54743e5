"""CPU tests of the concat-gradient correlation backward (fn2b200_correlation_backward_cat): argument errors are
reported before anything touches the device, and the Python surface exists with the documented signatures."""
import ctypes
import inspect

import pytest
import torch

P = ctypes.c_void_p
PRM = (20, 1, 20, 1, 2)          # FlowNetC: pad, kernel_size, max_displacement, stride1, stride2 -> D = 441


def _bwd_cat(cat_ptr, cat_channels, ch_offset, slope, B=1, C=64, H=8, W=8, prm=PRM):
    from flownet2_b200._lib import LIB
    one = P(16)                  # never dereferenced: validation fails (or B == 0 returns) first
    return LIB.fn2b200_correlation_backward_cat(one, one, one, cat_ptr, cat_channels, ch_offset, slope, one, one,
                                                B, C, H, W, *prm, 1, P(0), 0, 0, P(0))


def test_backward_cat_argument_validation():
    from flownet2_b200._lib import LIB
    one = P(16)
    # channel range does not fit the buffer
    assert _bwd_cat(one, 440, 0, 0.1) == -1 and b"do not fit" in LIB.fn2b200_last_error()
    assert _bwd_cat(one, 473, 33, 0.1) == -1 and b"do not fit" in LIB.fn2b200_last_error()
    assert _bwd_cat(one, 473, -1, 0.1) == -1
    # a negative slope: the sign of the activated output no longer gives the mask
    assert _bwd_cat(one, 473, 32, -0.1) == -1 and b"leaky_slope" in LIB.fn2b200_last_error()
    assert _bwd_cat(one, 473, 32, float("nan")) == -1
    # NULL cat needs slope 1 (no activation)
    assert _bwd_cat(P(0), 473, 32, 0.1) == -3 and b"null" in LIB.fn2b200_last_error()
    assert _bwd_cat(P(0), 473, 32, 0.0) == -3
    # stride1 != 1: unsupported, as for the plain backward
    assert _bwd_cat(one, 473, 32, 0.1, H=12, W=13, prm=(2, 1, 4, 2, 2)) == -2
    assert b"stride1" in LIB.fn2b200_last_error()
    # the 2^31-element guard on the concat buffer (offsets inside the kernels are 32-bit)
    # (the cost volume alone, 2048 x 441 x 40 x 40, stays below 2^31)
    assert _bwd_cat(one, 2000, 32, 0.1, B=2048, H=40, W=40) == -1
    assert b"correlation_backward_cat: tensor exceeds 2^31" in LIB.fn2b200_last_error()
    # B == 0 is a successful no-op, even with NULL pointers
    assert LIB.fn2b200_correlation_backward_cat(P(0), P(0), P(0), P(0), 473, 32, ctypes.c_float(0.1), P(0), P(0),
                                                0, 64, 8, 8, *PRM, 1, P(0), 0, 0, P(0)) == 0


def test_backward_cat_python_surface():
    import flownet2_b200 as f
    sig = inspect.signature(f.functional.correlation_backward_cat)
    assert list(sig.parameters)[:6] == ["input1", "input2", "grad_cat", "cat", "ch_offset", "leaky_slope"]
    assert (sig.parameters["need1"].default, sig.parameters["need2"].default, sig.parameters["workspace"].default) == (
        True, True, None)
    assert inspect.signature(f.functional.correlation_forward_cat).parameters["return_workspace"].default is False
    m = f.fused.CorrelationCat(20, 1, 20, 1, 2, 1)
    assert m.leaky_slope == 0.1 and not list(m.parameters())
    with pytest.raises(RuntimeError, match="CUDA tensors only"):
        m(torch.zeros(1, 32, 8, 8), torch.zeros(1, 64, 8, 8), torch.zeros(1, 64, 8, 8))


def test_train_forward_refuses_flownet2():
    import flownet2_b200 as f

    class FlowNet2(torch.nn.Module):
        pass

    with pytest.raises(TypeError, match="FlowNet2 has no differentiable fused data flow"):
        f.fused.train_forward(FlowNet2(), torch.zeros(1, 3, 2, 8, 8))
