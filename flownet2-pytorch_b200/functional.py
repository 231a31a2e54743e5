"""Tensor-level entry points: torch tensors in, libfn2b200's kernels on the current stream, outputs out.

These are the functions the ``*_cuda`` shim modules, the benchmarks and the tools share.  Each one sets its defaults
and makes one call into the operator library's host-side glue (``pybind/ext_common.h``), which the operators and the
compiled ``*_cuda`` modules call too: the device and shape checks, the checks on ``out=`` tensors, workspaces and the
C-ABI call live there, once.  Argument errors raise RuntimeError.  All arithmetic happens in libfn2b200's hand-written
sm_90a kernels.
"""
import ctypes

from ._lib import LIB, OPS, check


def _require_cuda(*tensors):
    for t in tensors:
        if t is not None and not t.is_cuda:
            raise RuntimeError(
                "flownet2-pytorch_b200 runs on CUDA tensors only (got a %s tensor); there is no CPU "
                "fallback -- the reference has none either (correlation.py:4)" % t.device.type)


def _img_strides(img):
    """An image's strides as the C ABI's int64_t[4], for calling the C ABI directly (the tests of its entry points)."""
    return (ctypes.c_int64 * 4)(*img.stride())


def correlation_out_shape(C, H, W, pad_size, kernel_size, max_displacement, stride1, stride2):
    D, oH, oW = ctypes.c_int(), ctypes.c_int(), ctypes.c_int()
    check(LIB.fn2b200_correlation_out_shape(C, H, W, pad_size, kernel_size, max_displacement, stride1,
                                            stride2, ctypes.byref(D), ctypes.byref(oH), ctypes.byref(oW)),
          "correlation_out_shape")
    return D.value, oH.value, oW.value


class CorrWorkspace(object):
    """Scratch of the tensor-core correlation path (bf16 hi/lo copies of input1/input2).  Returned by
    ``correlation_forward(..., return_workspace=True)`` and accepted by ``correlation_backward`` so the
    backward can skip the split pass when it runs on the SAME inputs (what autograd does)."""
    __slots__ = ("buf", "key")

    def __init__(self, buf, key):
        self.buf, self.key = buf, key


def _ws_key(a, b, prm):
    # the split is of the fp32-contiguous values of a and b: the same tensors (storage, layout, dtype), not modified
    # in place since, hold the same values
    return (a.data_ptr(), b.data_ptr(), a._version, b._version, tuple(a.shape), a.stride(), b.stride(), a.dtype,
            b.dtype) + tuple(prm)


def _workspace(ws, a, b, prm):
    return CorrWorkspace(ws, _ws_key(a, b, prm)) if ws.numel() else None


def _split(workspace, a, b, prm):
    """The forward's workspace when it still holds the split of these inputs, else None."""
    return workspace.buf if workspace is not None and workspace.key == _ws_key(a, b, prm) else None


def correlation_forward(input1, input2, pad_size, kernel_size, max_displacement, stride1, stride2,
                        corr_multiply=1, out=None, return_workspace=False):
    prm = (pad_size, kernel_size, max_displacement, stride1, stride2)
    out, ws = OPS.correlation_forward(input1, input2, out, False, 0, 1.0, *prm, corr_multiply)
    return (out, _workspace(ws, input1, input2, prm)) if return_workspace else out


def correlation_forward_cat(input1, input2, cat, ch_offset, leaky_slope, pad_size, kernel_size, max_displacement, stride1,
                            stride2, corr_multiply=1, return_workspace=False):
    """LeakyReLU(leaky_slope)(Correlation(...)(input1, input2)) written into cat[:, ch_offset : ch_offset + D] in place
    (FlowNetC.py:86-92: `torch.cat((out_conv_redir, corr_activation(corr)), 1)` without the activation pass and without
    the copy).  cat: contiguous fp32 [B, channels, oH, oW]; its other channels are left alone.  Returns cat, or
    (cat, CorrWorkspace or None) with return_workspace=True, for correlation_backward_cat."""
    prm = (pad_size, kernel_size, max_displacement, stride1, stride2)
    cat, ws = OPS.correlation_forward(input1, input2, cat, True, ch_offset, leaky_slope, *prm, corr_multiply)
    return (cat, _workspace(ws, input1, input2, prm)) if return_workspace else cat


def correlation_backward_cat(input1, input2, grad_cat, cat, ch_offset, leaky_slope, pad_size, kernel_size,
                             max_displacement, stride1, stride2, corr_multiply=1, need1=True, need2=True, workspace=None):
    """Backward of correlation_forward_cat: the input gradients of
    cat[:, ch_offset : ch_offset + D] = LeakyReLU(leaky_slope)(Correlation(...)(input1, input2)), read straight from
    grad_cat (the gradient of the whole concat) with LeakyReLU's derivative taken from `cat`, the buffer the forward
    wrote (may be None when leaky_slope == 1).  One kernel launch on the tensor-core path when `workspace` is what
    correlation_forward_cat(..., return_workspace=True) returned for the same inputs.  Returns (grad1, grad2)."""
    prm = (pad_size, kernel_size, max_displacement, stride1, stride2)
    return OPS.correlation_backward(input1, input2, grad_cat, True, cat, ch_offset, leaky_slope,
                                    _split(workspace, input1, input2, prm), *prm, corr_multiply, need1, need2, None, None)


def correlation_backward(input1, input2, grad_output, pad_size, kernel_size, max_displacement, stride1,
                         stride2, corr_multiply=1, need1=True, need2=True, out1=None, out2=None, workspace=None):
    prm = (pad_size, kernel_size, max_displacement, stride1, stride2)
    return OPS.correlation_backward(input1, input2, grad_output, False, None, 0, 1.0,
                                    _split(workspace, input1, input2, prm), *prm, corr_multiply, need1, need2, out1, out2)


def resample2d_forward(input1, input2, kernel_size=1, bilinear=True, out=None):
    return OPS.resample2d_forward(input1, input2, out, kernel_size, bilinear, 0, 1.0)


def resample2d_backward(input1, input2, grad_output, kernel_size=1, bilinear=True, need1=True, need2=True,
                        out1=None, out2=None, zero_out1=True):
    return OPS.resample2d_backward(input1, input2, grad_output, kernel_size, bilinear, need1, need2, out1, out2,
                                   zero_out1)


UPSAMPLE_MODES = {None: 0, "none": 0, 0: 0, "bilinear": 1, 1: 1, "nearest": 2, 2: 2}


def resample2d_forward_up(input1, flow_lr, upsample="bilinear", flow_mul=1.0, out=None):
    """Resample2d()(input1, nn.Upsample(scale_factor=4, mode=upsample)(flow_lr * flow_mul)) without materialising the
    full-resolution flow (models.py:130-133): the kernel interpolates the quarter-resolution flow per pixel."""
    return OPS.resample2d_forward(input1, flow_lr, out, 1, True, UPSAMPLE_MODES[upsample], flow_mul)


def _layout(C, ch_x, n_x, ch_warped, ch_flow, ch_flow_norm, ch_diff_norm):
    """models.py:138's concat1 layout (x | warped | flow / div_flow | diff norm) where an argument is None."""
    return (ch_x, 2 * C if n_x is None else n_x, 2 * C if ch_warped is None else ch_warped,
            3 * C if ch_flow is None else ch_flow, ch_flow_norm, 3 * C + 2 if ch_diff_norm is None else ch_diff_norm)


def warp_concat_forward(x, flow, C=3, upsample=None, flow_mul=1.0, flow_div=1.0, out=None, cat_channels=None, ch_x=0,
                        n_x=None, ch_warped=None, ch_flow=None, ch_flow_norm=-1, ch_diff_norm=None):
    """One kernel for the chain models.py:130-138 spells out with five modules and a torch.cat:

        flow_up = upsample(flow * flow_mul)            (upsample in {None, "bilinear", "nearest"}; None: flow is full-res)
        warped  = Resample2d()(x[:, C:2C], flow_up);   diff_norm = ChannelNorm()(x[:, :C] - warped)
        out[:, ch_x:ch_x+n_x] = x[:, :n_x];  out[:, ch_warped:+C] = warped;  out[:, ch_flow:+2] = flow_up / flow_div
        out[:, ch_flow_norm] = ChannelNorm()(flow_up);  out[:, ch_diff_norm] = diff_norm

    Defaults = models.py:138's 12-channel `concat1` (x | warped | flow / div_flow | diff norm).  A negative ch_* skips
    that product; channels nobody writes keep whatever `out` held.  x may be a strided view (unit stride along W)."""
    return OPS.warp_concat_forward(x, flow, out, C, UPSAMPLE_MODES[upsample], flow_mul, flow_div,
                                   3 * C + 3 if cat_channels is None else cat_channels,
                                   *_layout(C, ch_x, n_x, ch_warped, ch_flow, ch_flow_norm, ch_diff_norm))


def warp_concat_backward(x, flow, grad_cat, C=3, flow_div=1.0, ch_x=0, n_x=None, ch_warped=None, ch_flow=None,
                         ch_flow_norm=-1, ch_diff_norm=None, upsample=None, flow_mul=1.0, need_x=True, need_flow=True):
    """Backward of warp_concat_forward(x, flow, upsample=upsample, flow_mul=flow_mul, ...): returns (grad_x [B,2C,H,W],
    grad_flow shaped like flow -- the quarter-resolution flow's gradient when upsample is "bilinear" / "nearest").  The
    layout arguments must be the forward's; C <= 3.  need_x / need_flow = False skips that gradient (None is returned
    for it): without grad_x the kernel does no image-gradient scatter.  grad_flow is bit-identical from run to run and
    whether or not grad_x is computed."""
    return OPS.warp_concat_backward(x, flow, grad_cat, C, UPSAMPLE_MODES[upsample], flow_mul, flow_div,
                                    *_layout(C, ch_x, n_x, ch_warped, ch_flow, ch_flow_norm, ch_diff_norm), need_x,
                                    need_flow)


def channelnorm_forward(input1, norm_deg=2, out=None):
    """fp16 / bf16 inputs run natively (out in their dtype), anything else as fp32."""
    return OPS.channelnorm_forward(input1, out, norm_deg)


def channelnorm_backward(input1, output, grad_output, norm_deg=2, out=None):
    """Natively 16-bit when all three share an fp16 / bf16 dtype (out in that dtype), fp32 otherwise."""
    return OPS.channelnorm_backward(input1, output, grad_output, out, norm_deg)


def launch_count():
    """Kernel launches issued by libfn2b200 in this PROCESS so far (one atomic counter, all threads)."""
    return int(LIB.fn2b200_launch_count())
