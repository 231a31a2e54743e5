"""The layers and the fused ops as PyTorch operators: ``torch.ops.fn2b200.*``.

``pybind/fn2b200_ops.cc`` defines the operators (``TORCH_LIBRARY(fn2b200, m)``) and their CUDA kernels on the host-side
glue every route shares (``pybind/ext_common.h``); ``_lib`` loads that library, and this module registers, for each
forward, a fake kernel (shapes and dtypes without running anything, for torch.compile / torch.export) and an autograd
formula whose backward is the matching ``*_backward`` operator.  Only the gradients in ``ctx.needs_input_grad`` are
computed.  The modules and ``*Function`` classes of the package (``Correlation``, ``Resample2d``, ``ChannelNorm``,
``fused.CorrelationCat`` / ``WarpConcat`` / ``FusionConcat``) call these operators, so Dynamo traces them without a graph break, CUDA graphs capture them and
``torch.export`` records them as ``fn2b200.*`` calls.  An exported program needs only the operator library:
``torch.ops.load_library(flownet2_b200.ops.LIBRARY_PATH)``.

The correlation forward returns its tensor-core workspace (the bf16 hi/lo split of both inputs, uint8, empty when the
FP32-FMA kernels run) as a second output; autograd saves it and hands it to the backward, which then skips the split
pass.  Its size comes from ``fn2b200_correlation_forward_workspace`` at trace time, so a compiled graph is specialised
on the input sizes and on ``FN2B200_CORR_FWD``.
"""
import torch

from . import functional as F2
from ._lib import LIB, OPS_LIBRARY_PATH as LIBRARY_PATH  # noqa: F401  (importing _lib registers the operators)

#: every operator the library defines
OPS = ("correlation_forward", "correlation_backward", "correlation_forward_cat", "correlation_backward_cat",
       "resample2d_forward", "resample2d_backward", "channelnorm_forward", "channelnorm_backward",
       "warp_concat_forward", "warp_concat_backward", "fusion_concat", "fusion_concat_backward")

fn2b200 = torch.ops.fn2b200
_reg_fake = torch.library.register_fake
_reg_autograd = torch.library.register_autograd


def _nothing(t):
    """The placeholder output of a gradient that was not asked for."""
    return t.new_empty((0,), dtype=torch.float32)


def _f32(t, shape=None):
    return t.new_empty(tuple(t.shape) if shape is None else shape, dtype=torch.float32)


# ---- correlation ------------------------------------------------------------------------------------------------------

def _corr_geometry(input1, prm):
    """(B, C, H, W) and (D, oH, oW) from the C ABI (fn2b200_correlation_out_shape's float ceil); concrete sizes."""
    B, C, H, W = (int(s) for s in input1.shape)
    D, oH, oW = F2.correlation_out_shape(C, H, W, *prm)
    if oH <= 0 or oW <= 0:
        raise ValueError("correlation: empty output (%d x %d) for input %dx%d" % (oH, oW, H, W))
    return (B, C, H, W), (D, oH, oW)


def _corr_workspace(input1, bchw, prm):
    return input1.new_empty((int(LIB.fn2b200_correlation_forward_workspace(*bchw, *prm)),), dtype=torch.uint8)


@_reg_fake("fn2b200::correlation_forward")
def _(input1, input2, pad_size, kernel_size, max_displacement, stride1, stride2, corr_multiply=1):
    prm = (pad_size, kernel_size, max_displacement, stride1, stride2)
    bchw, (D, oH, oW) = _corr_geometry(input1, prm)
    return _f32(input1, (bchw[0], D, oH, oW)), _corr_workspace(input1, bchw, prm)


@_reg_fake("fn2b200::correlation_forward_cat")
def _(redir, input1, input2, pad_size, kernel_size, max_displacement, stride1, stride2, corr_multiply=1, leaky_slope=0.1):
    prm = (pad_size, kernel_size, max_displacement, stride1, stride2)
    bchw, (D, oH, oW) = _corr_geometry(input1, prm)
    return _f32(input1, (bchw[0], redir.shape[1] + D, oH, oW)), _corr_workspace(input1, bchw, prm)


@_reg_fake("fn2b200::correlation_backward")
def _(input1, input2, grad_output, workspace, pad_size, kernel_size, max_displacement, stride1, stride2,
      corr_multiply=1, need1=True, need2=True):
    return (_f32(input1) if need1 else _nothing(input1)), (_f32(input2) if need2 else _nothing(input2))


@_reg_fake("fn2b200::correlation_backward_cat")
def _(input1, input2, grad_cat, cat, workspace, ch_offset, leaky_slope, pad_size, kernel_size, max_displacement, stride1,
      stride2, corr_multiply=1, need1=True, need2=True):
    return (_f32(input1) if need1 else _nothing(input1)), (_f32(input2) if need2 else _nothing(input2))


def _corr_setup(ctx, inputs, output):
    input1, input2 = inputs[:2]
    ctx.prm = inputs[2:]
    # the workspace (two bf16 copies of both inputs) has no gradient: no zero-filled stand-in is made for it, and it is
    # kept only when a backward can follow
    ctx.set_materialize_grads(False)
    ctx.save_for_backward(input1, input2, output[1] if any(ctx.needs_input_grad[:2]) else None)


def _corr_backward(ctx, grad_output, _grad_workspace):
    input1, input2, ws = ctx.saved_tensors
    need1, need2 = ctx.needs_input_grad[:2]
    if grad_output is None:
        return (None,) * (2 + len(ctx.prm))
    g1, g2 = fn2b200.correlation_backward(input1, input2, grad_output, ws, *ctx.prm, need1, need2)
    return (g1 if need1 else None, g2 if need2 else None) + (None,) * len(ctx.prm)


_reg_autograd("fn2b200::correlation_forward", _corr_backward, setup_context=_corr_setup)


def _corr_cat_setup(ctx, inputs, output):
    redir, input1, input2 = inputs[:3]
    ctx.prm, ctx.leaky_slope = inputs[3:9], inputs[9]
    ctx.nredir, ctx.redir_dtype = redir.shape[1], redir.dtype
    ctx.set_materialize_grads(False)
    # conv3_1 keeps the concat alive anyway; LeakyReLU's derivative is read from it
    ctx.save_for_backward(input1, input2, output[0], output[1] if any(ctx.needs_input_grad[1:3]) else None)


def _corr_cat_backward(ctx, grad_cat, _grad_workspace):
    input1, input2, cat, ws = ctx.saved_tensors
    need_r, need1, need2 = ctx.needs_input_grad[:3]
    if grad_cat is None:
        return (None,) * 10
    gr = grad_cat[:, :ctx.nredir].to(ctx.redir_dtype) if need_r else None
    g1 = g2 = None
    if need1 or need2:
        g1, g2 = fn2b200.correlation_backward_cat(input1, input2, grad_cat, cat, ws, ctx.nredir, ctx.leaky_slope,
                                                  *ctx.prm, need1, need2)
    return (gr, g1 if need1 else None, g2 if need2 else None) + (None,) * 7


_reg_autograd("fn2b200::correlation_forward_cat", _corr_cat_backward, setup_context=_corr_cat_setup)


# ---- Resample2d -------------------------------------------------------------------------------------------------------

@_reg_fake("fn2b200::resample2d_forward")
def _(input1, input2, kernel_size=1, bilinear=True):
    B, _, H, W = input2.shape
    return _f32(input2, (B, input1.shape[1], H, W))


@_reg_fake("fn2b200::resample2d_backward")
def _(input1, input2, grad_output, kernel_size=1, bilinear=True, need1=True, need2=True):
    return (_f32(input2, tuple(input1.shape)) if need1 else _nothing(input2)), (_f32(input2) if need2 else _nothing(input2))


def _resample_setup(ctx, inputs, output):
    ctx.save_for_backward(*inputs[:2])
    ctx.kernel_size, ctx.bilinear = inputs[2:4]


def _resample_backward(ctx, grad_output):
    input1, input2 = ctx.saved_tensors
    need1, need2 = ctx.needs_input_grad[:2]
    g1, g2 = fn2b200.resample2d_backward(input1, input2, grad_output, ctx.kernel_size, ctx.bilinear, need1, need2)
    return g1 if need1 else None, g2 if need2 else None, None, None


_reg_autograd("fn2b200::resample2d_forward", _resample_backward, setup_context=_resample_setup)


# ---- ChannelNorm ------------------------------------------------------------------------------------------------------

_DT16 = (torch.float16, torch.bfloat16)


@_reg_fake("fn2b200::channelnorm_forward")
def _(input1, norm_deg=2):
    B, _, H, W = input1.shape
    return input1.new_empty((B, 1, H, W), dtype=input1.dtype if input1.dtype in _DT16 else torch.float32)


@_reg_fake("fn2b200::channelnorm_backward")
def _(input1, output, grad_output, norm_deg=2):
    native = input1.dtype in _DT16 and output.dtype == input1.dtype and grad_output.dtype == input1.dtype
    return input1.new_empty(input1.shape, dtype=input1.dtype if native else torch.float32)


def _cnorm_setup(ctx, inputs, output):
    ctx.save_for_backward(inputs[0], output)
    ctx.norm_deg = inputs[1]


def _cnorm_backward(ctx, grad_output):
    input1, output = ctx.saved_tensors
    return fn2b200.channelnorm_backward(input1, output, grad_output, ctx.norm_deg), None


_reg_autograd("fn2b200::channelnorm_forward", _cnorm_backward, setup_context=_cnorm_setup)


# ---- warp -> diff -> channel-norm -> concat ---------------------------------------------------------------------------

@_reg_fake("fn2b200::warp_concat_forward")
def _(x, flow, C, upsample_mode, flow_mul, flow_div, cat_channels, ch_x, n_x, ch_warped, ch_flow, ch_flow_norm,
      ch_diff_norm):
    return _f32(x, (x.shape[0], cat_channels, x.shape[2], x.shape[3]))


@_reg_fake("fn2b200::warp_concat_backward")
def _(x, flow, grad_cat, C, upsample_mode, flow_mul, flow_div, ch_x, n_x, ch_warped, ch_flow, ch_flow_norm, ch_diff_norm,
      need_x=True, need_flow=True):
    gx = _f32(x, (x.shape[0], 2 * C, x.shape[2], x.shape[3])) if need_x else _nothing(x)
    return gx, (_f32(flow) if need_flow else _nothing(flow))


def _pad_channels(gx, channels):
    """gx [B, 2C, H, W] -> [B, channels, H, W]: odd trailing channels of x take no part in the op."""
    if channels > gx.size(1):
        gx = torch.cat((gx, gx.new_zeros(gx.size(0), channels - gx.size(1), gx.size(2), gx.size(3))), 1)
    return gx


def _warp_setup(ctx, inputs, output):
    ctx.save_for_backward(*inputs[:2])
    ctx.args = inputs[2:]          # C, upsample_mode, flow_mul, flow_div, cat_channels, then the ch_* layout


def _warp_backward(ctx, grad_cat):
    x, flow = ctx.saved_tensors
    need_x, need_flow = ctx.needs_input_grad[:2]
    C, mode, flow_mul, flow_div, _, *layout = ctx.args
    gx, gf = fn2b200.warp_concat_backward(x, flow, grad_cat, C, mode, flow_mul, flow_div, *layout, need_x, need_flow)
    return (_pad_channels(gx, x.size(1)) if need_x else None, gf if need_flow else None) + (None,) * len(ctx.args)


_reg_autograd("fn2b200::warp_concat_forward", _warp_backward, setup_context=_warp_setup)


@_reg_fake("fn2b200::fusion_concat")
def _(x, sd_flow2, s2_flow2, div_flow):
    return _f32(x, (x.shape[0], 11, x.shape[2], x.shape[3]))


@_reg_fake("fn2b200::fusion_concat_backward")
def _(x, sd_flow2, s2_flow2, grad_cat, div_flow, need_x=True, need_sd=True, need_s2=True):
    return ((_f32(x, (x.shape[0], 6, x.shape[2], x.shape[3])) if need_x else _nothing(x)),
            (_f32(sd_flow2) if need_sd else _nothing(x)), (_f32(s2_flow2) if need_s2 else _nothing(x)))


def _fusion_setup(ctx, inputs, output):
    ctx.save_for_backward(*inputs[:3])
    ctx.div_flow = inputs[3]


def _fusion_backward(ctx, grad_cat):
    x, sd_flow2, s2_flow2 = ctx.saved_tensors
    need_x, need_sd, need_s2 = ctx.needs_input_grad[:3]
    gx, g_sd, g_s2 = fn2b200.fusion_concat_backward(x, sd_flow2, s2_flow2, grad_cat, ctx.div_flow, need_x, need_sd,
                                                    need_s2)
    return (_pad_channels(gx, x.size(1)) if need_x else None, g_sd if need_sd else None, g_s2 if need_s2 else None,
            None)


_reg_autograd("fn2b200::fusion_concat", _fusion_backward, setup_context=_fusion_setup)
