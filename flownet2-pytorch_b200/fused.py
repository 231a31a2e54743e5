"""Opt-in fused forwards for the reference's FlowNetC / FlowNet2C / FlowNet2 (SURVEY 8f rows 1-3).

The drop-in modules (``Correlation``, ``Resample2d``, ``ChannelNorm``) keep the reference's module graph: each layer
reads and writes whole tensors, and ``models.py`` glues them with ``nn.Upsample``, a subtraction, a division and
``torch.cat``.  The functions here take an UNMODIFIED, already constructed reference network (its sub-modules, weights
and hyper-parameters are used as they are) and run the same data flow with the glue folded into our kernels:

* ``flownetc_forward``  -- FlowNetC.py:70-126: ``LeakyReLU(0.1)(corr(a, b))`` is written by the correlation kernel's
  epilogue straight into channels 32..472 of the 473-channel input of ``conv3_1`` (8f-2): no activation pass over the
  cost volume, no ``torch.cat`` copy of it.
* ``flownet2_forward``  -- models.py:120-185: every ``upsample -> Resample2d -> diff -> ChannelNorm -> cat`` group is
  ONE kernel (``functional.warp_concat_forward``, 8f-1) that reads the quarter-resolution flow directly (8f-3) and writes
  the concat buffer the next sub-network consumes.

``flownetc_forward``, ``flownet2c_forward``, ``flownet2_forward`` and ``fused_forward`` are inference only
(``torch.no_grad`` is entered there).  For training:

* ``CorrelationCat`` / ``CorrelationCatFunction`` -- ``torch.cat((redir, LeakyReLU(slope)(corr(a, b))), 1)`` as one
  differentiable op.  Forward = the redir copy + ``correlation_forward_cat``; backward = one
  ``correlation_backward_cat`` call that reads the correlation's gradient straight out of the concat gradient and takes
  LeakyReLU's derivative from the saved concat (conv3_1 keeps it alive anyway): no masked copy of the cost volume, no
  separate correlation output kept for backward.  Gradients are bit-identical to the unfused
  ``Correlation`` -> ``LeakyReLU`` -> ``torch.cat`` graph.
* ``train_forward(net, inputs)`` -- FlowNetC / FlowNet2C with autograd on, through ``CorrelationCat``; returns what
  ``net.forward`` returns in the net's current mode (flow2..flow6 in training).  FlowNet2 is not covered: its warp
  groups would need the x4 upsample's backward inside ``warp_concat_backward``.
* ``WarpConcat`` / ``WarpConcatFunction`` (full-resolution flow, fused forward AND fused backward).

Results agree with the unfused graph to rounding (tests/test_gpu_parity.py::test_fused_forwards_match_unfused_models,
tests/test_gpu_corr_cat.py).
"""
import torch
from torch.autograd import Function
from torch.autograd.function import once_differentiable

from . import functional as F2


class WarpConcatFunction(Function):
    """concat1 = cat(x, Resample2d()(x[:, 3:], flow), flow / div_flow, ChannelNorm()(x[:, :3] - warped)) as one
    differentiable op (models.py:133-138, :145-150); flow is the full-resolution flow (keep nn.Upsample in front of it
    when training: its backward is torch's).  forward and backward are one kernel each."""

    @staticmethod
    def forward(ctx, x, flow, div_flow=20.0):
        ctx.save_for_backward(x, flow)
        ctx.div_flow = float(div_flow)
        return F2.warp_concat_forward(x, flow, C=x.size(1) // 2, flow_div=ctx.div_flow)

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_cat):
        x, flow = ctx.saved_tensors
        gx, gf = F2.warp_concat_backward(x, flow, grad_cat, C=x.size(1) // 2, flow_div=ctx.div_flow)
        if x.size(1) > gx.size(1):           # odd trailing channels of x take no part
            gx = torch.cat((gx, gx.new_zeros(gx.size(0), x.size(1) - gx.size(1), gx.size(2), gx.size(3))), 1)
        return (gx if ctx.needs_input_grad[0] else None), (gf if ctx.needs_input_grad[1] else None), None


class WarpConcat(torch.nn.Module):
    """nn.Module form of WarpConcatFunction: WarpConcat(div_flow)(x, flow) -> the (3C + 3)-channel concat."""

    def __init__(self, div_flow=20.0):
        super(WarpConcat, self).__init__()
        self.div_flow = div_flow

    def forward(self, x, flow):
        return WarpConcatFunction.apply(x, flow, self.div_flow)


class CorrelationCatFunction(Function):
    """torch.cat((redir, LeakyReLU(leaky_slope)(Correlation(...)(input1, input2))), 1) -> fp32 [B, R + D, oH, oW]
    (FlowNetC.py:86-92 from `out_corr = self.corr(...)` to `in_conv3_1`)."""

    @staticmethod
    def forward(ctx, redir, input1, input2, pad_size, kernel_size, max_displacement, stride1, stride2, corr_multiply=1,
                leaky_slope=0.1):
        B, C, H, W = input1.shape
        D, oH, oW = F2.correlation_out_shape(C, H, W, pad_size, kernel_size, max_displacement, stride1, stride2)
        R = redir.size(1)
        if redir.dim() != 4 or (redir.size(0), redir.size(2), redir.size(3)) != (B, oH, oW):
            raise ValueError("CorrelationCat: redir %s does not match the correlation output [%d, D, %d, %d]"
                             % (tuple(redir.shape), B, oH, oW))
        cat = torch.empty((B, R + D, oH, oW), dtype=torch.float32, device=input1.device)
        cat[:, :R].copy_(redir)
        cat, ws = F2.correlation_forward_cat(input1, input2, cat, R, leaky_slope, pad_size, kernel_size, max_displacement,
                                             stride1, stride2, corr_multiply, return_workspace=True)
        ctx.prm = (pad_size, kernel_size, max_displacement, stride1, stride2, corr_multiply)
        ctx.leaky_slope, ctx.nredir, ctx.redir_dtype = float(leaky_slope), R, redir.dtype
        # the bf16 hi/lo copies of the inputs, for a single-launch backward; dropped with ctx (see CorrelationFunction)
        ctx.workspace = ws if (ctx.needs_input_grad[1] or ctx.needs_input_grad[2]) else None
        ctx.save_for_backward(input1, input2, cat)
        return cat

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_cat):
        input1, input2, cat = ctx.saved_tensors
        need_r, need1, need2 = ctx.needs_input_grad[:3]
        gr = grad_cat[:, :ctx.nredir].to(ctx.redir_dtype) if need_r else None
        g1 = g2 = None
        if need1 or need2:
            pad_size, kernel_size, max_displacement, stride1, stride2, corr_multiply = ctx.prm
            g1, g2 = F2.correlation_backward_cat(input1, input2, grad_cat, cat, ctx.nredir, ctx.leaky_slope, pad_size,
                                                 kernel_size, max_displacement, stride1, stride2, corr_multiply,
                                                 need1=need1, need2=need2, workspace=ctx.workspace)
        ctx.workspace = None
        if g1 is not None and g1.dtype != input1.dtype:
            g1 = g1.to(input1.dtype)
        if g2 is not None and g2.dtype != input2.dtype:
            g2 = g2.to(input2.dtype)
        return (gr, g1, g2) + (None,) * 7


class CorrelationCat(torch.nn.Module):
    """nn.Module form of CorrelationCatFunction: CorrelationCat(pad_size, kernel_size, max_displacement, stride1, stride2,
    corr_multiply, leaky_slope)(redir, input1, input2) -> the fp32 concat `redir | LeakyReLU(corr(input1, input2))`."""

    def __init__(self, pad_size, kernel_size, max_displacement, stride1, stride2, corr_multiply=1, leaky_slope=0.1):
        super(CorrelationCat, self).__init__()
        self.pad_size, self.kernel_size, self.max_displacement = pad_size, kernel_size, max_displacement
        self.stride1, self.stride2, self.corr_multiply, self.leaky_slope = stride1, stride2, corr_multiply, leaky_slope

    def forward(self, redir, input1, input2):
        return CorrelationCatFunction.apply(redir, input1, input2, self.pad_size, self.kernel_size, self.max_displacement,
                                            self.stride1, self.stride2, self.corr_multiply, self.leaky_slope)


def _corr_module(net_c):
    """FlowNetC.corr is the Correlation module itself, or nn.Sequential(tofp32, Correlation, tofp16) in --fp16 mode
    (FlowNetC.py:25-31)."""
    corr = net_c.corr
    if isinstance(corr, torch.nn.Sequential):
        corr = [m for m in corr if hasattr(m, "max_displacement")][0]
    return corr


def flownetc_forward(net_c, x):
    """networks/FlowNetC.py:70-126 in eval mode -> (flow2,).  x: [B,6,H,W]."""
    with torch.no_grad():
        return _flownetc_pair(net_c, x[:, 0:3], x[:, 3:])[:1]


def _flownetc_pair(net_c, x1, x2):
    """FlowNetC on the two frames given separately (FlowNet2C feeds x[:,:,0] and x[:,:,1], models.py:192-194)
    -> (flow2, flow3, flow4, flow5, flow6); differentiable when grad mode is on."""
    out_conv1a = net_c.conv1(x1)
    out_conv2a = net_c.conv2(out_conv1a)
    out_conv3a = net_c.conv3(out_conv2a)
    out_conv3b = net_c.conv3(net_c.conv2(net_c.conv1(x2)))
    out_conv_redir = net_c.conv_redir(out_conv3a)
    corr = _corr_module(net_c)
    in_conv3_1 = CorrelationCat(corr.pad_size, corr.kernel_size, corr.max_displacement, corr.stride1, corr.stride2,
                                corr.corr_multiply, net_c.corr_activation.negative_slope)(out_conv_redir, out_conv3a,
                                                                                          out_conv3b)
    out_conv3_1 = net_c.conv3_1(in_conv3_1.to(out_conv_redir.dtype))
    out_conv4 = net_c.conv4_1(net_c.conv4(out_conv3_1))
    out_conv5 = net_c.conv5_1(net_c.conv5(out_conv4))
    out_conv6 = net_c.conv6_1(net_c.conv6(out_conv5))
    flow6 = net_c.predict_flow6(out_conv6)
    concat5 = torch.cat((out_conv5, net_c.deconv5(out_conv6), net_c.upsampled_flow6_to_5(flow6)), 1)
    flow5 = net_c.predict_flow5(concat5)
    concat4 = torch.cat((out_conv4, net_c.deconv4(concat5), net_c.upsampled_flow5_to_4(flow5)), 1)
    flow4 = net_c.predict_flow4(concat4)
    concat3 = torch.cat((out_conv3_1, net_c.deconv3(concat4), net_c.upsampled_flow4_to_3(flow4)), 1)
    flow3 = net_c.predict_flow3(concat3)
    concat2 = torch.cat((out_conv2a, net_c.deconv2(concat3), net_c.upsampled_flow3_to_2(flow3)), 1)
    return net_c.predict_flow2(concat2), flow3, flow4, flow5, flow6


def _normalise(inputs, rgb_max):
    """models.py:121-126: subtract the per-sample, per-channel mean over both frames, divide by rgb_max."""
    rgb_mean = inputs.contiguous().view(inputs.size()[:2] + (-1,)).mean(dim=-1).view(inputs.size()[:2] + (1, 1, 1,))
    return (inputs - rgb_mean) / rgb_max


def flownet2c_forward(net, inputs):
    """models.FlowNet2C.forward (models.py:189-243) in eval mode: upsample1(flow2 * div_flow)."""
    with torch.no_grad():
        x = _normalise(inputs, net.rgb_max)
        flow2 = _flownetc_pair(net, x[:, :, 0], x[:, :, 1])[0]
        return net.upsample1(flow2 * net.div_flow)


def flownet2_forward(net, inputs):
    """models.FlowNet2.forward (models.py:120-185) with the warp groups fused.  net: the reference's FlowNet2."""
    with torch.no_grad():
        div = float(net.div_flow)
        x = _normalise(inputs, net.rgb_max)
        x = torch.cat((x[:, :, 0], x[:, :, 1]), dim=1).float()
        B, _, H, W = x.shape
        # flownetc -> concat1 = (x | img1 warped | flow / div_flow | |img0 - warped|)            models.py:129-138
        flow2 = flownetc_forward(net.flownetc, x)[0]
        concat1 = F2.warp_concat_forward(x, flow2, upsample="bilinear", flow_mul=div, flow_div=div)
        # flownets1 -> concat2                                                                    models.py:141-150
        flow2 = net.flownets_1(concat1)[0]
        concat2 = F2.warp_concat_forward(x, flow2, upsample="bilinear", flow_mul=div, flow_div=div)
        del concat1
        # flownets2 and flownetsd -> concat3 = (img0 | sd flow | s2 flow | their norms | the two diff norms)   :153-174
        s2_flow2 = net.flownets_2(concat2)[0]
        del concat2
        sd_flow2 = net.flownets_d(x)[0]
        concat3 = torch.empty((B, 11, H, W), dtype=torch.float32, device=x.device)
        F2.warp_concat_forward(x, sd_flow2, upsample="nearest", flow_mul=1.0 / div, flow_div=1.0, out=concat3, ch_x=0, n_x=3,
                               ch_warped=-1, ch_flow=3, ch_flow_norm=7, ch_diff_norm=9)
        F2.warp_concat_forward(x, s2_flow2, upsample="nearest", flow_mul=div, flow_div=1.0, out=concat3, ch_x=-1, n_x=0,
                               ch_warped=-1, ch_flow=5, ch_flow_norm=8, ch_diff_norm=10)
        return net.flownetfusion(concat3)


def fused_forward(net, inputs):
    """Dispatch on the reference class name: FlowNet2, FlowNet2C or a bare FlowNetC."""
    name = type(net).__name__
    if name == "FlowNet2":
        return flownet2_forward(net, inputs)
    if name == "FlowNet2C":
        return flownet2c_forward(net, inputs)
    if name == "FlowNetC":
        return flownetc_forward(net, inputs)
    raise TypeError("fused_forward: no fused data flow for %s (FlowNet2, FlowNet2C, FlowNetC)" % name)


def train_forward(net, inputs):
    """net.forward with autograd, with the correlation -> LeakyReLU -> concat of FlowNetC fused (CorrelationCat).
    net: the reference's FlowNetC (inputs [B,6,H,W]) or FlowNet2C (inputs [B,3,2,H,W]).  Returns what net.forward
    returns in the net's current mode: (flow2, flow3, flow4, flow5, flow6) when net.training (FlowNetC.py:125-128,
    models.py:250-253), else FlowNetC's (flow2,) / FlowNet2C's upsample1(flow2 * div_flow)."""
    name = type(net).__name__
    if name == "FlowNet2":
        raise TypeError("train_forward: FlowNet2 has no differentiable fused data flow (its warp groups read the x4 "
                        "upsampled flow, whose backward warp_concat_backward does not include); train it on the drop-in "
                        "modules")
    if name == "FlowNet2C":
        x = _normalise(inputs, net.rgb_max)
        flows = _flownetc_pair(net, x[:, :, 0], x[:, :, 1])
        return flows if net.training else net.upsample1(flows[0] * net.div_flow)
    if name == "FlowNetC":
        flows = _flownetc_pair(net, inputs[:, 0:3], inputs[:, 3:])
        return flows if net.training else flows[:1]
    raise TypeError("train_forward: no fused data flow for %s (FlowNet2C, FlowNetC)" % name)
