"""Opt-in fused forwards for the reference's FlowNetC / FlowNet2C / FlowNet2CS / FlowNet2CSS / FlowNet2 (SURVEY 8f
rows 1-3).

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
* ``fused_forward`` on a FlowNet2CS / FlowNet2CSS -- models.py:392-416 / :469-505: the first one / two stages of the
  same data flow (``_stacked_flow2``, shared with FlowNet2), then the network's own output ``nn.Upsample``.

``flownetc_forward``, ``flownet2c_forward``, ``flownet2_forward`` and ``fused_forward`` are inference only
(``torch.no_grad`` is entered there).  For training:

* ``CorrelationCat`` / ``CorrelationCatFunction`` -- ``torch.cat((redir, LeakyReLU(slope)(corr(a, b))), 1)`` as one
  differentiable op.  Forward = the redir copy + ``correlation_forward_cat``; backward = one
  ``correlation_backward_cat`` call that reads the correlation's gradient straight out of the concat gradient and takes
  LeakyReLU's derivative from the saved concat (conv3_1 keeps it alive anyway): no masked copy of the cost volume, no
  separate correlation output kept for backward.  Gradients are bit-identical to the unfused
  ``Correlation`` -> ``LeakyReLU`` -> ``torch.cat`` graph.
* ``train_forward(net, inputs)`` -- FlowNetC / FlowNet2C / FlowNet2CS / FlowNet2CSS with autograd on, through
  ``CorrelationCat`` (and for CS / CSS ``WarpConcat(upsample="bilinear")`` for concat1 / concat2); returns what
  ``net.forward`` returns in the net's current mode (flow2..flow6 for FlowNetC / FlowNet2C in training, CS / CSS's
  full-resolution flow in either mode).  ``fused_forward`` on a CS / CSS is this function under ``torch.no_grad``.
  FlowNet2 has its own entry point:
* ``flownet2_train_forward(net, inputs)`` -- FlowNet2 with autograd on: ``CorrelationCat`` in the FlowNetC stage,
  ``WarpConcat(upsample="bilinear")`` for concat1 / concat2 and ``FusionConcat`` for concat3.  ``flownet2_forward`` is
  this function under ``torch.no_grad``, so inference and training share one data flow.
* ``WarpConcat`` / ``WarpConcatFunction`` -- ``upsample -> Resample2d -> diff -> ChannelNorm -> cat`` with a fused
  forward AND a fused backward.  With ``upsample`` the op takes the quarter-resolution flow2 and its backward returns
  that flow's gradient directly: the x4 upsample's adjoint runs inside the backward kernel, deterministically (torch's
  own upsample backward uses atomics), and the full-resolution flow gradient is never written.  The image gradient is
  only computed when x requires one -- in FlowNet2, x is the normalised input and does not.
* ``FusionConcat`` / ``FusionConcatFunction`` -- the 11-channel concat3 of the fusion stage from x and the
  quarter-resolution FlowNetSD / FlowNetS2 flows, same scheme (nearest upsample).

Each of these ops is one ``torch.ops.fn2b200`` operator with a fake kernel and an autograd formula (``ops``): the
training and inference forwards trace under torch.compile without a graph break and capture into CUDA graphs.

Results agree with the unfused graph to rounding (tests/test_gpu_parity.py::test_fused_forwards_match_unfused_models,
tests/test_gpu_corr_cat.py).
"""
import torch

from . import functional as F2
from .ops import fn2b200


def warp_concat(x, flow, div_flow=20.0, upsample=None):
    """torch.ops.fn2b200.warp_concat_forward with models.py:138's concat1 layout (differentiable): x [B, 2C, H, W] ->
    cat(x, Resample2d()(x[:, C:], flow_up), flow_up / div_flow, ChannelNorm()(x[:, :C] - warped)), 3C + 3 channels."""
    F2._require_cuda(x, flow)
    C = x.size(1) // 2
    div = float(div_flow)
    return fn2b200.warp_concat_forward(x, flow, C, F2.UPSAMPLE_MODES[upsample], div, div, 3 * C + 3, 0, 2 * C, 2 * C, 3 * C,
                                       -1, 3 * C + 2)


class WarpConcatFunction(object):
    """concat1 = cat(x, Resample2d()(x[:, 3:], flow_up), flow_up / div_flow, ChannelNorm()(x[:, :3] - warped)) as one
    differentiable op (models.py:133-138, :145-150).  upsample=None: flow is the full-resolution flow_up.
    upsample="bilinear" / "nearest": flow is the quarter-resolution flow2 and flow_up = nn.Upsample(scale_factor=4,
    mode=upsample)(flow2 * div_flow) (models.py:130, :142) -- folded into the kernels, so the full-resolution flow and
    its gradient are never materialised.  forward is one kernel; backward one kernel plus the passes that finish the
    gradients asked for (only those in ctx.needs_input_grad are computed).  ``apply(x, flow, div_flow, upsample)`` is
    ``warp_concat``."""
    apply = staticmethod(warp_concat)


class WarpConcat(torch.nn.Module):
    """nn.Module form of warp_concat: WarpConcat(div_flow, upsample)(x, flow) -> the (3C + 3)-channel concat."""

    def __init__(self, div_flow=20.0, upsample=None):
        super(WarpConcat, self).__init__()
        self.div_flow, self.upsample = div_flow, upsample

    def forward(self, x, flow):
        return warp_concat(x, flow, self.div_flow, self.upsample)


def fusion_concat(x, sd_flow2, s2_flow2, div_flow=20.0):
    """torch.ops.fn2b200.fusion_concat (differentiable): concat3 of models.py:153-179, (x [B,6,H,W], sd_flow2, s2_flow2
    [B,2,H/4,W/4]) -> [B,11,H,W] = (img0 | sd flow | s2 flow | their norms | the two diff norms), each flow the nearest
    x4 upsample of its quarter-resolution flow2.  forward = two warp-concat kernels into one buffer; backward = two
    warp-concat backward passes, each reading its own channels of the concat gradient, the x gradients summed."""
    F2._require_cuda(x, sd_flow2, s2_flow2)
    return fn2b200.fusion_concat(x, sd_flow2, s2_flow2, float(div_flow))


class FusionConcatFunction(object):
    """concat3 of models.py:153-179 as one differentiable op: ``apply(x, sd_flow2, s2_flow2, div_flow)`` is
    ``fusion_concat``."""
    apply = staticmethod(fusion_concat)


class FusionConcat(torch.nn.Module):
    """nn.Module form of fusion_concat: FusionConcat(div_flow)(x, sd_flow2, s2_flow2) -> the 11-channel concat3."""

    def __init__(self, div_flow=20.0):
        super(FusionConcat, self).__init__()
        self.div_flow = div_flow

    def forward(self, x, sd_flow2, s2_flow2):
        return fusion_concat(x, sd_flow2, s2_flow2, self.div_flow)


def correlation_cat(redir, input1, input2, pad_size, kernel_size, max_displacement, stride1, stride2, corr_multiply=1,
                    leaky_slope=0.1):
    """torch.ops.fn2b200.correlation_forward_cat (differentiable): torch.cat((redir, LeakyReLU(leaky_slope)(
    Correlation(...)(input1, input2))), 1) -> fp32 [B, R + D, oH, oW] (FlowNetC.py:86-92 from `out_corr = self.corr(...)`
    to `in_conv3_1`).  The backward is one correlation_backward_cat launch on the tensor-core path: it reads the
    correlation's gradient straight out of the concat gradient and LeakyReLU's derivative from the saved concat."""
    F2._require_cuda(redir, input1, input2)
    return fn2b200.correlation_forward_cat(redir, input1, input2, pad_size, kernel_size, max_displacement, stride1,
                                           stride2, corr_multiply, float(leaky_slope))[0]


class CorrelationCatFunction(object):
    """torch.cat((redir, LeakyReLU(leaky_slope)(Correlation(...)(input1, input2))), 1) as one differentiable op:
    ``apply(redir, input1, input2, pad_size, kernel_size, max_displacement, stride1, stride2, corr_multiply,
    leaky_slope)`` is ``correlation_cat``."""
    apply = staticmethod(correlation_cat)


class CorrelationCat(torch.nn.Module):
    """nn.Module form of correlation_cat: CorrelationCat(pad_size, kernel_size, max_displacement, stride1, stride2,
    corr_multiply, leaky_slope)(redir, input1, input2) -> the fp32 concat `redir | LeakyReLU(corr(input1, input2))`."""

    def __init__(self, pad_size, kernel_size, max_displacement, stride1, stride2, corr_multiply=1, leaky_slope=0.1):
        super(CorrelationCat, self).__init__()
        self.pad_size, self.kernel_size, self.max_displacement = pad_size, kernel_size, max_displacement
        self.stride1, self.stride2, self.corr_multiply, self.leaky_slope = stride1, stride2, corr_multiply, leaky_slope

    def forward(self, redir, input1, input2):
        return correlation_cat(redir, input1, input2, self.pad_size, self.kernel_size, self.max_displacement, self.stride1,
                               self.stride2, self.corr_multiply, self.leaky_slope)


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
    in_conv3_1 = correlation_cat(out_conv_redir, out_conv3a, out_conv3b, corr.pad_size, corr.kernel_size,
                                 corr.max_displacement, corr.stride1, corr.stride2, corr.corr_multiply,
                                 net_c.corr_activation.negative_slope)
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


def _stacked_flow2(net, inputs, n_s):
    """The C -> S1 -> S2 branch FlowNet2, FlowNet2CS and FlowNet2CSS share (models.py:120-150, :392-413, :469-502),
    differentiable when grad mode is on: FlowNetC through CorrelationCat, then the n_s FlowNetS stages
    net.flownets_1 .. net.flownets_<n_s>, each fed by concat = (x | img1 warped | flow / div_flow | |img0 - warped|) of
    the previous stage's flow through WarpConcat(upsample="bilinear").  Returns (x, the last stage's quarter-resolution
    flow2)."""
    div = float(net.div_flow)
    x = _normalise(inputs, net.rgb_max)
    x = torch.cat((x[:, :, 0], x[:, :, 1]), dim=1).float()
    flow2 = _flownetc_pair(net.flownetc, x[:, 0:3], x[:, 3:])[0]
    for i in range(1, n_s + 1):
        concat = warp_concat(x, flow2, div, upsample="bilinear")
        flow2 = getattr(net, "flownets_%d" % i)(concat)[0]
        del concat
    return x, flow2


def flownet2_train_forward(net, inputs):
    """models.FlowNet2.forward (models.py:120-185) with the warp groups fused, differentiable when grad mode is on.
    net: the reference's FlowNet2; inputs [B,3,2,H,W].  Returns what net.forward returns (flownetfusion's flow).
    The FlowNetC stage runs through CorrelationCat, concat1 / concat2 through WarpConcat(upsample="bilinear") and
    concat3 through FusionConcat: neither the x4 upsampled flows nor their gradients are materialised."""
    x, s2_flow2 = _stacked_flow2(net, inputs, 2)
    # flownetsd -> concat3 = (img0 | sd flow | s2 flow | their norms | the two diff norms)         models.py:153-179
    sd_flow2 = net.flownets_d(x)[0]
    return net.flownetfusion(fusion_concat(x, sd_flow2, s2_flow2, float(net.div_flow)))


def flownet2_forward(net, inputs):
    """models.FlowNet2.forward (models.py:120-185) with the warp groups fused, for inference: flownet2_train_forward
    under torch.no_grad.  net: the reference's FlowNet2."""
    with torch.no_grad():
        return flownet2_train_forward(net, inputs)


def fused_forward(net, inputs):
    """Dispatch on the reference class name: FlowNet2, FlowNet2CSS, FlowNet2CS, FlowNet2C or a bare FlowNetC
    (inference, torch.no_grad)."""
    name = type(net).__name__
    if name == "FlowNet2":
        return flownet2_forward(net, inputs)
    if name in ("FlowNet2CS", "FlowNet2CSS"):
        with torch.no_grad():
            return train_forward(net, inputs)
    if name == "FlowNet2C":
        return flownet2c_forward(net, inputs)
    if name == "FlowNetC":
        return flownetc_forward(net, inputs)
    raise TypeError("fused_forward: no fused data flow for %s (FlowNet2, FlowNet2CSS, FlowNet2CS, FlowNet2C, FlowNetC)"
                    % name)


def train_forward(net, inputs):
    """net.forward with autograd, with the correlation -> LeakyReLU -> concat of FlowNetC fused (CorrelationCat).
    net: the reference's FlowNetC (inputs [B,6,H,W]), FlowNet2C, FlowNet2CS or FlowNet2CSS (inputs [B,3,2,H,W]).
    Returns what net.forward returns in the net's current mode: (flow2, flow3, flow4, flow5, flow6) when net.training
    (FlowNetC.py:125-128, models.py:250-253), else FlowNetC's (flow2,) / FlowNet2C's upsample1(flow2 * div_flow).
    FlowNet2CS / FlowNet2CSS return their full-resolution flow in either mode (models.py:414-416, :503-505): the last
    FlowNetS stage's flow2 from _stacked_flow2, times div_flow, through the network's own upsample2 / upsample3."""
    name = type(net).__name__
    if name == "FlowNet2":
        raise TypeError("train_forward: FlowNet2 has no differentiable fused data flow here (train_forward covers "
                        "FlowNetC, FlowNet2C, FlowNet2CS and FlowNet2CSS); use "
                        "fused.flownet2_train_forward(net, inputs)")
    if name == "FlowNet2CS":
        return net.upsample2(_stacked_flow2(net, inputs, 1)[1] * net.div_flow)
    if name == "FlowNet2CSS":
        return net.upsample3(_stacked_flow2(net, inputs, 2)[1] * net.div_flow)
    if name == "FlowNet2C":
        x = _normalise(inputs, net.rgb_max)
        flows = _flownetc_pair(net, x[:, :, 0], x[:, :, 1])
        return flows if net.training else net.upsample1(flows[0] * net.div_flow)
    if name == "FlowNetC":
        flows = _flownetc_pair(net, inputs[:, 0:3], inputs[:, 3:])
        return flows if net.training else flows[:1]
    raise TypeError("train_forward: no fused data flow for %s (FlowNet2CSS, FlowNet2CS, FlowNet2C, FlowNetC)" % name)
