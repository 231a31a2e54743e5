"""GPU tests of the warp-concat backward through the x4 flow upsample (fn2b200_warp_concat_backward_up,
functional.warp_concat_backward(upsample=...), fused.WarpConcat(upsample=...), fused.FusionConcat,
fused.flownet2_train_forward).

The flow gradient is the quarter-resolution flow's: the upsample's adjoint runs inside the backward, in a fixed order,
so it must be bit-identical from run to run and whether or not the image gradient is computed.
"""
import ctypes
from types import SimpleNamespace

import numpy as np
import pytest
import torch
import torch.nn as nn

import upsample_ref as ur
from oracle import cpu as orc
from oracle import ref as oref
from test_gpu_corr_cat import FlowNetC, _conv, _deconv, _deterministic
from util import assert_close, rel_err

pytestmark = pytest.mark.gpu
TOL = 1e-4
NAMES = {1: "bilinear", 2: "nearest"}
# (what, forward layout, flow_mul): concat1 / concat2 (models.py:130-138) and the two halves of concat3 (:153-179)
LAYOUTS = [
    ("concat1", dict(flow_div=20.0), 20.0),
    ("concat3_sd", dict(flow_div=1.0, cat_channels=11, ch_x=0, n_x=3, ch_warped=-1, ch_flow=3, ch_flow_norm=7,
                        ch_diff_norm=9), 1.0 / 20.0),
    ("concat3_s2", dict(flow_div=1.0, cat_channels=11, ch_x=-1, n_x=0, ch_warped=-1, ch_flow=5, ch_flow_norm=8,
                        ch_diff_norm=10), 20.0),
]


def _f2():
    import flownet2_b200
    return flownet2_b200


def _bwd_layout(layout):
    return {k: v for k, v in layout.items() if k != "cat_channels"}


# (B, fh, fw, flow sigma in full-resolution pixels, strided x)
CASES = [
    (2, 10, 18, 3.0, False),       # H, W = 40, 72: neither a multiple of the 16 x 32 tile
    (1, 1, 5, 3.0, False),         # fh = 1: every bilinear tap clamps to row 0
    (2, 6, 1, 3.0, False),         # fw = 1
    (1, 12, 20, 64.0, False),      # sigma = 64 px: most taps clamp to the border
    (2, 8, 16, 3.0, True),         # x a channel slice of a wider tensor
]


@pytest.mark.parametrize("mode", [1, 2])
@pytest.mark.parametrize("case", CASES, ids=["ragged", "fh1", "fw1", "sigma64", "strided"])
@pytest.mark.parametrize("what,layout,mul", LAYOUTS, ids=[l[0] for l in LAYOUTS])
def test_backward_up_vs_oracle(mode, case, what, layout, mul):
    F2 = _f2().functional
    B, fh, fw, sigma, strided = case
    H, W = 4 * fh, 4 * fw
    g = torch.Generator().manual_seed(fh * 31 + fw + mode)
    if strided:
        big = torch.rand(B, 9, H, W, generator=g) - 0.5
        xd = big.cuda()[:, 2:8]
        assert not xd.is_contiguous()
        x = big[:, 2:8].contiguous()
    else:
        x = torch.rand(B, 6, H, W, generator=g) - 0.5
        xd = x.cuda()
    lr = torch.randn(B, 2, fh, fw, generator=g) * (sigma / abs(mul))
    cat = orc.warp_concat_forward(x.numpy(), lr.numpy(), upsample_mode=mode, flow_mul=mul, **layout)
    gc = torch.randn(cat.shape, generator=g)
    got = F2.warp_concat_forward(xd, lr.cuda(), upsample=NAMES[mode], flow_mul=mul,
                                 out=torch.zeros(cat.shape, device="cuda") if "cat_channels" in layout else None,
                                 **_bwd_layout(layout))
    assert_close(got.cpu().numpy(), cat, TOL, "%s forward" % what)
    gx, gf = F2.warp_concat_backward(xd, lr.cuda(), gc.cuda(), upsample=NAMES[mode], flow_mul=mul, **_bwd_layout(layout))
    rx, rf = ur.warp_concat_backward(x.numpy(), lr.numpy(), gc.numpy(), upsample_mode=mode, flow_mul=mul,
                                     **_bwd_layout(layout))
    assert gf.shape == (B, 2, fh, fw)
    assert_close(gx.cpu().numpy(), rx, TOL, "%s mode %d grad_x" % (what, mode))
    assert_close(gf.cpu().numpy(), rf, TOL, "%s mode %d grad_flow" % (what, mode))


def _unfused_group(R, x, lr, div, mode):
    """models.py:130-138 on the drop-in modules: nn.Upsample, Resample2d, subtraction, ChannelNorm, torch.cat."""
    up = nn.Upsample(scale_factor=4, mode=NAMES[mode])(lr * div)
    warped = R.Resample2d()(x[:, 3:], up)
    return torch.cat((x, warped, up / div, R.ChannelNorm()(x[:, :3] - warped)), 1)


def _unfused_concat3(R, x, sd_flow2, s2_flow2, div):
    """models.py:153-179 on the drop-in modules."""
    s2 = nn.Upsample(scale_factor=4, mode="nearest")(s2_flow2 * div)
    d_s2 = R.ChannelNorm()(x[:, :3] - R.Resample2d()(x[:, 3:], s2))
    sd = nn.Upsample(scale_factor=4, mode="nearest")(sd_flow2 / div)
    d_sd = R.ChannelNorm()(x[:, :3] - R.Resample2d()(x[:, 3:], sd))
    return torch.cat((x[:, :3], sd, s2, R.ChannelNorm()(sd), R.ChannelNorm()(s2), d_sd, d_s2), 1)


def _leaves(seed, B, fh, fw, grads, nflows=1, sigma=0.2):
    g = torch.Generator().manual_seed(seed)
    x = (torch.rand(B, 6, 4 * fh, 4 * fw, generator=g) - 0.5).cuda()
    flows = [(torch.randn(B, 2, fh, fw, generator=g) * sigma).cuda() for _ in range(nflows)]
    return [t.requires_grad_(r) for t, r in zip([x] + flows, grads)]


@pytest.mark.parametrize("mode", [1, 2])
@pytest.mark.parametrize("grads", [(True, True), (False, True), (True, False)], ids=["both", "flow_only", "x_only"])
def test_warp_concat_module_matches_unfused_graph(mode, grads):
    f = _f2()
    ours, ref = _leaves(40 + mode, 2, 10, 18, grads), _leaves(40 + mode, 2, 10, 18, grads)
    n0 = f.functional.launch_count()
    out = f.fused.WarpConcat(20.0, upsample=NAMES[mode])(*ours)
    n1 = f.functional.launch_count()
    base = _unfused_group(f, *ref, 20.0, mode)
    assert out.shape == base.shape == (2, 12, 40, 72)
    assert rel_err(out.detach().cpu().numpy(), base.detach().cpu().numpy()) < 1e-6
    g = torch.randn(out.shape, generator=torch.Generator().manual_seed(43)).cuda()
    n2 = f.functional.launch_count()
    out.backward(g)
    n3 = f.functional.launch_count()
    base.backward(g)
    for t, r, what in zip(ours, ref, ("x", "flow2")):
        assert (t.grad is None) == (r.grad is None) == (not t.requires_grad)
        if t.grad is not None:
            assert_close(t.grad.cpu().numpy(), r.grad.cpu().numpy(), 1e-5, "WarpConcat(%s) grad %s" % (NAMES[mode], what))
    # launches: the forward is one kernel; the backward one kernel, + the bilinear partials' sum, + the scatter transpose
    assert n1 - n0 == 1
    assert n3 - n2 == 1 + (mode == 1 and grads[1]) + grads[0]


# requires_grad of (x, sd_flow2, s2_flow2) -> backward launches: one kernel per flow half that has a gradient to give,
# plus the scatter transpose of each half when x needs a gradient
FUSION_GRADS = [((True, True, True), 4), ((False, True, True), 2), ((False, False, True), 1), ((True, True, False), 4)]


@pytest.mark.parametrize("grads,bwd_launches", FUSION_GRADS, ids=["all", "x_frozen", "sd_frozen", "s2_frozen"])
def test_fusion_concat_matches_unfused_graph(grads, bwd_launches):
    f = _f2()
    ours, ref = _leaves(50, 2, 10, 18, grads, 2, 1.0), _leaves(50, 2, 10, 18, grads, 2, 1.0)
    n0 = f.functional.launch_count()
    out = f.fused.FusionConcat(20.0)(*ours)
    n1 = f.functional.launch_count()
    base = _unfused_concat3(f, *ref, 20.0)
    assert out.shape == base.shape == (2, 11, 40, 72)
    assert rel_err(out.detach().cpu().numpy(), base.detach().cpu().numpy()) < 1e-6
    g = torch.randn(out.shape, generator=torch.Generator().manual_seed(51)).cuda()
    n2 = f.functional.launch_count()
    out.backward(g)
    n3 = f.functional.launch_count()
    base.backward(g)
    for t, r, what in zip(ours, ref, ("x", "sd_flow2", "s2_flow2")):
        assert (t.grad is None) == (r.grad is None) == (not t.requires_grad)
        if t.grad is not None:
            assert_close(t.grad.cpu().numpy(), r.grad.cpu().numpy(), 1e-5, "FusionConcat grad %s" % what)
    assert (n1 - n0, n3 - n2) == (2, bwd_launches)


@pytest.mark.parametrize("mode", [0, 1, 2])
def test_flow_gradient_is_deterministic_and_independent_of_grad_x(mode):
    """Bit-identical flow gradient over two runs and with or without the image gradient; sigma = 8 px flows make many
    pixels of a tile feed the same cells."""
    F2 = _f2().functional
    g = torch.Generator(device="cuda").manual_seed(60 + mode)
    fh, fw = (112, 256) if mode else (448, 1024)
    x = torch.rand(2, 6, 448, 1024, device="cuda", generator=g) - 0.5
    fl = torch.randn(2, 2, fh, fw, device="cuda", generator=g) * (0.4 if mode else 8.0)
    gc = torch.randn(2, 12, 448, 1024, device="cuda", generator=g)
    kw = dict(flow_div=20.0, upsample=NAMES.get(mode), flow_mul=20.0)
    gx1, gf1 = F2.warp_concat_backward(x, fl, gc, **kw)
    gx2, gf2 = F2.warp_concat_backward(x, fl, gc, **kw)
    none, gf3 = F2.warp_concat_backward(x, fl, gc, need_x=False, **kw)
    gx4, none2 = F2.warp_concat_backward(x, fl, gc, need_flow=False, **kw)
    assert none is None and none2 is None
    assert torch.equal(gf1, gf2) and torch.equal(gf1, gf3)
    # the img1 half of the image gradient comes from a scatter with atomics: equal to rounding only
    assert torch.equal(gx1[:, :3], gx4[:, :3])
    assert_close(gx4.cpu().numpy(), gx1.cpu().numpy(), 1e-5, "grad_x without grad_flow")


def test_mode0_through_up_equals_plain_entry_point():
    f = _f2()
    F2, L = f.functional, f._lib.LIB
    g = torch.Generator(device="cuda").manual_seed(70)
    x = torch.rand(2, 6, 40, 72, device="cuda", generator=g) - 0.5
    fl = torch.randn(2, 2, 40, 72, device="cuda", generator=g) * 4
    gc = torch.randn(2, 12, 40, 72, device="cuda", generator=g)
    gx_up, gf_up = F2.warp_concat_backward(x, fl, gc, flow_div=20.0)
    gx, gf = torch.empty_like(gx_up), torch.empty_like(gf_up)
    ws_bytes = int(L.fn2b200_warp_concat_backward_workspace(2, 3, 40, 72))
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device="cuda")
    P = lambda t: ctypes.c_void_p(t.data_ptr())
    st = (ctypes.c_int64 * 4)(*x.stride())
    n0 = F2.launch_count()
    f._lib.check(L.fn2b200_warp_concat_backward(P(x), st, 3, P(fl), P(gc), 12, 0, 6, 6, 9, 20.0, -1, 11, P(gx), P(gf), P(ws),
                                                ws_bytes, 2, 40, 72, ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)),
                 "warp_concat_backward")
    assert F2.launch_count() - n0 == 2
    torch.cuda.synchronize()
    assert torch.equal(gf, gf_up)
    assert_close(gx.cpu().numpy(), gx_up.cpu().numpy(), 1e-6, "plain vs _up grad_x")


def test_full_size():
    """x [8,6,448,1024], flow2 [8,2,112,256]: one sample against the oracle, the whole tensor against the unfused graph."""
    f = _f2()
    g = torch.Generator(device="cuda").manual_seed(80)
    x = torch.rand(8, 6, 448, 1024, device="cuda", generator=g) - 0.5
    lr = torch.randn(8, 2, 112, 256, device="cuda", generator=g) * 0.3
    gc = torch.randn(8, 12, 448, 1024, device="cuda", generator=g)
    gx, gf = f.functional.warp_concat_backward(x, lr, gc, flow_div=20.0, upsample="bilinear", flow_mul=20.0)
    n = 5
    rx, rf = ur.warp_concat_backward(x[n:n + 1].cpu().numpy(), lr[n:n + 1].cpu().numpy(), gc[n:n + 1].cpu().numpy(),
                                     upsample_mode=1, flow_mul=20.0, flow_div=20.0)
    assert_close(gx[n:n + 1].cpu().numpy(), rx, TOL, "full size grad_x")
    assert_close(gf[n:n + 1].cpu().numpy(), rf, TOL, "full size grad_flow")
    xs, ls = x.clone().requires_grad_(), lr.clone().requires_grad_()
    _unfused_group(f, xs, ls, 20.0, 1).backward(gc)
    assert_close(gx.cpu().numpy(), xs.grad.cpu().numpy(), 1e-5, "full size grad_x vs unfused")
    assert_close(gf.cpu().numpy(), ls.grad.cpu().numpy(), 1e-5, "full size grad_flow vs unfused")


# ------------------------------------------------------------------------------------------------
# flownet2_train_forward on a FlowNet2-shaped network
# ------------------------------------------------------------------------------------------------
class FlowNetS(nn.Module):
    """A small stand-in for FlowNetS / FlowNetSD: flow2 at a quarter of the input resolution; (flow2, flow3) in
    training, (flow2,) otherwise, as the reference's sub-networks return."""

    def __init__(self, cin):
        super(FlowNetS, self).__init__()
        self.conv1, self.conv2, self.conv3 = _conv(cin, 16, 3, 2), _conv(16, 32, 3, 2), _conv(32, 32, 3, 2)
        self.deconv2 = _deconv(32, 16)
        self.predict_flow3, self.predict_flow2 = nn.Conv2d(32, 2, 3, 1, 1), nn.Conv2d(50, 2, 3, 1, 1)
        self.upsampled_flow3_to_2 = nn.ConvTranspose2d(2, 2, 4, 2, 1)

    def forward(self, x):
        out_conv2 = self.conv2(self.conv1(x))
        out_conv3 = self.conv3(out_conv2)
        flow3 = self.predict_flow3(out_conv3)
        flow2 = self.predict_flow2(torch.cat((out_conv2, self.deconv2(out_conv3), self.upsampled_flow3_to_2(flow3)), 1))
        return (flow2, flow3) if self.training else (flow2,)


class FlowNetFusion(nn.Module):
    """A small stand-in for FlowNetFusion: the 11-channel concat3 in, a full-resolution flow out."""

    def __init__(self):
        super(FlowNetFusion, self).__init__()
        self.conv0, self.conv1 = _conv(11, 16), _conv(16, 32, 3, 2)
        self.deconv0 = _deconv(32, 16)
        self.predict_flow0 = nn.Conv2d(32, 2, 3, 1, 1)

    def forward(self, x):
        out_conv0 = self.conv0(x)
        return self.predict_flow0(torch.cat((out_conv0, self.deconv0(self.conv1(out_conv0))), 1))


class FlowNet2(nn.Module):
    """FlowNet2's structure and attribute names on small sub-networks; forward = models.py:120-185 on the drop-in
    Resample2d / ChannelNorm modules."""

    def __init__(self, div_flow=20.0, rgb_max=255.0):
        super(FlowNet2, self).__init__()
        import flownet2_b200 as f
        self.div_flow, self.rgb_max = div_flow, rgb_max
        self.channelnorm = f.ChannelNorm()
        self.flownetc = FlowNetC()
        self.upsample1 = nn.Upsample(scale_factor=4, mode="bilinear")
        self.resample1 = f.Resample2d()
        self.flownets_1 = FlowNetS(12)
        self.upsample2 = nn.Upsample(scale_factor=4, mode="bilinear")
        self.resample2 = f.Resample2d()
        self.flownets_2 = FlowNetS(12)
        self.flownets_d = FlowNetS(6)
        self.upsample3 = nn.Upsample(scale_factor=4, mode="nearest")
        self.upsample4 = nn.Upsample(scale_factor=4, mode="nearest")
        self.resample3, self.resample4 = f.Resample2d(), f.Resample2d()
        self.flownetfusion = FlowNetFusion()

    def forward(self, inputs):
        rgb_mean = inputs.contiguous().view(inputs.size()[:2] + (-1,)).mean(dim=-1).view(inputs.size()[:2] + (1, 1, 1,))
        x = (inputs - rgb_mean) / self.rgb_max
        x = torch.cat((x[:, :, 0, :, :], x[:, :, 1, :, :]), dim=1)
        flownetc_flow = self.upsample1(self.flownetc(x)[0] * self.div_flow)
        resampled_img1 = self.resample1(x[:, 3:, :, :], flownetc_flow)
        norm_diff_img0 = self.channelnorm(x[:, :3, :, :] - resampled_img1)
        concat1 = torch.cat((x, resampled_img1, flownetc_flow / self.div_flow, norm_diff_img0), dim=1)
        flownets1_flow = self.upsample2(self.flownets_1(concat1)[0] * self.div_flow)
        resampled_img1 = self.resample2(x[:, 3:, :, :], flownets1_flow)
        norm_diff_img0 = self.channelnorm(x[:, :3, :, :] - resampled_img1)
        concat2 = torch.cat((x, resampled_img1, flownets1_flow / self.div_flow, norm_diff_img0), dim=1)
        flownets2_flow = self.upsample4(self.flownets_2(concat2)[0] * self.div_flow)
        norm_flownets2_flow = self.channelnorm(flownets2_flow)
        diff_flownets2_img1 = self.channelnorm((x[:, :3, :, :] - self.resample4(x[:, 3:, :, :], flownets2_flow)))
        flownetsd_flow = self.upsample3(self.flownets_d(x)[0] / self.div_flow)
        norm_flownetsd_flow = self.channelnorm(flownetsd_flow)
        diff_flownetsd_img1 = self.channelnorm((x[:, :3, :, :] - self.resample3(x[:, 3:, :, :], flownetsd_flow)))
        concat3 = torch.cat((x[:, :3, :, :], flownetsd_flow, flownets2_flow, norm_flownetsd_flow, norm_flownets2_flow,
                             diff_flownetsd_img1, diff_flownets2_img1), dim=1)
        return self.flownetfusion(concat3)


def _parent_flownet2_forward(net, inputs):
    """The fused inference data flow as functional calls (flownet2_forward before it was built on the modules)."""
    f = _f2()
    F2 = f.functional
    with torch.no_grad():
        div = float(net.div_flow)
        x = f.fused._normalise(inputs, net.rgb_max)
        x = torch.cat((x[:, :, 0], x[:, :, 1]), dim=1).float()
        B, _, H, W = x.shape
        flow2 = f.fused.flownetc_forward(net.flownetc, x)[0]
        concat1 = F2.warp_concat_forward(x, flow2, upsample="bilinear", flow_mul=div, flow_div=div)
        flow2 = net.flownets_1(concat1)[0]
        concat2 = F2.warp_concat_forward(x, flow2, upsample="bilinear", flow_mul=div, flow_div=div)
        s2_flow2 = net.flownets_2(concat2)[0]
        sd_flow2 = net.flownets_d(x)[0]
        concat3 = torch.empty((B, 11, H, W), dtype=torch.float32, device=x.device)
        F2.warp_concat_forward(x, sd_flow2, upsample="nearest", flow_mul=1.0 / div, flow_div=1.0, out=concat3, ch_x=0,
                               n_x=3, ch_warped=-1, ch_flow=3, ch_flow_norm=7, ch_diff_norm=9)
        F2.warp_concat_forward(x, s2_flow2, upsample="nearest", flow_mul=div, flow_div=1.0, out=concat3, ch_x=-1, n_x=0,
                               ch_warped=-1, ch_flow=5, ch_flow_norm=8, ch_diff_norm=10)
        return net.flownetfusion(concat3)


def _compare_flownet2_training_step(net, inputs, out_tol=1e-4, grad_tol=1e-3):
    """net(inputs) (unfused) and flownet2_train_forward in train mode: the same flow, the same parameter gradients.
    Returns (output error, largest parameter-gradient error) as max|d| / max|ref|."""
    f = _f2()
    params = [p for p in net.parameters() if p.requires_grad]
    results = []
    for run in (net, lambda inp: f.fused.flownet2_train_forward(net, inp)):
        out = run(inputs)
        w = torch.randn(out.shape, generator=torch.Generator().manual_seed(400)).cuda()
        results.append((out.detach(), torch.autograd.grad((out * w).sum(), params, allow_unused=True)))
    (out_u, grads_u), (out_f, grads_f) = results
    e_out = rel_err(out_f.cpu().numpy(), out_u.cpu().numpy())
    assert out_f.shape == out_u.shape and e_out <= out_tol, e_out
    # parameters the output does not depend on (the sub-networks' coarser flows) get no gradient in either graph
    assert [a is None for a in grads_f] == [b is None for b in grads_u]
    params, grads_f, grads_u = zip(*[(p, a, b) for p, a, b in zip(params, grads_f, grads_u) if a is not None])
    errs = [rel_err(a.cpu().numpy(), b.cpu().numpy()) for a, b in zip(grads_f, grads_u)]
    worst = max(range(len(errs)), key=lambda i: errs[i])
    assert errs[worst] <= grad_tol, (tuple(params[worst].shape), errs[worst])
    print("[flownet2_train_forward] %s: output max|d|/max|ref| = %.2e, parameter gradients: max %.2e, median %.2e"
          % (type(net).__name__, e_out, errs[worst], float(np.median(errs))))
    return e_out, errs[worst]


def test_flownet2_train_forward_stand_in():
    f = _f2()
    _deterministic()
    torch.manual_seed(0)
    net = FlowNet2().cuda().train()
    g = torch.Generator().manual_seed(401)
    inputs = (torch.rand(2, 3, 2, 128, 192, generator=g) * 255.0).cuda()
    assert f._lib.LIB.fn2b200_correlation_path(64, 16, 24, 20, 1, 20, 1, 2) == 2
    _compare_flownet2_training_step(net, inputs)
    # inference and training share one data flow: bit for bit under no_grad, in either mode, and equal to the
    # functional-call data flow flownet2_forward had before
    for mode in ("train", "eval"):
        getattr(net, mode)()
        with torch.no_grad():
            a = f.fused.flownet2_train_forward(net, inputs)
        b = f.fused.flownet2_forward(net, inputs)
        assert torch.equal(a, b) and torch.equal(b, _parent_flownet2_forward(net, inputs))
        assert torch.equal(f.fused.fused_forward(net, inputs), b)


needs_models = pytest.mark.skipif(not (oref.available() and oref.python_tree_available()),
                                  reason="reference python tree / extensions not installed under baseline/_ref, oracle/_ref")


@needs_models
def test_flownet2_train_forward_reference_flownet2():
    f = _f2()
    from flownet2_b200 import compat
    _deterministic()
    compat.uninstall()
    compat.install("B2")
    try:
        models = oref.import_reference_models(fresh=True)
        torch.manual_seed(0)
        net = models.FlowNet2(SimpleNamespace(rgb_max=255.0, fp16=False)).cuda().train()
        g = torch.Generator().manual_seed(402)
        inputs = (torch.rand(2, 3, 2, 128, 192, generator=g) * 255.0).cuda()
        _compare_flownet2_training_step(net, inputs)
        with torch.no_grad():
            a = f.fused.flownet2_train_forward(net, inputs)
        assert torch.equal(a, f.fused.flownet2_forward(net, inputs))
    finally:
        compat.uninstall()
