"""GPU tests of the fused correlation -> LeakyReLU -> concat backward (fn2b200_correlation_backward_cat,
functional.correlation_backward_cat, fused.CorrelationCat, fused.train_forward).

The backward masks every gradOutput value with LeakyReLU's derivative before any other arithmetic, so on every kernel
family it must be bit-identical to masking in torch and running the plain correlation backward on the result.
"""
from types import SimpleNamespace

import numpy as np
import pytest
import torch
import torch.nn as nn

from oracle import cpu as orc
from oracle import ref as oref
from util import assert_close, rel_err

pytestmark = pytest.mark.gpu
FLOWNETC = (20, 1, 20, 1, 2)


def _f2():
    import flownet2_b200
    return flownet2_b200


def _randn(shape, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).float()


# (shape, (pad, k, md, s1, s2), expected path of the plain entry points, FN2B200_CORR_BWD)
FAMILIES = [
    ((2, 64, 12, 20), FLOWNETC, 2, None),          # tensor cores
    ((1, 20, 13, 64), FLOWNETC, 1, None),          # TMA-tiled FP32 FMA
    ((1, 6, 10, 12), (4, 3, 4, 1, 2), 0, None),    # generic, kernel_size 3: the mask applies inside the window sum
    ((2, 64, 12, 20), FLOWNETC, 2, "fma"),         # tensor-core shape forced onto the tiled FMA kernels
]


@pytest.mark.parametrize("shape,prm,path,bwd_env", FAMILIES)
@pytest.mark.parametrize("slope", [0.1, 0.0, 1.0])
def test_backward_cat_equals_masked_plain_backward(shape, prm, path, bwd_env, slope, monkeypatch):
    f = _f2()
    F2 = f.functional
    assert f._lib.LIB.fn2b200_correlation_path(shape[1], shape[2], shape[3], *prm) == path
    if bwd_env:
        monkeypatch.setenv("FN2B200_CORR_BWD", bwd_env)
    a, b = _randn(shape, 90).cuda(), _randn(shape, 91).cuda()
    D, oH, oW = F2.correlation_out_shape(shape[1], shape[2], shape[3], *prm)
    # channels before AND after the correlation's range
    cat = torch.full((shape[0], 32 + D + 3, oH, oW), 5.0, device="cuda")
    cat, ws = F2.correlation_forward_cat(a, b, cat, 32, slope, *prm, return_workspace=True)
    assert (ws is not None) == (path == 2)
    gcat = _randn(tuple(cat.shape), 92).cuda()
    g1, g2 = F2.correlation_backward_cat(a, b, gcat, cat, 32, slope, *prm, workspace=ws)
    act, gs = cat[:, 32:32 + D], gcat[:, 32:32 + D]
    masked = torch.where(act > 0, gs, gs * slope).contiguous()
    r1, r2 = F2.correlation_backward(a, b, masked, *prm)
    assert torch.equal(g1, r1) and torch.equal(g2, r2)
    if slope == 1.0:                                  # no activation: the concat buffer is not needed
        h1, h2 = F2.correlation_backward_cat(a, b, gcat, None, 32, 1.0, *prm)
        assert torch.equal(h1, r1) and torch.equal(h2, r2)
    o1, o2 = orc.correlation_backward(a.cpu().numpy(), b.cpu().numpy(), masked.cpu().numpy(), *prm)
    assert_close(g1.cpu().numpy(), o1, 1e-4, "backward_cat gI1 %s slope %g" % (shape, slope))
    assert_close(g2.cpu().numpy(), o2, 1e-4, "backward_cat gI2 %s slope %g" % (shape, slope))
    # one gradient at a time gives the same bits
    only1, none2 = F2.correlation_backward_cat(a, b, gcat, cat, 32, slope, *prm, need2=False, workspace=ws)
    none1, only2 = F2.correlation_backward_cat(a, b, gcat, cat, 32, slope, *prm, need1=False, workspace=ws)
    assert none1 is None and none2 is None and torch.equal(only1, r1) and torch.equal(only2, r2)


def _unfused(redir, f1, f2, slope=0.1, prm=FLOWNETC):
    """FlowNetC.py:86-92 on the drop-in module: Correlation, in-place LeakyReLU, torch.cat."""
    corr = _f2().Correlation(*prm, 1)(f1, f2)
    return torch.cat((redir, nn.functional.leaky_relu(corr, slope, inplace=True)), 1)


def _leaves(seed, B=2, C=64, H=12, W=20, R=32, redir_dtype=torch.float32, grads=(True, True, True)):
    redir = _randn((B, R, H, W), seed).cuda().to(redir_dtype)
    f1, f2 = _randn((B, C, H, W), seed + 1).cuda(), _randn((B, C, H, W), seed + 2).cuda()
    return [t.requires_grad_(r) for t, r in zip((redir, f1, f2), grads)]


@pytest.mark.parametrize("case", ["all", "noncontiguous_grad", "f1_frozen", "redir_frozen", "half_redir"])
def test_correlation_cat_module_matches_unfused_graph(case):
    f = _f2()
    kw = {"f1_frozen": dict(grads=(True, False, True)), "redir_frozen": dict(grads=(False, True, True)),
          "half_redir": dict(redir_dtype=torch.float16)}.get(case, {})
    ours, ref = _leaves(100, **kw), _leaves(100, **kw)
    out = f.fused.CorrelationCat(*FLOWNETC, 1, 0.1)(*ours)
    base = _unfused(*ref)
    assert out.dtype == torch.float32 and out.shape == base.shape == (2, 32 + 441, 12, 20)
    # forward: bit-identical to correlation_forward_cat plus the redir copy
    with torch.no_grad():
        fc = torch.empty_like(out)
        fc[:, :32].copy_(ours[0])
        f.functional.correlation_forward_cat(ours[1], ours[2], fc, 32, 0.1, *FLOWNETC)
    assert torch.equal(out, fc) and torch.equal(out, base)
    g = _randn(tuple(out.shape), 103).cuda()
    if case == "noncontiguous_grad":
        g = g.transpose(2, 3).contiguous().transpose(2, 3)
        assert not g.is_contiguous()
    out.backward(g)
    base.backward(g)
    for t, r in zip(ours, ref):
        assert (t.grad is None) == (r.grad is None) == (not t.requires_grad)
        if t.grad is not None:
            assert t.grad.dtype == t.dtype and torch.equal(t.grad, r.grad)


def test_correlation_cat_launches_on_tensor_cores():
    """forward_cat = split + correlation (2 launches); the backward reuses the forward's split: exactly 1 launch."""
    f = _f2()
    redir, f1, f2 = _leaves(110)
    n0 = f.functional.launch_count()
    out = f.fused.CorrelationCat(*FLOWNETC)(redir, f1, f2)
    n1 = f.functional.launch_count()
    out.backward(_randn(tuple(out.shape), 111).cuda())
    n2 = f.functional.launch_count()
    assert (n1 - n0, n2 - n1) == (2, 1)


def test_full_size_fused_gradients_equal_unfused():
    """FlowNet2's FlowNetC shape at 448x1024, bs 8: the correlation input [8,256,56,128], cost volume [8,441,56,128]."""
    f = _f2()
    gen = torch.Generator(device="cuda").manual_seed(7)
    mk = lambda *s: torch.randn(*s, device="cuda", generator=gen)
    f1, f2, redir = mk(8, 256, 56, 128), mk(8, 256, 56, 128), mk(8, 32, 56, 128)
    g = mk(8, 473, 56, 128)
    assert f._lib.LIB.fn2b200_correlation_path(256, 56, 128, *FLOWNETC) == 2
    grads = []
    for fused in (True, False):
        leaves = [t.clone().requires_grad_() for t in (redir, f1, f2)]
        out = f.fused.CorrelationCat(*FLOWNETC)(*leaves) if fused else _unfused(*leaves)
        grads.append(torch.autograd.grad(out, leaves, g))
        del out
    for x, y in zip(*grads):
        assert torch.equal(x, y)


# ------------------------------------------------------------------------------------------------
# train_forward on a FlowNetC-shaped network
# ------------------------------------------------------------------------------------------------
def _conv(cin, cout, k=3, s=1):
    return nn.Sequential(nn.Conv2d(cin, cout, k, s, (k - 1) // 2), nn.LeakyReLU(0.1, inplace=True))


def _deconv(cin, cout):
    return nn.Sequential(nn.ConvTranspose2d(cin, cout, 4, 2, 1), nn.LeakyReLU(0.1, inplace=True))


class FlowNetC(nn.Module):
    """A small network with FlowNetC's structure and attribute names (conv3 gives the correlation 64 channels, so it
    runs on tensor cores).  forward = the unfused graph on the drop-in Correlation module."""

    def __init__(self):
        super(FlowNetC, self).__init__()
        import flownet2_b200 as f
        self.conv1, self.conv2, self.conv3 = _conv(3, 16, 3, 2), _conv(16, 32, 3, 2), _conv(32, 64, 3, 2)
        self.conv_redir = _conv(64, 32, 1)
        self.corr = f.Correlation(*FLOWNETC, 1)
        self.corr_activation = nn.LeakyReLU(0.1, inplace=True)
        self.conv3_1 = _conv(473, 64)
        self.conv4, self.conv4_1 = _conv(64, 64, 3, 2), _conv(64, 64)
        self.conv5, self.conv5_1 = _conv(64, 64, 3, 2), _conv(64, 64)
        self.conv6, self.conv6_1 = _conv(64, 64, 3, 2), _conv(64, 64)
        self.deconv5, self.deconv4, self.deconv3, self.deconv2 = _deconv(64, 32), _deconv(98, 32), _deconv(98, 32), _deconv(98, 16)
        self.predict_flow6, self.predict_flow5, self.predict_flow4 = (nn.Conv2d(c, 2, 3, 1, 1) for c in (64, 98, 98))
        self.predict_flow3, self.predict_flow2 = nn.Conv2d(98, 2, 3, 1, 1), nn.Conv2d(50, 2, 3, 1, 1)
        (self.upsampled_flow6_to_5, self.upsampled_flow5_to_4, self.upsampled_flow4_to_3,
         self.upsampled_flow3_to_2) = (nn.ConvTranspose2d(2, 2, 4, 2, 1) for _ in range(4))

    def forward(self, x):
        out_conv2a = self.conv2(self.conv1(x[:, 0:3]))
        out_conv3a = self.conv3(out_conv2a)
        out_conv3b = self.conv3(self.conv2(self.conv1(x[:, 3:])))
        out_corr = self.corr_activation(self.corr(out_conv3a, out_conv3b))
        out_conv3_1 = self.conv3_1(torch.cat((self.conv_redir(out_conv3a), out_corr), 1))
        out_conv4 = self.conv4_1(self.conv4(out_conv3_1))
        out_conv5 = self.conv5_1(self.conv5(out_conv4))
        out_conv6 = self.conv6_1(self.conv6(out_conv5))
        flow6 = self.predict_flow6(out_conv6)
        concat5 = torch.cat((out_conv5, self.deconv5(out_conv6), self.upsampled_flow6_to_5(flow6)), 1)
        flow5 = self.predict_flow5(concat5)
        concat4 = torch.cat((out_conv4, self.deconv4(concat5), self.upsampled_flow5_to_4(flow5)), 1)
        flow4 = self.predict_flow4(concat4)
        concat3 = torch.cat((out_conv3_1, self.deconv3(concat4), self.upsampled_flow4_to_3(flow4)), 1)
        flow3 = self.predict_flow3(concat3)
        concat2 = torch.cat((out_conv2a, self.deconv2(concat3), self.upsampled_flow3_to_2(flow3)), 1)
        flow2 = self.predict_flow2(concat2)
        return (flow2, flow3, flow4, flow5, flow6) if self.training else (flow2,)


def _deterministic():
    torch.backends.cudnn.deterministic = True
    torch.backends.cudnn.benchmark = False
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False


def _compare_training_step(net, x, fwd):
    """The unfused net(x) and fwd(net, x) in train mode: the same five flows, the same parameter gradients."""
    params = [p for p in net.parameters() if p.requires_grad]
    results = []
    for run in (net, lambda inp: fwd(net, inp)):
        flows = run(x)
        assert isinstance(flows, tuple) and len(flows) == 5
        w = [_randn(tuple(fl.shape), 200 + i).cuda() for i, fl in enumerate(flows)]
        loss = sum((fl * wi).sum() for fl, wi in zip(flows, w))
        results.append(([fl.detach() for fl in flows], torch.autograd.grad(loss, params)))
    (flows_u, grads_u), (flows_f, grads_f) = results
    for a, b in zip(flows_f, flows_u):
        assert a.shape == b.shape and rel_err(a.cpu().numpy(), b.cpu().numpy()) <= 1e-6
    for p, a, b in zip(params, grads_f, grads_u):
        e = rel_err(a.cpu().numpy(), b.cpu().numpy())
        assert e <= 1e-4, (tuple(p.shape), e)


def test_train_forward_flownetc_stand_in():
    f = _f2()
    _deterministic()
    torch.manual_seed(0)
    net = FlowNetC().cuda().train()
    x = _randn((2, 6, 128, 192), 300).cuda()
    _compare_training_step(net, x, f.fused.train_forward)
    # eval mode: what net.forward returns there
    net.eval()
    with torch.no_grad():
        assert torch.equal(f.fused.train_forward(net, x)[0], f.fused.flownetc_forward(net, x)[0])


needs_models = pytest.mark.skipif(not (oref.available() and oref.python_tree_available()),
                                  reason="reference python tree / extensions not installed under baseline/_ref, oracle/_ref")


@needs_models
def test_train_forward_reference_flownet2c():
    f = _f2()
    from flownet2_b200 import compat
    _deterministic()
    compat.uninstall()
    compat.install("B2")
    try:
        models = oref.import_reference_models(fresh=True)
        torch.manual_seed(0)
        net = models.FlowNet2C(SimpleNamespace(rgb_max=255.0, fp16=False)).cuda().train()
        g = torch.Generator().manual_seed(301)
        x = (torch.rand(2, 3, 2, 128, 192, generator=g) * 255.0).cuda()
        _compare_training_step(net, x, f.fused.train_forward)
    finally:
        compat.uninstall()
