"""GPU tests of FlowNet2CS and FlowNet2CSS through the fused data flow (fused.train_forward / fused.fused_forward ->
fused._stacked_flow2): CorrelationCat in the FlowNetC stage, WarpConcat(upsample="bilinear") for concat1 / concat2,
the network's own nn.Upsample for the full-resolution output.

Stand-in cases run on small networks with the reference's attribute names; the reference-model cases run the
unmodified models.FlowNet2CS / FlowNet2CSS where the reference's model code and kernels are installed.
"""
from types import SimpleNamespace

import numpy as np
import pytest
import torch
import torch.nn as nn

from oracle import ref as oref
from test_gpu_corr_cat import FlowNetC, _deterministic
from test_gpu_warp_concat_train import FlowNetS
from util import rel_err

pytestmark = pytest.mark.gpu
NAMES = ["FlowNet2CS", "FlowNet2CSS"]
# libfn2b200 launches of one inference forward, (module graph, fused).  Module graph: the Correlation module (split +
# tensor-core forward = 2), then per warp group Resample2d (1) and ChannelNorm (1).  Fused: correlation_cat (split +
# forward_cat = 2), then one warp-concat kernel per group.  The output nn.Upsample is torch's in both.
LAUNCHES = {"FlowNet2CS": (2 + 2, 2 + 1), "FlowNet2CSS": (2 + 2 * 2, 2 + 2 * 1)}


def _f2():
    import flownet2_b200
    return flownet2_b200


class FlowNet2CS(nn.Module):
    """FlowNet2CS's structure and attribute names on small sub-networks; forward = models.py:392-416 on the drop-in
    Resample2d / ChannelNorm modules: FlowNetC, one warp group, FlowNetS, a bilinear x4 output upsample."""

    def __init__(self, div_flow=20.0, rgb_max=255.0):
        super(FlowNet2CS, self).__init__()
        import flownet2_b200 as f
        self.div_flow, self.rgb_max = div_flow, rgb_max
        self.channelnorm = f.ChannelNorm()
        self.flownetc = FlowNetC()
        self.upsample1 = nn.Upsample(scale_factor=4, mode="bilinear")
        self.resample1 = f.Resample2d()
        self.flownets_1 = FlowNetS(12)
        self.upsample2 = nn.Upsample(scale_factor=4, mode="bilinear")

    def _group(self, x, flow, resample):
        """(x | img1 warped by the full-resolution flow | flow / div_flow | |img0 - warped|)"""
        warped = resample(x[:, 3:, :, :], flow)
        return torch.cat((x, warped, flow / self.div_flow, self.channelnorm(x[:, :3, :, :] - warped)), dim=1)

    def _first_two_stages(self, inputs):
        """-> (x, FlowNetS1's full-resolution flow)."""
        rgb_mean = inputs.contiguous().view(inputs.size()[:2] + (-1,)).mean(dim=-1).view(inputs.size()[:2] + (1, 1, 1,))
        x = (inputs - rgb_mean) / self.rgb_max
        x = torch.cat((x[:, :, 0, :, :], x[:, :, 1, :, :]), dim=1)
        flownetc_flow = self.upsample1(self.flownetc(x)[0] * self.div_flow)
        concat1 = self._group(x, flownetc_flow, self.resample1)
        return x, self.upsample2(self.flownets_1(concat1)[0] * self.div_flow)

    def forward(self, inputs):
        return self._first_two_stages(inputs)[1]


class FlowNet2CSS(FlowNet2CS):
    """FlowNet2CSS on the same sub-networks; forward = models.py:469-505: FlowNet2CS's stages, a second warp group,
    a second FlowNetS and a nearest x4 output upsample."""

    def __init__(self, div_flow=20.0, rgb_max=255.0):
        super(FlowNet2CSS, self).__init__(div_flow, rgb_max)
        import flownet2_b200 as f
        self.resample2 = f.Resample2d()
        self.flownets_2 = FlowNetS(12)
        self.upsample3 = nn.Upsample(scale_factor=4, mode="nearest")

    def forward(self, inputs):
        x, flownets1_flow = self._first_two_stages(inputs)
        concat2 = self._group(x, flownets1_flow, self.resample2)
        return self.upsample3(self.flownets_2(concat2)[0] * self.div_flow)


STANDINS = {"FlowNet2CS": FlowNet2CS, "FlowNet2CSS": FlowNet2CSS}


def _standin(name, mode="train"):
    torch.manual_seed(0)
    return getattr(STANDINS[name]().cuda(), mode)()


def _inputs(seed, B=2, H=128, W=192):
    return (torch.rand(B, 3, 2, H, W, generator=torch.Generator().manual_seed(seed)) * 255.0).cuda()


def _compare_training_step(net, inputs, out_tol=1e-4, grad_tol=1e-3):
    """net(inputs) (unfused) and fused.train_forward in train mode: the same flow, the same parameter gradients.
    Returns (output error, largest parameter-gradient error) as max|d| / max|ref|."""
    f = _f2()
    params = [p for p in net.parameters() if p.requires_grad]
    results = []
    for run in (net, lambda inp: f.fused.train_forward(net, inp)):
        out = run(inputs)
        w = torch.randn(out.shape, generator=torch.Generator().manual_seed(500)).cuda()
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
    print("[train_forward] %s: output max|d|/max|ref| = %.2e, parameter gradients: max %.2e, median %.2e"
          % (type(net).__name__, e_out, errs[worst], float(np.median(errs))))
    return e_out, errs[worst]


# ---- stand-ins -------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("name", NAMES)
def test_train_forward_stand_in(name):
    f = _f2()
    _deterministic()
    net = _standin(name)
    inputs = _inputs(501)
    assert f._lib.LIB.fn2b200_correlation_path(64, 16, 24, 20, 1, 20, 1, 2) == 2
    out = f.fused.train_forward(net, inputs)
    assert out.shape == (2, 2, 128, 192)
    _compare_training_step(net, inputs)


@pytest.mark.parametrize("name", NAMES)
def test_fused_forward_stand_in(name):
    """Inference and training share one data flow: bit for bit under no_grad, in either mode (both models return the
    full-resolution flow in both), and equal to net.forward on the drop-in modules to rounding."""
    f = _f2()
    _deterministic()
    net = _standin(name)
    inputs = _inputs(502)
    for mode in ("train", "eval"):
        getattr(net, mode)()
        with torch.no_grad():
            a = f.fused.train_forward(net, inputs)
            base = net(inputs)
        b = f.fused.fused_forward(net, inputs)
        assert not b.requires_grad
        assert torch.equal(a, b), mode
        assert b.shape == base.shape == (2, 2, 128, 192)
        assert rel_err(b.cpu().numpy(), base.cpu().numpy()) <= 1e-4, (mode, rel_err(b.cpu().numpy(), base.cpu().numpy()))


@pytest.mark.parametrize("name", NAMES)
def test_fused_forward_launches_stand_in(name):
    f = _f2()
    net = _standin(name, "eval")
    inputs = _inputs(503)
    with torch.no_grad():
        n0 = f.functional.launch_count()
        net(inputs)
        n1 = f.functional.launch_count()
    f.fused.fused_forward(net, inputs)
    n2 = f.functional.launch_count()
    assert (n1 - n0, n2 - n1) == LAUNCHES[name]


def _step(net, run, x):
    out = run(x)
    out.square().mean().backward()
    grads = [p.grad.clone() for p in net.parameters()]
    net.zero_grad(set_to_none=True)
    return out.detach(), grads


def _rel(p, q):
    return float((p - q).abs().max() / q.abs().max().clamp_min(1e-30))


@pytest.mark.parametrize("name", NAMES)
def test_train_forward_compiles_without_graph_breaks(name):
    """torch.compile(fullgraph=True, backend="aot_eager") of the fused training forward, forward and backward.
    FlowNet2CSS's output upsample is nearest, which AOT traces into an exact gather whose backward is an index_put
    accumulation instead of torch's upsample_nearest2d_backward: held to rounding, 1e-6 (bit-identical on an H100).
    FlowNet2CS's is bilinear, which AOT decomposes into elementwise aten ops that round differently from torch's eager
    upsample kernel (INTEGRATION section 4): held to 1e-4 (1.8e-6 at worst on an H100)."""
    f = _f2()
    _deterministic()
    net = _standin(name)
    x = _inputs(504)
    run = lambda inp: f.fused.train_forward(net, inp)
    torch._dynamo.reset()
    exp = torch._dynamo.explain(run)(x)
    assert exp.graph_break_count == 0 and exp.graph_count == 1, exp.break_reasons
    torch._dynamo.reset()
    out, grads = _step(net, run, x)
    cout, cgrads = _step(net, torch.compile(run, fullgraph=True, backend="aot_eager"), x)
    torch._dynamo.reset()
    errs = [_rel(cout, out)] + [_rel(p, q) for p, q in zip(cgrads, grads)]
    print("[aot_eager] %s: output %.2e, worst parameter gradient %.2e" % (name, errs[0], max(errs[1:])))
    assert max(errs) <= (1e-6 if name == "FlowNet2CSS" else 1e-4), errs


def _capture(fn_, static_inputs):
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            fn_(*static_inputs)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = fn_(*static_inputs)
    return g, out


@pytest.mark.parametrize("name", NAMES)
def test_cuda_graph_fused_forward(name):
    f = _f2()
    _deterministic()
    net = _standin(name, "eval")
    static = _inputs(505, H=448, W=1024)
    g, out = _capture(lambda x: f.fused.fused_forward(net, x), (static,))
    for seed in (506, 507):
        new = _inputs(seed, H=448, W=1024)
        static.copy_(new)
        g.replay()
        assert torch.equal(out, f.fused.fused_forward(net, new))


# ---- the unmodified reference models ----------------------------------------------------------------------------------

needs_models = pytest.mark.skipif(not (oref.available() and oref.python_tree_available()),
                                  reason="reference python tree / extensions not installed under baseline/_ref, oracle/_ref")


def _build_ref_model(name, level, mode="eval"):
    """The UNMODIFIED reference models.<name> on (a) the reference kernels, (b) our B1 extension shims, (c) our B2
    layer modules; seed 0 weights."""
    from flownet2_b200 import compat
    compat.uninstall()
    if level == "ref":
        oref.install_reference_extensions()
    else:
        compat.install(level)
    models = oref.import_reference_models(fresh=True)
    torch.manual_seed(0)
    return getattr(getattr(models, name)(SimpleNamespace(rgb_max=255.0, fp16=False)).cuda(), mode)()


@needs_models
@pytest.mark.parametrize("name", NAMES)
def test_unmodified_reference_models_run_on_our_layers(name):
    """models.FlowNet2CS / FlowNet2CSS load our layers unchanged -- B1 (Python *_cuda shims) and B2 (our modules) --
    and agree with the reference kernels on identical weights and inputs."""
    from flownet2_b200 import compat
    _deterministic()
    x = _inputs(508, B=1)
    outs = {}
    try:
        for level in ("ref", "B1", "B2"):
            net = _build_ref_model(name, level)
            with torch.no_grad():
                outs[level] = net(x).float().cpu().numpy()
            kinds = {type(m).__module__ for m in net.modules()
                     if type(m).__name__ in ("Correlation", "Resample2d", "ChannelNorm")}
            assert kinds and all(k.startswith("flownet2_b200" if level == "B2" else "networks.") for k in kinds), kinds
            del net
    finally:
        compat.uninstall()
    assert outs["ref"].shape == (1, 2, 128, 192) and np.isfinite(outs["ref"]).all()
    for level in ("B1", "B2"):
        assert rel_err(outs[level], outs["ref"]) < 1e-3, (level, rel_err(outs[level], outs["ref"]))


@needs_models
@pytest.mark.parametrize("name", NAMES)
def test_full_size_output_flow_agreement(name):
    """448x1024, bs 8, seed 0 weights, U(0,255) input, deterministic cuDNN with TF32 off: the output flow of the
    unmodified model on our layers (B2) and through fused.fused_forward against the same network on the reference's
    own kernels; the fused forward issues the launches counted in LAUNCHES."""
    f = _f2()
    from flownet2_b200 import compat
    _deterministic()
    g = torch.Generator().manual_seed(0)
    x = (torch.rand(8, 3, 2, 448, 1024, generator=g) * 255.0).cuda()
    try:
        net = _build_ref_model(name, "ref")
        with torch.no_grad():
            ref = net(x).float().cpu().numpy()
        del net
        torch.cuda.empty_cache()
        net = _build_ref_model(name, "B2")
        n0 = f.functional.launch_count()
        with torch.no_grad():
            ours = net(x).float().cpu().numpy()
        n1 = f.functional.launch_count()
        fz = f.fused.fused_forward(net, x).float().cpu().numpy()
        n2 = f.functional.launch_count()
        del net
    finally:
        compat.uninstall()
        torch.cuda.empty_cache()
    assert ref.shape == (8, 2, 448, 1024) and np.isfinite(ref).all()
    assert (n1 - n0, n2 - n1) == LAUNCHES[name]
    print("[full size] %s: B2 %.2e, fused %.2e against the reference kernels" % (name, rel_err(ours, ref),
                                                                                rel_err(fz, ref)))
    assert rel_err(ours, ref) < 1e-3, rel_err(ours, ref)
    assert rel_err(fz, ref) < 1e-3, rel_err(fz, ref)
    assert rel_err(fz, ours) < 1e-3, rel_err(fz, ours)


@needs_models
@pytest.mark.parametrize("name", NAMES)
def test_train_forward_reference_models(name):
    f = _f2()
    from flownet2_b200 import compat
    _deterministic()
    try:
        net = _build_ref_model(name, "B2", "train")
        inputs = _inputs(509)
        _compare_training_step(net, inputs)
        with torch.no_grad():
            a = f.fused.train_forward(net, inputs)
        assert torch.equal(a, f.fused.fused_forward(net, inputs))
    finally:
        compat.uninstall()
