"""torch.ops.fn2b200 on the GPU: opcheck of every operator, the modules against the functional (C-ABI) calls bit for bit,
launch counts, graph-break-free tracing, torch.compile, CUDA-graph capture and torch.export."""
import os
import subprocess
import sys

import pytest
import torch

import flownet2_b200 as f
from flownet2_b200 import functional as F2
from flownet2_b200 import fused, ops
from oracle import ref as oref
from test_gpu_corr_cat import FlowNetC, _deterministic
from test_gpu_warp_concat_train import FlowNet2

pytestmark = pytest.mark.gpu
fn = torch.ops.fn2b200
FLOWNETC = (20, 1, 20, 1, 2)
HERE = os.path.dirname(os.path.abspath(__file__))


def _randn(shape, seed, scale=1.0, grad=False, dtype=torch.float32):
    g = torch.Generator().manual_seed(seed)
    t = (torch.randn(*shape, generator=g) * scale).to(dtype).cuda()
    return t.requires_grad_() if grad else t


def _grads(out, leaves, seed):
    go = _randn(tuple(out.shape), seed, dtype=out.dtype)
    return go, torch.autograd.grad(out, leaves, go)


# ---- opcheck -----------------------------------------------------------------------------------------------------------

def _opcheck_cases():
    a, b = _randn((1, 64, 8, 16), 1, grad=True), _randn((1, 64, 8, 16), 2, grad=True)
    prm = (4, 1, 4, 1, 1, 1)
    out, ws = fn.correlation_forward(a, b, *prm)
    redir = _randn((1, 8, 8, 16), 3, grad=True)
    cat, ws2 = fn.correlation_forward_cat(redir, a, b, *prm, 0.1)
    img, flow = _randn((2, 3, 12, 20), 4, grad=True), _randn((2, 2, 12, 20), 5, 2.0, grad=True)
    x, lr = _randn((2, 6, 16, 24), 6, grad=True), _randn((2, 2, 4, 6), 7, 0.2, grad=True)
    h = _randn((2, 3, 12, 20), 8, dtype=torch.float16, grad=True)
    d = lambda t: t.detach()  # noqa: E731
    return [
        ("correlation_forward", (a, b) + prm),
        ("correlation_backward", (d(a), d(b), d(out), ws) + prm + (True, True)),
        ("correlation_backward", (d(a), d(b), d(out), ws[:0]) + prm + (False, True)),
        ("correlation_forward_cat", (redir, a, b) + prm + (0.1,)),
        ("correlation_backward_cat", (d(a), d(b), d(cat), d(cat), ws2, 8, 0.1) + prm + (True, True)),
        ("resample2d_forward", (img, flow, 1, True)),
        ("resample2d_forward", (img[:, 1:], flow, 1, False)),
        ("resample2d_backward", (d(img), d(flow), d(img), 1, True, True, True)),
        ("channelnorm_forward", (img, 2)),
        ("channelnorm_forward", (h, 2)),
        ("channelnorm_backward", (d(h), fn.channelnorm_forward(d(h), 2), _randn((2, 1, 12, 20), 9, dtype=torch.float16), 2)),
        ("warp_concat_forward", (x, lr, 3, 1, 20.0, 20.0, 12, 0, 6, 6, 9, -1, 11)),
        ("warp_concat_forward", (x, lr, 3, 2, 0.05, 1.0, 11, 0, 3, -1, 3, 7, 9)),
        ("warp_concat_forward", (x, _randn((2, 2, 16, 24), 10, 2.0, grad=True), 3, 0, 1.0, 20.0, 12, 0, 6, 6, 9, -1, 11)),
        ("warp_concat_backward", (d(x), d(lr), _randn((2, 12, 16, 24), 11), 3, 1, 20.0, 20.0, 0, 6, 6, 9, -1, 11, True, True)),
        ("fusion_concat", (x, lr, _randn((2, 2, 4, 6), 12, 0.2, grad=True), 20.0)),
        ("fusion_concat_backward", (d(x), d(lr), d(lr), _randn((2, 11, 16, 24), 13), 20.0, True, True, False)),
    ]


def test_opcheck_every_op():
    seen, bad = set(), {}
    for name, args in _opcheck_cases():
        try:
            torch.library.opcheck(getattr(fn, name).default, args)
        except Exception as e:
            bad[name] = str(e)[:1500]
        seen.add(name)
    assert seen == set(ops.OPS)
    assert not bad, bad


# ---- the modules against the functional layer (the parent's path), bit for bit ----------------------------------------

def test_layer_modules_equal_functional_calls():
    a, b = _randn((2, 64, 24, 32), 20, grad=True), _randn((2, 64, 24, 32), 21, grad=True)
    out = f.Correlation(*FLOWNETC, 1)(a, b)
    go, (g1, g2) = _grads(out, (a, b), 22)
    ref, ws = F2.correlation_forward(a.detach(), b.detach(), *FLOWNETC, return_workspace=True)
    r1, r2 = F2.correlation_backward(a.detach(), b.detach(), go, *FLOWNETC, workspace=ws)
    assert torch.equal(out, ref) and torch.equal(g1, r1) and torch.equal(g2, r2)
    # FP32-FMA family (C % 64 != 0), and only one gradient asked for
    a2 = _randn((1, 24, 20, 28), 23, grad=True)
    b2 = _randn((1, 24, 20, 28), 24)
    out = f.Correlation(4, 1, 4, 1, 1, 1)(a2, b2)
    go, (g1,) = _grads(out, (a2,), 25)
    assert torch.equal(out, F2.correlation_forward(a2.detach(), b2, 4, 1, 4, 1, 1))
    assert torch.equal(g1, F2.correlation_backward(a2.detach(), b2, go, 4, 1, 4, 1, 1, need2=False)[0])

    x = _randn((2, 6, 40, 56), 26, grad=True)
    flow = _randn((2, 2, 40, 56), 27, 3.0, grad=True)
    w = f.Resample2d()(x[:, 3:], flow)
    go, (gx, gf) = _grads(w, (x, flow), 28)
    assert torch.equal(w, F2.resample2d_forward(x.detach()[:, 3:], flow.detach()))
    rx, rf = F2.resample2d_backward(x.detach()[:, 3:], flow.detach(), go)
    assert torch.equal(gf, rf) and torch.allclose(gx[:, 3:], rx, rtol=0, atol=1e-5) and not gx[:, :3].any()

    for dt in (torch.float32, torch.float16, torch.bfloat16):
        c = _randn((2, 3, 24, 40), 29, dtype=dt, grad=True)
        n = f.ChannelNorm()(c)
        go, (gc,) = _grads(n, (c,), 30)
        rn = F2.channelnorm_forward(c.detach())
        assert n.dtype == dt and torch.equal(n, rn)
        assert torch.equal(gc, F2.channelnorm_backward(c.detach(), rn, go))


def test_fused_modules_equal_functional_calls():
    _, C, H, W = 2, 64, 24, 32
    a, b = _randn((2, C, H, W), 40, grad=True), _randn((2, C, H, W), 41, grad=True)
    redir = _randn((2, 32, H, W), 42, grad=True)
    n0 = F2.launch_count()
    cat = fused.CorrelationCat(*FLOWNETC, 1, 0.1)(redir, a, b)
    n1 = F2.launch_count()
    go, (gr, g1, g2) = _grads(cat, (redir, a, b), 43)
    assert (n1 - n0, F2.launch_count() - n1) == (2, 1), "tensor cores: split + forward, then one backward launch"
    ref = torch.empty_like(cat)
    ref[:, :32].copy_(redir.detach())
    ref, ws = F2.correlation_forward_cat(a.detach(), b.detach(), ref, 32, 0.1, *FLOWNETC, return_workspace=True)
    r1, r2 = F2.correlation_backward_cat(a.detach(), b.detach(), go, ref, 32, 0.1, *FLOWNETC, workspace=ws)
    assert torch.equal(cat, ref) and torch.equal(g1, r1) and torch.equal(g2, r2) and torch.equal(gr, go[:, :32])

    x, lr = _randn((2, 6, 64, 96), 44), _randn((2, 2, 16, 24), 45, 0.3, grad=True)
    for up, mode in (("bilinear", 1), ("nearest", 2)):
        out = fused.WarpConcat(20.0, upsample=up)(x, lr)
        go, (gf,) = _grads(out, (lr,), 46)
        assert torch.equal(out, F2.warp_concat_forward(x, lr.detach(), upsample=up, flow_mul=20.0, flow_div=20.0))
        assert torch.equal(gf, F2.warp_concat_backward(x, lr.detach(), go, flow_div=20.0, upsample=up, flow_mul=20.0,
                                                       need_x=False)[1])
    sd, s2 = lr, _randn((2, 2, 16, 24), 47, 0.3, grad=True)
    out = fused.FusionConcat(20.0)(x, sd, s2)
    go, (g_sd, g_s2) = _grads(out, (sd, s2), 48)
    ref = torch.empty_like(out)
    lay_sd = dict(ch_x=0, n_x=3, ch_warped=-1, ch_flow=3, ch_flow_norm=7, ch_diff_norm=9)
    lay_s2 = dict(ch_x=-1, n_x=0, ch_warped=-1, ch_flow=5, ch_flow_norm=8, ch_diff_norm=10)
    F2.warp_concat_forward(x, sd.detach(), upsample="nearest", flow_mul=1.0 / 20.0, flow_div=1.0, out=ref, **lay_sd)
    F2.warp_concat_forward(x, s2.detach(), upsample="nearest", flow_mul=20.0, flow_div=1.0, out=ref, **lay_s2)
    assert torch.equal(out, ref)
    r_sd = F2.warp_concat_backward(x, sd.detach(), go, flow_div=1.0, upsample="nearest", flow_mul=1.0 / 20.0,
                                   need_x=False, **lay_sd)[1]
    r_s2 = F2.warp_concat_backward(x, s2.detach(), go, flow_div=1.0, upsample="nearest", flow_mul=20.0, need_x=False,
                                   **lay_s2)[1]
    assert torch.equal(g_sd, r_sd) and torch.equal(g_s2, r_s2)


# ---- Dynamo, torch.compile -------------------------------------------------------------------------------------------

def _standins():
    torch.manual_seed(0)
    c = FlowNetC().cuda().train()
    n2 = FlowNet2().cuda().train()
    g = torch.Generator().manual_seed(60)
    xc = torch.rand(2, 6, 128, 192, generator=g).cuda()
    x2 = (torch.rand(2, 3, 2, 128, 192, generator=g) * 255.0).cuda()
    return [("FlowNetC module", c, c, xc), ("FlowNetC fused.train_forward", c, lambda x: fused.train_forward(c, x), xc),
            ("FlowNet2 modules", n2, n2, x2),
            ("FlowNet2 fused.flownet2_train_forward", n2, lambda x: fused.flownet2_train_forward(n2, x), x2)]


def _step(net, run, x):
    out = run(x)
    out = out[0] if isinstance(out, (tuple, list)) else out
    out.float().square().mean().backward()
    grads = [p.grad.clone() for p in net.parameters()]
    net.zero_grad(set_to_none=True)
    return out.detach(), grads


def _rel(p, q):
    return float((p - q).abs().max() / q.abs().max().clamp_min(1e-30))


def test_no_graph_breaks_and_aot_eager_is_bit_identical():
    _deterministic()
    for what, net, run, x in _standins():
        torch._dynamo.reset()
        exp = torch._dynamo.explain(run)(x)
        assert exp.graph_break_count == 0 and exp.graph_count == 1, (what, exp.break_reasons)
        torch._dynamo.reset()
        out, grads = _step(net, run, x)
        cout, cgrads = _step(net, torch.compile(run, fullgraph=True, backend="aot_eager"), x)
        if what == "FlowNet2 modules":
            # the unfused graph's nn.Upsample(mode="bilinear") is decomposed into elementwise aten ops when AOT traces
            # it, which rounds differently from torch's eager upsample kernel; the fused forward has no such upsample
            assert max([_rel(cout, out)] + [_rel(p, q) for p, q in zip(cgrads, grads)]) <= 1e-3, what
            continue
        assert torch.equal(out, cout), what
        assert all(torch.equal(p, q) for p, q in zip(grads, cgrads)), what
    torch._dynamo.reset()


def test_inductor_within_tolerance():
    _deterministic()
    what, net, run, x = _standins()[3]
    out, grads = _step(net, run, x)
    torch._dynamo.reset()
    cout, cgrads = _step(net, torch.compile(run, fullgraph=True), x)
    torch._dynamo.reset()
    assert _rel(cout, out) <= 1e-4
    assert max(_rel(p, q) for p, q in zip(cgrads, grads)) <= 1e-4


# ---- CUDA graphs -------------------------------------------------------------------------------------------------------

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


def test_cuda_graph_flownet2_forward():
    _deterministic()
    torch.manual_seed(0)
    net = FlowNet2().cuda().eval()
    gen = torch.Generator().manual_seed(70)
    static = (torch.rand(2, 3, 2, 448, 1024, generator=gen) * 255.0).cuda()
    g, out = _capture(lambda x: fused.flownet2_forward(net, x), (static,))
    for seed in (71, 72):
        new = (torch.rand(2, 3, 2, 448, 1024, generator=torch.Generator().manual_seed(seed)) * 255.0).cuda()
        static.copy_(new)
        g.replay()
        assert torch.equal(out, fused.flownet2_forward(net, new))


def test_cuda_graph_correlation_cat_and_warp_concat_training_step():
    """One training step of FlowNet2's fused groups at 448x1024, batch 2: CorrelationCat at 1/8 resolution and
    WarpConcat with the quarter-resolution flow, forward and backward in one graph."""
    corr_cat, warp_concat = fused.CorrelationCat(*FLOWNETC, 1, 0.1), fused.WarpConcat(20.0, upsample="bilinear")
    shapes = [(2, 32, 56, 128), (2, 256, 56, 128), (2, 256, 56, 128), (2, 6, 448, 1024), (2, 2, 112, 256)]
    static = [_randn(s, 80 + i, 0.3) for i, s in enumerate(shapes)]
    for t in static[:3] + static[4:]:
        t.requires_grad_()
    wc = _randn((2, 473, 56, 128), 90)
    ww = _randn((2, 12, 448, 1024), 91)

    def step(redir, a, b, x, flow):
        loss = (corr_cat(redir, a, b) * wc).sum() + (warp_concat(x, flow) * ww).sum()
        return torch.autograd.grad(loss, (redir, a, b, flow))

    g, grads = _capture(step, static)
    for seed in (100, 200):
        new = [_randn(s, seed + i, 0.3) for i, s in enumerate(shapes)]
        for t, n in zip(static, new):
            t.detach().copy_(n)
        g.replay()
        ref = step(*[n.requires_grad_(i != 3) for i, n in enumerate(new)])
        assert all(torch.equal(p, q) for p, q in zip(grads, ref))


# ---- the unmodified reference models (compat B2) in a child interpreter -------------------------------------------------

needs_models = pytest.mark.skipif(not oref.python_tree_available(),
                                  reason="reference python tree not installed under baseline/_ref")


def _child(*args):
    r = subprocess.run([sys.executable, os.path.join(HERE, "torch_ops_child.py")] + list(args), capture_output=True,
                       text=True, timeout=1800)
    assert r.returncode == 0 and r.stdout.strip().splitlines()[-1].startswith("OK"), (r.stdout[-3000:], r.stderr[-4000:])
    return r.stdout.strip().splitlines()[-1]


@needs_models
def test_reference_models_trace_compile_and_export(tmp_path):
    _child("models", str(tmp_path))
    _child("exported", str(tmp_path))
