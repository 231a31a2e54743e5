#!/usr/bin/env python3
"""Child process of tests/test_gpu_torch_ops.py: the unmodified reference models on our layer modules (compat B2) under
Dynamo, torch.compile and torch.export, in an interpreter of their own (compat rewrites sys.modules).

    python tests/torch_ops_child.py models <dir>     explain / compile the three networks; export FlowNet2C into <dir>
    python tests/torch_ops_child.py exported <dir>   run that exported program with only the operator library loaded
Prints one line starting with "OK" on success; any failure is an exception (non-zero exit).
"""
import glob
import os
import sys
from types import SimpleNamespace

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _rel(a, b):
    return float((a.float() - b.float()).abs().max() / b.float().abs().max().clamp_min(1e-30))


def _step(net, run, x):
    out = run(x)
    out = out[0] if isinstance(out, (tuple, list)) else out
    out.float().square().mean().backward()
    grads = [p.grad.clone() for p in net.parameters()]
    net.zero_grad(set_to_none=True)
    return out.detach(), grads


def models(tmp):
    for p in (ROOT, os.path.join(ROOT, "tests")):
        sys.path.insert(0, p)
    from oracle import ref as oref
    from test_gpu_corr_cat import _deterministic
    from flownet2_b200 import compat, fused
    _deterministic()
    compat.install("B2")
    mods = oref.import_reference_models(fresh=True)
    from networks.FlowNetC import FlowNetC
    args = SimpleNamespace(rgb_max=255.0, fp16=False)
    g = torch.Generator().manual_seed(0)
    x5 = (torch.rand(1, 3, 2, 128, 192, generator=g) * 255.0).cuda()
    x4 = torch.rand(1, 6, 128, 192, generator=g).cuda()
    torch.manual_seed(0)
    nets = {"FlowNetC": (FlowNetC(args, batchNorm=False).cuda().train(), x4, fused.train_forward),
            "FlowNet2C": (mods.FlowNet2C(args).cuda().train(), x5, fused.train_forward),
            "FlowNet2": (mods.FlowNet2(args).cuda().train(), x5, fused.flownet2_train_forward)}
    for name, (net, x, fused_fn) in nets.items():
        for what, run in (("module", net), ("fused", lambda inp, net=net, fused_fn=fused_fn: fused_fn(net, inp))):
            torch._dynamo.reset()
            exp = torch._dynamo.explain(run)(x)
            assert exp.graph_break_count == 0, (name, what, exp.break_reasons)
            torch._dynamo.reset()
            out, grads = _step(net, run, x)
            cout, cgrads = _step(net, torch.compile(run, fullgraph=True, backend="aot_eager"), x)
            same = torch.equal(out, cout) and all(torch.equal(p, q) for p, q in zip(grads, cgrads))
            worst = max([_rel(cout, out)] + [_rel(p, q) for p, q in zip(cgrads, grads)])
            print("%s %s: 0 graph breaks, aot_eager bit-identical %s (max rel %.2e)" % (name, what, same, worst), flush=True)
            # FlowNet2's unfused graph holds nn.Upsample(mode="bilinear"), which AOT tracing decomposes into elementwise
            # aten ops that round differently from torch's eager kernel; every other graph is bit-identical
            assert same or (name, what) == ("FlowNet2", "module") and worst <= 1e-3, (name, what, worst)
    net, x, _ = nets["FlowNet2C"]
    torch._dynamo.reset()
    out, grads = _step(net, net, x)
    cout, cgrads = _step(net, torch.compile(net, fullgraph=True), x)
    worst = max([_rel(cout, out)] + [_rel(p, q) for p, q in zip(cgrads, grads)])
    assert worst <= 1e-4, worst
    print("FlowNet2C inductor: max rel %.2e" % worst, flush=True)
    torch._dynamo.reset()
    net.eval()
    with torch.no_grad():
        ref = net(x5)
        ep = torch.export.export(net, (x5,))
        got = ep.module()(x5)
    assert torch.equal(got, ref), _rel(got, ref)
    assert any("fn2b200" in str(n.target) for n in ep.graph.nodes)
    torch.export.save(ep, os.path.join(tmp, "flownet2c.pt2"))
    torch.save({"x": x5.cpu(), "out": ref.cpu()}, os.path.join(tmp, "flownet2c_io.pt"))
    print("OK models")


def exported(tmp):
    torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = True, False      # as models() ran the net
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    torch.ops.load_library(glob.glob(os.path.join(ROOT, "flownet2-pytorch_b200", "pybind", "fn2b200_ops*.so"))[0])
    ep = torch.export.load(os.path.join(tmp, "flownet2c.pt2"))
    io = torch.load(os.path.join(tmp, "flownet2c_io.pt"))
    with torch.no_grad():
        got = ep.module()(io["x"].cuda())
    assert not any(k.startswith("flownet2_b200") for k in sys.modules), "the package was imported"
    assert torch.equal(got.cpu(), io["out"]), _rel(got.cpu(), io["out"])
    print("OK exported")


if __name__ == "__main__":
    {"models": models, "exported": exported}[sys.argv[1]](sys.argv[2])
