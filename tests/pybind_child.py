#!/usr/bin/env python3
"""Child process of the B1p tests: the compiled pybind modules correlation_cuda / resample2d_cuda / channelnorm_cuda.
pybind11 caches extension modules by name per interpreter, so they cannot share a process with the reference's own
extension modules of the same names (oracle/_ref) -- the parent test computes whatever needs those and hands it over as
.npy files.

    python tests/pybind_child.py ops
    python tests/pybind_child.py model <FlowNet2C|FlowNet2> <x.npy> <ref_out.npy>
    python tests/pybind_child.py refusals
Prints one line starting with "OK" on success (refusals: one JSON line, what tests/test_gpu_host_routes.py's cases give
through the compiled modules); any failure is an exception (non-zero exit).
"""
import faulthandler
import json
import os
import sys

faulthandler.enable()
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)
import numpy as np
import torch

from oracle import cpu as orc
from oracle import ref as oref
from util import assert_close, rel_err
import flownet2_b200
from flownet2_b200 import compat

TOL = 1e-4


def _randn(shape, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(*shape, generator=g).float()


def ops():
    compat.install("B1p")
    cc, rs, cn = sys.modules["correlation_cuda"], sys.modules["resample2d_cuda"], sys.modules["channelnorm_cuda"]
    for m in (cc, rs, cn):
        assert os.path.dirname(m.__file__).endswith("pybind"), m.__file__
    n0 = flownet2_b200.functional.launch_count()
    a, b = _randn((1, 64, 12, 20), 90).cuda(), _randn((1, 64, 12, 20), 91).cuda()
    out, r1, r2 = a.new(), a.new(), a.new()            # the reference's calling convention: empty outputs (correlation.py:20-22)
    assert cc.forward(a, b, r1, r2, out, 20, 1, 20, 1, 2, 1) == 1
    assert_close(out.cpu().numpy(), orc.correlation_forward(a.cpu().numpy(), b.cpu().numpy(), 20, 1, 20, 1, 2), TOL, "pybind corr fwd")
    go = _randn(tuple(out.shape), 92).cuda()
    g1, g2 = a.new(), a.new()
    assert cc.backward(a, b, r1, r2, go, g1, g2, 20, 1, 20, 1, 2, 1) == 1
    q1, q2 = orc.correlation_backward(a.cpu().numpy(), b.cpu().numpy(), go.cpu().numpy(), 20, 1, 20, 1, 2)
    assert_close(g1.cpu().numpy(), q1, TOL, "pybind corr gI1")
    assert_close(g2.cpu().numpy(), q2, TOL, "pybind corr gI2")
    g = torch.Generator().manual_seed(93)
    x = torch.rand(2, 6, 24, 40, generator=g).cuda()
    img, flow = x[:, 3:], (torch.randn(2, 2, 24, 40, generator=g) * 3).cuda()
    wo = torch.zeros(2, 3, 24, 40, device="cuda")      # pre-zeroed outputs (resample2d.py:18,31-32)
    rs.forward(img, flow, wo, 1, True)
    assert_close(wo.cpu().numpy(), orc.resample2d_forward(img.contiguous().cpu().numpy(), flow.cpu().numpy()), TOL, "pybind resample fwd")
    gw = torch.randn(2, 3, 24, 40, generator=g).cuda()
    gi, gf = torch.zeros(2, 3, 24, 40, device="cuda"), torch.zeros_like(flow)
    rs.backward(img, flow, gw, gi, gf, 1, True)
    e1, e2 = orc.resample2d_backward(img.contiguous().cpu().numpy(), flow.cpu().numpy(), gw.cpu().numpy())
    assert_close(gi.cpu().numpy(), e1, TOL, "pybind resample gImg")
    assert_close(gf.cpu().numpy(), e2, TOL, "pybind resample gFlow")
    no = torch.zeros(2, 1, 24, 40, device="cuda")
    cn.forward(wo, no, 2)
    nref = orc.channelnorm_forward(wo.cpu().numpy())
    assert_close(no.cpu().numpy(), nref, 1e-6, "pybind cnorm fwd")
    gn = torch.randn(2, 1, 24, 40, generator=g).cuda()
    gwo = torch.zeros_like(wo)
    cn.backward(wo, no, gn, gwo, 2)
    assert_close(gwo.cpu().numpy(), orc.channelnorm_backward(wo.cpu().numpy(), nref, gn.cpu().numpy()), 1e-5, "pybind cnorm bwd")
    xh = wo.half()
    nh = torch.zeros(2, 1, 24, 40, device="cuda", dtype=torch.float16)
    cn.forward(xh, nh, 2)                              # the reference dispatches on half too (channelnorm_kernel.cu:111)
    assert torch.allclose(nh.float(), no, atol=2e-3, rtol=2e-3)
    assert flownet2_b200.functional.launch_count() - n0 >= 9      # our library did the work
    print("parity through the compiled modules: ok", flush=True)
    for bad, pat in ((lambda: cc.forward(a.cpu(), b.cpu(), r1, r2, out, 20, 1, 20, 1, 2, 1), "CUDA tensor"),
                     (lambda: cc.backward(a, b, r1, r2, go, g1, g2, 20, 1, 20, 2, 2, 1), "stride1"),
                     (lambda: rs.forward(img, flow, wo, 2, True), "kernel_size")):
        print("expecting an error mentioning %r ..." % pat, flush=True)
        try:
            bad()
        except RuntimeError as e:
            assert pat in str(e), str(e)
        else:
            raise AssertionError("no error for " + pat)
    # the reference's OWN Python wrappers on top of the compiled modules (correlation.py / resample2d.py / channelnorm.py)
    if oref.python_tree_available():
        models = oref.import_reference_models(fresh=True)
        corr_mod = sys.modules["networks.correlation_package.correlation"]
        assert corr_mod.correlation_cuda is cc
        ar, br = a.clone().requires_grad_(), b.clone().requires_grad_()
        o = corr_mod.Correlation(20, 1, 20, 1, 2, 1)(ar, br)
        o.backward(go)                                  # autograd worker thread calls correlation_cuda.backward
        assert_close(ar.grad.cpu().numpy(), q1, TOL, "reference wrapper + pybind gI1")
    print("OK ops")


def model(name, x_path, ref_path):
    from types import SimpleNamespace
    torch.backends.cudnn.deterministic = True
    torch.backends.cudnn.benchmark = False
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    x = torch.from_numpy(np.load(x_path)).cuda()
    ref = np.load(ref_path)
    outs = {}
    for level in ("B1p", "B1"):
        compat.uninstall()
        compat.install(level)
        models = oref.import_reference_models(fresh=True)
        torch.manual_seed(0)
        net = getattr(models, name)(SimpleNamespace(rgb_max=255.0, fp16=False)).cuda().eval()
        kinds = {type(m).__module__ for m in net.modules() if type(m).__name__ in ("Correlation", "Resample2d", "ChannelNorm")}
        assert all(k.startswith("networks.") for k in kinds), kinds       # the reference's own wrapper classes
        if level == "B1p":
            assert os.path.dirname(sys.modules["correlation_cuda"].__file__).endswith("pybind")
        with torch.no_grad():
            outs[level] = net(x).float().cpu().numpy()
        del net
    compat.uninstall()
    assert np.array_equal(outs["B1p"], outs["B1"]), rel_err(outs["B1p"], outs["B1"])   # compiled glue == Python shims, bit for bit
    e = rel_err(outs["B1p"], ref)
    assert e < 1e-3, e
    print("OK model %s rel_err_vs_reference_kernels=%.3e" % (name, e))


def refusals():
    compat.install("B1p")
    from test_gpu_host_routes import ext_refusals
    print(json.dumps(ext_refusals(*(sys.modules[n] for n in ("correlation_cuda", "resample2d_cuda", "channelnorm_cuda")))))


if __name__ == "__main__":
    if sys.argv[1] == "ops":
        ops()
    elif sys.argv[1] == "refusals":
        refusals()
    else:
        model(sys.argv[2], sys.argv[3], sys.argv[4])
