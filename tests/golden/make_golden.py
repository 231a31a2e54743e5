#!/usr/bin/env python3
"""Generate tests/golden/*.npz = outputs of the REFERENCE's own CUDA kernels (oracle/_ref, rebuilt
for sm_90a by oracle/build_ref.py) on small seeded inputs.  Run on a GPU machine where oracle/_ref is built:

    python tests/golden/make_golden.py <out_dir>     # then copy the .npz files to tests/golden/

correlation_* / resample2d_* / channelnorm_c*: whole tensors; they pin the CPU restatement
(tests/test_oracle_cpu.py::test_oracle_matches_reference_kernel_golden).
refk_*: what tests/test_gpu_parity.py compares our kernels with -- the reference kernels' results on the inputs those
tests generate from their seeds; tensors larger than SAMPLE elements are stored as the values at sample_index(n).
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import ref as oref  # noqa: E402


SAMPLE = 16384


def sample_index(n):
    """Fixed, sorted sample of SAMPLE flat indices into a tensor of n elements (all of them when n <= SAMPLE)."""
    if n <= SAMPLE:
        return np.arange(n)
    return np.sort(np.random.RandomState(7).choice(n, SAMPLE, replace=False))


def _sampled(t):
    a = t.detach().cpu().numpy().ravel()
    return a[sample_index(a.size)]


def _randn(shape, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(*shape, generator=g).float()


def reference_kernel_cases(out_dir, corr, rs, cn):
    """The inputs of test_gpu_parity's *_vs_reference_* tests (same seeds, same order of generator calls)."""
    for shape in ((1, 256, 48, 64), (2, 20, 13, 36)):
        a, b = _randn(shape, 41).cuda(), _randn(shape, 42).cuda()
        r1, r2, rout = a.new_empty(0), a.new_empty(0), a.new_empty(0)
        corr.forward(a, b, r1, r2, rout, 20, 1, 20, 1, 2, 1)
        go = _randn(tuple(rout.shape), 43).cuda()
        gi1, gi2 = a.new_empty(0), a.new_empty(0)
        corr.backward(a, b, a.new_empty(0), a.new_empty(0), go, gi1, gi2, 20, 1, 20, 1, 2, 1)
        np.savez_compressed(os.path.join(out_dir, "refk_correlation_%s.npz" % "x".join(map(str, shape))),
                            output=_sampled(rout), grad_input1=_sampled(gi1), grad_input2=_sampled(gi2),
                            output_shape=np.array(rout.shape))
    g = torch.Generator().manual_seed(44)
    img = torch.rand(2, 3, 32, 48, generator=g).cuda()
    flow = (torch.randn(2, 2, 32, 48, generator=g) * 6).cuda()
    go = torch.randn(2, 3, 32, 48, generator=g).cuda()
    rout = torch.zeros_like(img)
    rs.forward(img, flow, rout, 1, True)
    rg1, rg2 = torch.zeros_like(img), torch.zeros_like(flow)
    rs.backward(img, flow, go, rg1, rg2, 1, True)
    x = torch.randn(2, 3, 32, 48, generator=g).cuda()
    ro = torch.zeros(2, 1, 32, 48, device="cuda")
    cn.forward(x, ro, 2)
    gon = torch.randn(2, 1, 32, 48, generator=g).cuda()
    rgi = torch.zeros_like(x)
    cn.backward(x, ro, gon, rgi, 2)
    np.savez_compressed(os.path.join(out_dir, "refk_resample_channelnorm.npz"), resample_output=rout.cpu().numpy(),
                        resample_grad_img=rg1.cpu().numpy(), resample_grad_flow=rg2.cpu().numpy(),
                        channelnorm_output=ro.cpu().numpy(), channelnorm_grad_input=rgi.cpu().numpy())
    for shape in ((2, 3, 16, 24), (1, 2, 7, 9), (2, 3, 64, 128)):
        x = _randn(shape, 35).cuda().half()
        ro = torch.zeros(shape[0], 1, shape[2], shape[3], device="cuda", dtype=torch.float16)
        cn.forward(x, ro, 2)
        go = _randn(tuple(ro.shape), 36).cuda().half()
        rgi = torch.zeros_like(x)
        cn.backward(x, ro, go, rgi, 2)
        np.savez_compressed(os.path.join(out_dir, "refk_channelnorm_half_%s.npz" % "x".join(map(str, shape))),
                            output=ro.cpu().numpy(), grad_input=rgi.cpu().numpy())


def main(out_dir):
    os.makedirs(out_dir, exist_ok=True)
    corr = oref.load_extension("correlation_cuda")
    rs = oref.load_extension("resample2d_cuda")
    cn = oref.load_extension("channelnorm_cuda")
    g = torch.Generator().manual_seed(1234)
    cases = [("flownetc", (20, 1, 20, 1, 2), (1, 16, 12, 16)), ("k3", (4, 3, 4, 1, 2), (1, 6, 10, 9)),
             ("s2_1", (3, 1, 3, 1, 1), (2, 5, 8, 6)), ("padgt", (6, 1, 4, 1, 2), (1, 33, 7, 8))]
    for name, prm, shape in cases:
        a = torch.randn(*shape, generator=g).cuda()
        b = torch.randn(*shape, generator=g).cuda()
        out = a.new_empty(0)
        corr.forward(a, b, a.new_empty(0), a.new_empty(0), out, *prm, 1)
        go = torch.randn(out.shape, generator=g).cuda()
        g1, g2 = a.new_empty(0), a.new_empty(0)
        corr.backward(a, b, a.new_empty(0), a.new_empty(0), go, g1, g2, *prm, 1)
        np.savez_compressed(os.path.join(out_dir, "correlation_%s.npz" % name), op="correlation", params=np.array(prm),
                            input1=a.cpu().numpy(), input2=b.cpu().numpy(), output=out.cpu().numpy(),
                            grad_output=go.cpu().numpy(), grad_input1=g1.cpu().numpy(), grad_input2=g2.cpu().numpy())
    for name, sigma, bilinear in (("sigma4", 4.0, True), ("sigma40", 40.0, True), ("nearest", 3.0, False)):
        img = torch.rand(2, 3, 12, 16, generator=g).cuda()
        flow = (torch.randn(2, 2, 12, 16, generator=g) * sigma).cuda()
        go = torch.randn(2, 3, 12, 16, generator=g).cuda()
        out = torch.zeros_like(img)
        rs.forward(img, flow, out, 1, bilinear)
        g1, g2 = torch.zeros_like(img), torch.zeros_like(flow)
        rs.backward(img, flow, go, g1, g2, 1, bilinear)
        np.savez_compressed(os.path.join(out_dir, "resample2d_%s.npz" % name), op="resample2d", bilinear=bilinear,
                            input1=img.cpu().numpy(), input2=flow.cpu().numpy(), output=out.cpu().numpy(),
                            grad_output=go.cpu().numpy(), grad_input1=g1.cpu().numpy(), grad_input2=g2.cpu().numpy())
    for C in (2, 3):
        x = torch.randn(2, C, 10, 12, generator=g).cuda()
        x[0, :, 0, 0] = 0
        out = torch.zeros(2, 1, 10, 12, device="cuda")
        cn.forward(x, out, 2)
        go = torch.randn(2, 1, 10, 12, generator=g).cuda()
        gi = torch.zeros_like(x)
        cn.backward(x, out, go, gi, 2)
        np.savez_compressed(os.path.join(out_dir, "channelnorm_c%d.npz" % C), op="channelnorm", input1=x.cpu().numpy(),
                            output=out.cpu().numpy(), grad_output=go.cpu().numpy(), grad_input1=gi.cpu().numpy())
    reference_kernel_cases(out_dir, corr, rs, cn)
    torch.cuda.synchronize()
    print("wrote", sorted(os.listdir(out_dir)))


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "gpurun_out", "golden"))
