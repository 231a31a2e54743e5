"""CPU tests that PIN the oracle (oracle/oracle.c) -- no GPU needed.

The reference ships no golden vectors (SURVEY section 4), so the restatement is pinned against
(1) stock-PyTorch formulations + autograd in fp64 (tests/torch_ref.py), (2) hand-derived
known-answer cases (SURVEY 8c), and (3) committed outputs of the reference's OWN kernels rebuilt for
sm_90a and run on an H100 (tests/golden/*.npz, produced by tests/golden/make_golden.py).
"""
import glob
import os

import numpy as np
import pytest
import torch

import torch_ref as tr
from oracle import cpu as orc
from util import assert_close, rel_err

CORR_CASES = [
    # (pad, k, md, s1, s2), (B, C, H, W)
    ((4, 1, 4, 1, 2), (2, 7, 9, 11)),
    ((3, 1, 3, 1, 1), (1, 5, 8, 6)),
    ((4, 3, 4, 1, 2), (1, 6, 10, 9)),     # kernel_size 3
    ((6, 1, 4, 1, 2), (1, 33, 7, 8)),     # pad > md: output larger than input; C not multiple of 32
    ((2, 1, 4, 1, 2), (1, 4, 12, 13)),    # pad < md: output smaller than input
    ((5, 1, 5, 1, 2), (1, 3, 8, 8)),      # md not a multiple of stride2
    ((20, 1, 20, 1, 2), (1, 8, 12, 16)),  # FlowNetC parameters on a tiny map
]


@pytest.mark.parametrize("params,shape", CORR_CASES)
def test_correlation_forward_backward_vs_torch(params, shape):
    pad, k, md, s1, s2 = params
    g = torch.Generator().manual_seed(1)
    f1 = torch.randn(*shape, dtype=torch.float64, generator=g, requires_grad=True)
    f2 = torch.randn(*shape, dtype=torch.float64, generator=g, requires_grad=True)
    ref = tr.correlation(f1, f2, pad, k, md, s1, s2)
    out = orc.correlation_forward(f1.detach().numpy(), f2.detach().numpy(), pad, k, md, s1, s2)
    assert_close(out, ref.detach().numpy(), 2e-6, "oracle corr fwd")
    go = torch.randn(ref.shape, dtype=torch.float64, generator=g)
    ref.backward(go)
    g1, g2 = orc.correlation_backward(f1.detach().numpy(), f2.detach().numpy(), go.numpy(), pad, k, md, s1, s2)
    assert_close(g1, f1.grad.numpy(), 2e-6, "oracle corr gI1")
    assert_close(g2, f2.grad.numpy(), 2e-6, "oracle corr gI2")


def test_correlation_forward_stride1_2_vs_torch():
    f1 = torch.randn(1, 4, 12, 13, dtype=torch.float64)
    f2 = torch.randn(1, 4, 12, 13, dtype=torch.float64)
    ref = tr.correlation(f1, f2, 2, 1, 4, 2, 2)
    out = orc.correlation_forward(f1.numpy(), f2.numpy(), 2, 1, 4, 2, 2)
    assert_close(out, ref.numpy(), 2e-6, "oracle corr fwd stride1=2")
    with pytest.raises(RuntimeError):
        orc.correlation_backward(f1.numpy(), f2.numpy(), out, 2, 1, 4, 2, 2)


def test_correlation_known_answers():
    # (1) ones x ones: every displacement fully inside the image = 1.0; displacements reaching into the
    #     zero padding = 0 (k=1 -> a single product per channel).
    C, H, W = 5, 8, 8
    ones = np.ones((1, C, H, W), np.float32)
    out = orc.correlation_forward(ones, ones, 4, 1, 4, 1, 2)
    assert out.shape == (1, 25, 8, 8)
    centre = out[0, 12]
    assert np.allclose(centre, 1.0)
    assert np.isclose(out[0, 0, 0, 0], 0.0) and np.isclose(out[0, 0, 4, 4], 1.0)
    # (2) f2 = f1 shifted by (2a, 2b) -> arg-max channel = (a+dr)*ds + (b+dr)
    rng = np.random.RandomState(0)
    f1 = rng.randn(1, 16, 16, 16).astype(np.float32)
    a, b = 1, -2
    f2 = np.roll(f1, (2 * a, 2 * b), axis=(2, 3))
    out = orc.correlation_forward(f1, f2, 4, 1, 4, 1, 2)
    assert int(out[0, :, 8, 8].argmax()) == (a + 2) * 5 + (b + 2)
    # (3) D and output-shape arithmetic of correlation_cuda.cc:19-34
    assert orc.correlation_out_shape(256, 48, 64, 20, 1, 20, 1, 2) == (441, 48, 64)
    assert orc.correlation_out_shape(8, 12, 13, 2, 1, 4, 2, 2) == (25, 4, 5)


def test_resample2d_vs_grid_sample():
    g = torch.Generator().manual_seed(2)
    img = torch.rand(2, 3, 9, 13, dtype=torch.float64, generator=g, requires_grad=True)
    flow = (torch.randn(2, 2, 9, 13, dtype=torch.float64, generator=g) * 4).requires_grad_()
    ref = tr.resample2d(img, flow)
    go = torch.randn(ref.shape, dtype=torch.float64, generator=g)
    ref.backward(go)
    out = orc.resample2d_forward(img.detach().numpy(), flow.detach().numpy())
    g1, g2 = orc.resample2d_backward(img.detach().numpy(), flow.detach().numpy(), go.numpy())
    assert_close(out, ref.detach().numpy(), 1e-5, "oracle resample fwd")
    assert_close(g1, img.grad.numpy(), 1e-5, "oracle resample gImg")
    assert_close(g2, flow.grad.numpy(), 1e-5, "oracle resample gFlow")


def test_resample2d_known_answers():
    rng = np.random.RandomState(3)
    img = rng.rand(1, 2, 6, 7).astype(np.float32)
    zero = np.zeros((1, 2, 6, 7), np.float32)
    assert np.array_equal(orc.resample2d_forward(img, zero), img)            # zero flow = identity
    flow = zero.copy()
    flow[:, 0] = 2.0
    flow[:, 1] = -1.0                                                         # integer flow = shifted copy
    out = orc.resample2d_forward(img, flow)
    ys = np.clip(np.arange(6) - 1, 0, 5)
    xs = np.clip(np.arange(7) + 2, 0, 6)
    assert np.allclose(out, img[:, :, ys][:, :, :, xs])                      # with border replication
    near = orc.resample2d_forward(img, flow + 0.4, bilinear=False)
    assert np.allclose(near, img[:, :, ys][:, :, :, xs])
    # zero flow: flow-gradient = forward differences of the image weighted by grad_output
    go = np.ones_like(img)
    _, gf = orc.resample2d_backward(img, zero, go)
    dx = np.zeros_like(img)
    dx[..., :-1] = img[..., 1:] - img[..., :-1]
    assert np.allclose(gf[0, 0], dx.sum(1)[0], atol=1e-6)


def test_channelnorm_known_answers_and_torch():
    x = np.zeros((1, 3, 1, 2), np.float32)
    x[0, :, 0, 0] = (3, 4, 0)
    out = orc.channelnorm_forward(x)
    assert out.shape == (1, 1, 1, 2) and out[0, 0, 0, 0] == 5.0 and out[0, 0, 0, 1] == 0.0
    gi = orc.channelnorm_backward(x, out, np.ones_like(out))
    assert np.allclose(gi[0, :, 0, 0], (0.6, 0.8, 0.0)) and np.all(gi[0, :, 0, 1] == 0)   # N-1: 0/1e-9 = 0
    t = torch.randn(2, 3, 5, 7, dtype=torch.float64, requires_grad=True)
    ref = tr.channelnorm(t)
    go = torch.randn_like(ref)
    ref.backward(go)
    o = orc.channelnorm_forward(t.detach().numpy())
    assert_close(o, ref.detach().numpy(), 1e-6, "oracle cnorm fwd")
    assert_close(orc.channelnorm_backward(t.detach().numpy(), o, go.numpy()), t.grad.numpy(), 1e-6, "oracle cnorm bwd")


GOLDEN = sorted(p for p in glob.glob(os.path.join(os.path.dirname(__file__), "golden", "*.npz"))
                if not os.path.basename(p).startswith("refk_"))   # refk_*: test_gpu_parity's reference-kernel results


@pytest.mark.parametrize("path", GOLDEN or [None])
def test_oracle_matches_reference_kernel_golden(path):
    """Fixtures = outputs of the REFERENCE kernels (oracle/_ref, rebuilt for sm_90a) run on an H100."""
    if path is None:
        pytest.skip("no golden fixtures committed yet (generate with tests/golden/make_golden.py on a GPU box)")
    z = np.load(path)
    op = str(z["op"])
    if op == "correlation":
        prm = [int(v) for v in z["params"]]
        out = orc.correlation_forward(z["input1"], z["input2"], *prm)
        assert_close(out, z["output"], 1e-5, "golden corr fwd")
        g1, g2 = orc.correlation_backward(z["input1"], z["input2"], z["grad_output"], *prm)
        assert_close(g1, z["grad_input1"], 1e-5, "golden corr gI1")
        assert_close(g2, z["grad_input2"], 1e-5, "golden corr gI2")
    elif op == "resample2d":
        out = orc.resample2d_forward(z["input1"], z["input2"], 1, bool(z["bilinear"]))
        assert_close(out, z["output"], 1e-5, "golden resample fwd")
        g1, g2 = orc.resample2d_backward(z["input1"], z["input2"], z["grad_output"])
        assert_close(g1, z["grad_input1"], 1e-4, "golden resample gImg")   # atomics: order-dependent rounding
        assert_close(g2, z["grad_input2"], 1e-5, "golden resample gFlow")
    elif op == "channelnorm":
        out = orc.channelnorm_forward(z["input1"])
        assert_close(out, z["output"], 1e-6, "golden cnorm fwd")
        assert_close(orc.channelnorm_backward(z["input1"], z["output"], z["grad_output"]), z["grad_input1"], 1e-6,
                     "golden cnorm bwd")
    else:
        raise AssertionError(op)


def test_upsample4_matches_torch_interpolate():
    """orc_upsample4 restates nn.Upsample(scale_factor=4) (models.py:42,56,72-73); pinned against torch on CPU."""
    import torch
    g = torch.Generator().manual_seed(0)
    f = torch.randn(2, 2, 7, 9, generator=g)
    for mode, name, tol in ((1, "bilinear", 1e-6), (2, "nearest", 0.0)):
        ref = torch.nn.Upsample(scale_factor=4, mode=name)(f * 20.0).numpy()
        out = orc.upsample4(f.numpy(), mode, 20.0)
        assert out.shape == ref.shape
        assert np.abs(out - ref).max() <= tol * np.abs(ref).max()
    import pytest
    with pytest.raises(ValueError):
        orc.upsample4(f.numpy(), 3)


def test_warp_concat_compositions_against_fp64_autograd():
    """The oracle's compositions for the fused warp -> diff -> norm -> concat op (forward and backward) against an
    independent fp64 formulation: grid_sample(border, align_corners=True) is Resample2d's bilinear warp for in-range and
    clamped samples alike (SURVEY R-2), the rest is plain torch."""
    import torch
    g = torch.Generator().manual_seed(1)
    x = torch.rand(1, 6, 12, 16, generator=g) - 0.5
    fl = torch.randn(1, 2, 12, 16, generator=g) * 2
    gc = torch.randn(1, 12, 12, 16, generator=g)
    cat = orc.warp_concat_forward(x.numpy(), fl.numpy(), flow_div=20.0)
    rx, rf = orc.warp_concat_backward(x.numpy(), fl.numpy(), gc.numpy(), flow_div=20.0)
    xd, fd = x.double().requires_grad_(), fl.double().requires_grad_()
    H, W = 12, 16
    yy, xx = torch.meshgrid(torch.arange(H).double(), torch.arange(W).double(), indexing="ij")
    gx = (xx + fd[:, 0]) / (W - 1) * 2 - 1
    gy = (yy + fd[:, 1]) / (H - 1) * 2 - 1
    warped = torch.nn.functional.grid_sample(xd[:, 3:], torch.stack((gx, gy), -1), mode="bilinear", padding_mode="border",
                                             align_corners=True)
    diff = xd[:, :3] - warped
    ref = torch.cat((xd, warped, fd / 20.0, diff.pow(2).sum(1, keepdim=True).sqrt()), 1)
    assert np.abs(cat - ref.detach().numpy()).max() < 1e-5
    ref.backward(gc.double())
    assert np.abs(rx - xd.grad.numpy()).max() < 1e-5 * max(1.0, np.abs(rx).max())
    assert np.abs(rf - fd.grad.numpy()).max() < 1e-5 * max(1.0, np.abs(rf).max())
    # the fusion-stage layout: quarter-resolution flow, nearest upsample, flow + its norm + the diff norm
    lr = torch.randn(1, 2, 3, 4, generator=g)
    c3 = orc.warp_concat_forward(x.numpy(), lr.numpy(), upsample_mode=2, flow_mul=0.05, cat_channels=11, ch_x=0, n_x=3,
                                 ch_warped=-1, ch_flow=3, flow_div=1.0, ch_flow_norm=7, ch_diff_norm=9)
    up = torch.nn.Upsample(scale_factor=4, mode="nearest")(lr * 0.05)
    assert np.abs(c3[:, 3:5] - up.numpy()).max() < 1e-7
    assert np.abs(c3[:, 7] - up.pow(2).sum(1).sqrt().numpy()).max() < 1e-6
    assert (c3[:, 5:7] == 0).all() and (c3[:, 8] == 0).all() and (c3[:, 10] == 0).all()
