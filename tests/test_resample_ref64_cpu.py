"""tests/resample_ref64.py pinned without a GPU: against the CPU oracle (oracle/oracle.c) and the stored results of the
reference's own kernels within the fp32 bound, against fp64 autograd through grid_sample where the semantics agree, and
against answers worked out by hand at the edges."""
import os

import numpy as np
import pytest
import torch

import resample_ref64 as r64
import torch_ref
import upsample_ref
from oracle import cpu as orc

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _within(x, ref, E, what):
    """|x - ref| <= E + r64.ETA element by element (ETA: the absolute error of roundings into the subnormal range)."""
    d = (torch.as_tensor(np.asarray(x, np.float64)) - ref).abs()
    bad = d > E + r64.ETA
    assert not bool(bad.any()), "%s: %d elements beyond the bound; the first at %s: |d| = %.3e, bound %.3e" % (
        what, int(bad.sum()), tuple(int(v) for v in bad.nonzero()[0]), float(d[bad].max()), float(E[bad].max()))


def _fp32_bounds(img, flow, gout):
    """The reference computation's own fp32 rounding: forward 4 products rounded from fp64 and summed in fp32 (8
    roundings); K7 C channels of 4 products each, added one by one in fp32 (<= 4 + 4 C roundings per term); K6 one
    product of three roundings per contribution, atomics in any order."""
    C = img.shape[1]
    f, S = r64.forward(img, flow)
    b = r64.backward(img, flow, gout)
    return (f, r64.gamma(8) * S), (b["gflow"], r64.gamma(4 * C + 6) * b["S_K7"]), \
        (b["gimg"], r64.gamma(b["n_K6"] + 4) * b["S_K6"])


@pytest.mark.parametrize("C,B,H,W,iB,iH,iW,edges", [
    (3, 2, 12, 16, 2, 12, 16, False), (1, 2, 9, 33, 3, 13, 40, True), (2, 1, 1, 31, 1, 3, 32, True),
    (3, 2, 17, 1, 2, 20, 4, True), (5, 2, 8, 9, 3, 11, 12, True)])
def test_matches_oracle(C, B, H, W, iB, iH, iW, edges):
    """Forward (bilinear and nearest), K7 and K6 against the oracle, random and edge flows, image larger than the
    flow in its dims and its batch."""
    img = torch.rand(iB, C, iH, iW, generator=torch.Generator().manual_seed(C + H)) - 0.5
    if edges:
        flow, where = r64.edge_flow(B, H, W, 10 * C + W)
        assert sum(int(m.sum()) for m in where.values()) > 0
    else:
        flow = torch.randn(B, 2, H, W, generator=torch.Generator().manual_seed(3)) * 4
    gout = torch.randn(B, C, H, W, generator=torch.Generator().manual_seed(4))
    (f, Ef), (gf, Egf), (gi, Egi) = _fp32_bounds(img, flow, gout)
    _within(orc.resample2d_forward(img.numpy(), flow.numpy()), f, Ef, "forward")
    n, _ = r64.forward(img, flow, bilinear=False)
    assert np.array_equal(orc.resample2d_forward(img.numpy(), flow.numpy(), bilinear=False), n.float().numpy())
    ogi, ogf = orc.resample2d_backward(img.numpy(), flow.numpy(), gout.numpy())
    _within(ogf, gf, Egf, "K7")
    _within(ogi[:B], gi, Egi, "K6")
    assert (ogi[B:] == 0).all()


@pytest.mark.parametrize("name", ["resample2d_sigma4", "resample2d_sigma40", "resample2d_nearest"])
def test_matches_reference_kernel_golden(name):
    z = np.load(os.path.join(GOLDEN, name + ".npz"))
    img, flow, go = (torch.from_numpy(z[k]) for k in ("input1", "input2", "grad_output"))
    (f, Ef), (gf, Egf), (gi, Egi) = _fp32_bounds(img, flow, go)
    if bool(z["bilinear"]):
        _within(z["output"], f, Ef, name + " forward")
    else:
        assert np.array_equal(z["output"], r64.forward(img, flow, bilinear=False)[0].float().numpy())
    _within(z["grad_input2"], gf, Egf, name + " K7")
    _within(z["grad_input1"], gi, Egi, name + " K6")


def test_matches_reference_kernel_golden_refk():
    """refk_resample_channelnorm.npz: the reference kernels on the inputs of seed 44 (tests/golden/make_golden.py)."""
    z = np.load(os.path.join(GOLDEN, "refk_resample_channelnorm.npz"))
    g = torch.Generator().manual_seed(44)
    img = torch.rand(2, 3, 32, 48, generator=g)
    flow = torch.randn(2, 2, 32, 48, generator=g) * 6
    go = torch.randn(2, 3, 32, 48, generator=g)
    (f, Ef), (gf, Egf), (gi, Egi) = _fp32_bounds(img, flow, go)
    _within(z["resample_output"], f, Ef, "forward")
    _within(z["resample_grad_flow"], gf, Egf, "K7")
    _within(z["resample_grad_img"], gi, Egi, "K6")


def test_matches_grid_sample_autograd():
    """Same-size image: the forward and K7 equal fp64 autograd through grid_sample(border, align_corners=True).  The
    flows are multiples of 2^-10, so x + dx is exact in fp32 and fp64 alike.  The flow gradient at integer coordinates
    is left out: grid_sample's normalise / unnormalise round trip can move an integer by an ulp to the other side of the
    kink, and at 0 its clamp zeroes the gradient (test_known_answers pins K7's one-sided difference there)."""
    B, C, H, W = 2, 3, 11, 14
    img = torch.rand(B, C, H, W, generator=torch.Generator().manual_seed(5)).double()
    flow = torch.round(torch.randn(B, 2, H, W, generator=torch.Generator().manual_seed(6)) * 4 * 1024) / 1024
    gout = torch.randn(B, C, H, W, generator=torch.Generator().manual_seed(7)).double()
    fl = flow.double().requires_grad_()
    out = torch_ref.resample2d(img, fl)
    out.backward(gout)
    ref, _ = r64.forward(img, flow)
    assert torch.allclose(out.detach(), ref, rtol=0, atol=1e-13)
    xf, yf = r64.coords(flow)
    keep = ((xf != torch.floor(xf)) & (yf != torch.floor(yf))).unsqueeze(1).expand(B, 2, H, W)
    gf = r64.backward(img, flow, gout)["gflow"]
    assert torch.allclose(fl.grad[keep], gf[keep], rtol=0, atol=1e-12)


def test_known_answers():
    """By hand, on I[y, x] = 100 y + x (4 x 6, image 6 x 9): an integer shift, the nearest tie, 0.49999997f, a bilinear
    point, and the clamps on all four sides (with the FLOW's dims, not the larger image's)."""
    H, W = 4, 6
    img = (100 * torch.arange(6.0).view(6, 1) + torch.arange(9.0).view(1, 9)).view(1, 1, 6, 9)
    flow = torch.zeros(1, 2, H, W)
    flow[0, 0, 0, 0], flow[0, 1, 0, 0] = 2.0, 1.0                  # integer shift -> I[1, 2]
    flow[0, 0, 0, 1] = 1.5                                         # xf = 2.5: nearest -> 3 (half up)
    flow[0, 0, 3, 0] = torch.nextafter(torch.tensor(0.5), torch.tensor(0.0))   # xf = 0.49999997: nearest -> 0
    flow[0, 0, 1, 1], flow[0, 1, 1, 1] = 0.25, 0.5                 # bilinear (1.25, 1.5) -> 151.25
    flow[0, 0, 2, 2] = -50.0                                       # left: x -> 0
    flow[0, 0, 2, 3] = 50.0                                        # right: x -> W-1 = 5, not iW-1 = 8
    flow[0, 1, 3, 4] = 50.0                                        # bottom: y -> H-1 = 3
    flow[0, 1, 0, 5] = -50.0                                       # top: y -> 0
    out, _ = r64.forward(img, flow)
    near, _ = r64.forward(img, flow, bilinear=False)
    o, n = out[0, 0], near[0, 0]
    assert o[0, 0] == 102 and n[0, 0] == 102
    assert n[0, 1] == 3 and o[0, 1] == 2.5
    assert n[3, 0] == 300                                          # fp32 xf + 0.5f would round to 1: 301
    assert abs(float(o[1, 1]) - 151.25) < 1e-12
    assert o[2, 2] == 200 and o[2, 3] == 205 and o[3, 4] == 304 and o[0, 5] == 5
    # the oracle agrees at every one of these points
    assert np.array_equal(orc.resample2d_forward(img.numpy(), flow.numpy(), bilinear=False), near.float().numpy())
    assert np.allclose(orc.resample2d_forward(img.numpy(), flow.numpy()), out.numpy(), rtol=0, atol=1e-4)
    # K7 at an integer coordinate takes the right difference; at a right clamp it is 0
    g = r64.backward(img, flow, torch.ones(1, 1, H, W))["gflow"][0]
    assert g[0, 0, 0] == 1 and g[1, 0, 0] == 100
    assert g[0, 2, 3] == 0 and g[1, 3, 4] == 0


def test_k6_truncation_equals_floor():
    """For finite |xf| < 2^31, K6's truncation-based fractions scatter the same as floor-based ones: where trunc !=
    floor (xf negative and not an integer) both taps of that axis clamp to column (row) 0, and the two weights of one
    axis add up to 1 either way."""
    B, C, H, W = 2, 2, 7, 9
    flow, _ = r64.edge_flow(B, H, W, 77, sigma=6.0)
    flow[0, :, 0] = -torch.rand(2, W, generator=torch.Generator().manual_seed(8)) * 2 ** 30
    img = torch.rand(B, C, H + 2, W + 3, generator=torch.Generator().manual_seed(9))
    gout = torch.randn(B, C, H, W, generator=torch.Generator().manual_seed(10))
    a = r64.backward(img, flow, gout)
    b = r64.backward(img, flow, gout, variant="k6_floor")
    assert torch.allclose(a["gimg"], b["gimg"], rtol=1e-12, atol=1e-12)
    xf, yf = r64.coords(flow)
    xL, xR, yT, yB = r64.floor_taps(xf, yf, W + 3, H + 2)
    neg = torch.trunc(xf) != torch.floor(xf)
    assert bool(neg.any()) and bool((xL[neg] == 0).all()) and bool((xR[neg] == 0).all())
    neg = torch.trunc(yf) != torch.floor(yf)
    assert bool(neg.any()) and bool((yT[neg] == 0).all()) and bool((yB[neg] == 0).all())


@pytest.mark.parametrize("mode", [1, 2])
def test_upsample_flow32(mode):
    """The fp32 restatement of load_flow's upsample equals the oracle's nn.Upsample restatement within a few ulp and
    reads every cell the fp64 interpolation matrices read."""
    lr = torch.randn(2, 2, 3, 5, generator=torch.Generator().manual_seed(11)) * 3
    up = r64.upsample_flow32(lr, mode, 20.0)
    ref = orc.upsample4(lr.numpy(), mode, 20.0)
    assert np.allclose(up.numpy(), ref, rtol=4 * 2.0 ** -24, atol=0)
    A = torch.from_numpy(upsample_ref.upsample4_matrix(3, mode))
    Bm = torch.from_numpy(upsample_ref.upsample4_matrix(5, mode))
    r64x = 20.0 * torch.einsum("yi,bcij,xj->bcyx", A, lr.double(), Bm)
    assert torch.allclose(up.double(), r64x, rtol=1e-6, atol=1e-5)


def test_warp_concat_chain_matches_oracle():
    """The fused chain's forward and backward against the oracle's composition of the reference's modules."""
    C, B, fh, fw, mul = 3, 2, 3, 5, 20.0
    H, W = 4 * fh, 4 * fw
    x = torch.rand(B, 2 * C, H, W, generator=torch.Generator().manual_seed(12)) - 0.5
    lr = torch.randn(B, 2, fh, fw, generator=torch.Generator().manual_seed(13)) * 0.2
    lay = r64.layout(C, flow_div=20.0)
    gcat = torch.randn(B, lay["cat_channels"], H, W, generator=torch.Generator().manual_seed(14))
    f32 = r64.upsample_flow32(lr, 1, mul)
    cat, _ = r64.warp_concat_forward(x, f32, C, lay)
    ocat = orc.warp_concat_forward(x.numpy(), lr.numpy(), C=C, upsample_mode=1, flow_mul=mul, flow_div=20.0)
    assert np.allclose(ocat, cat.numpy(), rtol=0, atol=1e-5 * float(cat.abs().max()))
    kw = {k: v for k, v in lay.items() if k != "cat_channels"}
    ogx, ogf = upsample_ref.warp_concat_backward(x.numpy(), lr.numpy(), gcat.numpy(), C=C, upsample_mode=1,
                                                 flow_mul=mul, **kw)
    r = r64.warp_concat_backward(x, f32, gcat, C, lay, mode=1, mul=mul)
    assert np.allclose(ogx, r["gx"].numpy(), rtol=0, atol=1e-5 * float(r["gx"].abs().max()))
    assert np.allclose(ogf, r["gflow"].numpy(), rtol=0, atol=1e-5 * float(r["gflow"].abs().max()))
