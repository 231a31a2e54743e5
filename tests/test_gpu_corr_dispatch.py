"""GPU tests of the correlation dispatch.  The plain and *_ws entry points are the *_cat ones with the identity placement
(cat_channels = D, ch_offset = 0, leaky_slope = 1), so on every kernel family they must give the same bits with the same
number of launches; and operands that are not 16-byte aligned must move a tiled-family call onto the generic kernels."""
import ctypes

import pytest
import torch

from oracle import cpu as orc
from util import assert_close

pytestmark = pytest.mark.gpu
P = ctypes.c_void_p
FLOWNETC = (20, 1, 20, 1, 2)

# (shape, (pad, kernel_size, max_displacement, stride1, stride2), family with a workspace, environment)
FAMILIES = {
    "tensor_cores": ((2, 64, 12, 20), FLOWNETC, 2, {}),
    "tiled": ((1, 20, 13, 64), FLOWNETC, 1, {}),
    "generic": ((1, 6, 10, 12), (4, 3, 4, 1, 2), 0, {}),        # kernel_size 3
    "tensor_core_shape_on_fma": ((2, 64, 12, 20), FLOWNETC, 1, {"FN2B200_CORR_FWD": "fma", "FN2B200_CORR_BWD": "fma"}),
}


def _f2():
    import flownet2_b200
    return flownet2_b200


def _randn(shape, seed):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed)).float()


def _ptr(t):
    return P(t.data_ptr()) if t is not None else P(0)


def _launches(call):
    """Kernel launches of one C call, which must succeed."""
    L = _f2()._lib.LIB
    n0 = L.fn2b200_launch_count()
    assert call() == 0, L.fn2b200_last_error()
    return L.fn2b200_launch_count() - n0


def _all_equal(results, names):
    return all(torch.equal(results[names[0]], results[n]) for n in names[1:])


@pytest.mark.parametrize("family", list(FAMILIES))
def test_entry_points_run_the_same_kernels(family, monkeypatch):
    shape, prm, code, env = FAMILIES[family]
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    f = _f2()
    L, F2 = f._lib.LIB, f.functional
    B, C, H, W = shape
    assert L.fn2b200_correlation_path(C, H, W, *prm) == code
    D, oH, oW = F2.correlation_out_shape(C, H, W, *prm)
    a0, b0 = _randn(shape, 1), _randn(shape, 2)
    a, b = a0.cuda(), b0.cuda()
    pa, pb, st = _ptr(a), _ptr(b), P(torch.cuda.current_stream().cuda_stream)
    ws = torch.empty(8 * a.numel(), dtype=torch.uint8, device="cuda")    # hi/lo bf16 copies of both inputs
    pw, nw = _ptr(ws), ws.numel()
    tc = code == 2

    fwd = {
        "plain": lambda o: L.fn2b200_correlation_forward(pa, pb, o, *shape, *prm, 1, st),
        "ws_null": lambda o: L.fn2b200_correlation_forward_ws(pa, pb, o, *shape, *prm, 1, P(0), 0, st),
        "cat_null": lambda o: L.fn2b200_correlation_forward_cat(pa, pb, o, D, 0, 1.0, *shape, *prm, 1, P(0), 0, st),
        "ws": lambda o: L.fn2b200_correlation_forward_ws(pa, pb, o, *shape, *prm, 1, pw, nw, st),
        "cat": lambda o: L.fn2b200_correlation_forward_cat(pa, pb, o, D, 0, 1.0, *shape, *prm, 1, pw, nw, st),
    }
    outs, counts = {}, {}
    for name, call in fwd.items():
        outs[name] = torch.full((B, D, oH, oW), float("nan"), device="cuda")
        counts[name] = _launches(lambda: call(_ptr(outs[name])))
    # without a workspace the tensor-core shape runs on the tiled kernels
    assert counts == {"plain": 1, "ws_null": 1, "cat_null": 1, "ws": 2 if tc else 1, "cat": 2 if tc else 1}
    assert _all_equal(outs, ["plain", "ws_null", "cat_null"]) and _all_equal(outs, ["ws", "cat"])
    assert tc or torch.equal(outs["plain"], outs["ws"])
    ref = orc.correlation_forward(a0.numpy(), b0.numpy(), *prm)
    for name in ("plain", "ws"):
        assert_close(outs[name].cpu().numpy(), ref, 1e-4, "%s forward %s" % (family, name))

    g0 = _randn((B, D, oH, oW), 3)
    g = g0.cuda()
    pg = _ptr(g)
    bwd = {
        "plain": lambda g1, g2: L.fn2b200_correlation_backward(pa, pb, pg, g1, g2, *shape, *prm, 1, st),
        "ws_null": lambda g1, g2: L.fn2b200_correlation_backward_ws(pa, pb, pg, g1, g2, *shape, *prm, 1, P(0), 0, 0, st),
        "cat_null": lambda g1, g2: L.fn2b200_correlation_backward_cat(pa, pb, pg, P(0), D, 0, 1.0, g1, g2, *shape, *prm, 1,
                                                                      P(0), 0, 0, st),
    }
    for split in (0, 1):                 # the forwards above left the split of (a, b) in the workspace
        bwd["ws_split%d" % split] = lambda g1, g2, s=split: L.fn2b200_correlation_backward_ws(
            pa, pb, pg, g1, g2, *shape, *prm, 1, pw, nw, s, st)
        bwd["cat_split%d" % split] = lambda g1, g2, s=split: L.fn2b200_correlation_backward_cat(
            pa, pb, pg, P(0), D, 0, 1.0, g1, g2, *shape, *prm, 1, pw, nw, s, st)
    grads, counts = {}, {}
    for name, call in bwd.items():
        g1, g2 = torch.full_like(a, float("nan")), torch.full_like(b, float("nan"))
        counts[name] = _launches(lambda: call(_ptr(g1), _ptr(g2)))
        grads[name] = torch.cat((g1, g2))
    assert counts == {"plain": 2, "ws_null": 2, "cat_null": 2, "ws_split0": 2, "ws_split1": 1 if tc else 2,
                      "cat_split0": 2, "cat_split1": 1 if tc else 2}
    with_ws = ["ws_split0", "ws_split1", "cat_split0", "cat_split1"]
    assert _all_equal(grads, ["plain", "ws_null", "cat_null"]) and _all_equal(grads, with_ws)
    assert tc or torch.equal(grads["plain"], grads["ws_split0"])
    r1, r2 = orc.correlation_backward(a0.numpy(), b0.numpy(), g0.numpy(), *prm)
    for name in ("plain", "ws_split1"):
        assert_close(grads[name][:B].cpu().numpy(), r1, 1e-4, "%s gI1 %s" % (family, name))
        assert_close(grads[name][B:].cpu().numpy(), r2, 1e-4, "%s gI2 %s" % (family, name))


@pytest.mark.parametrize("family", list(FAMILIES))
def test_correlation_module_launch_counts(family, monkeypatch):
    """The autograd module hands the forward's workspace to its backward: 2 + 1 launches on tensor cores."""
    shape, prm, code, env = FAMILIES[family]
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    f = _f2()
    a, b = (_randn(shape, s).cuda().requires_grad_() for s in (4, 5))
    n0 = f.functional.launch_count()
    out = f.Correlation(*prm, 1)(a, b)
    n1 = f.functional.launch_count()
    out.backward(_randn(tuple(out.shape), 6).cuda())
    n2 = f.functional.launch_count()
    assert (n1 - n0, n2 - n1) == ((2, 1) if code == 2 else (1, 2))


def _misaligned(t):
    """A contiguous copy of t that starts one element (4 bytes) past a 16-byte boundary."""
    v = torch.empty(t.numel() + 1, device="cuda")[1:].view(t.shape)
    v.copy_(t)
    assert v.is_contiguous() and v.data_ptr() % 16 == 4
    return v


def test_misaligned_operands_run_the_generic_kernels():
    """A tiled-family shape with 4-byte aligned inputs and gradOutput: the generic kernels run (the tiled ones would
    fail to encode their tensor maps).  Outputs stay aligned."""
    f = _f2()
    shape, prm = FAMILIES["tiled"][:2]
    assert f._lib.LIB.fn2b200_correlation_path(*shape[1:], *prm) == 1
    a0, b0 = _randn(shape, 7), _randn(shape, 8)
    a, b = _misaligned(a0.cuda()), _misaligned(b0.cuda())
    n0 = f.functional.launch_count()
    out = f.functional.correlation_forward(a, b, *prm)
    n1 = f.functional.launch_count()
    assert n1 - n0 == 1
    assert_close(out.cpu().numpy(), orc.correlation_forward(a0.numpy(), b0.numpy(), *prm), 1e-4, "misaligned forward")
    g0 = _randn(tuple(out.shape), 9)
    g1, g2 = f.functional.correlation_backward(a, b, _misaligned(g0.cuda()), *prm)
    assert f.functional.launch_count() - n1 == 2
    r1, r2 = orc.correlation_backward(a0.numpy(), b0.numpy(), g0.numpy(), *prm)
    assert_close(g1.cpu().numpy(), r1, 1e-4, "misaligned gI1")
    assert_close(g2.cpu().numpy(), r2, 1e-4, "misaligned gI2")
