"""Every route into libfn2b200 refuses the same bad operands with the same message, before anything is launched.

Four routes reach the C ABI: ``functional``, the B1 shim modules (Python ``*_cuda`` modules over ``functional``), the
B1p modules (the compiled ``*_cuda`` extension modules) and the ``torch.ops.fn2b200`` operators.  All of them go through
one host-side check per op (pybind/ext_common.h), so an operand the kernels would overrun -- a batch smaller than the
flow's, an output or gradient of the wrong shape, dtype or layout, an empty correlation output -- raises RuntimeError
with one message whichever route it arrives by, and ``functional.launch_count()`` does not move.

Each too-small operand is carved out of a larger allocation (``_carve``): a route that trusted the larger shape would
still stay inside allocated memory.  The B1p modules run in a child process (tests/pybind_child.py refusals) because
pybind11 caches extension modules by name.
"""
import json
import math
import os
import subprocess
import sys

import pytest
import torch

from flownet2_b200 import functional as F2

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
B, C, H, W = 2, 3, 8, 8
PRM = (4, 1, 4, 1, 1)                  # D = 81, oH = oW = 8 on an 8 x 8 input
EMPTY = (0, 1, 4, 1, 1)                # oH = oW = 0 on an 8 x 8 input


def _randn(*shape):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(sum(shape))).cuda()


def _carve(shape, full):
    """A contiguous tensor of `shape` at the start of an allocation of `full`'s size."""
    return _randn(*full).view(-1)[:math.prod(shape)].view(shape)


def _cases(cc, rs, cn):
    """name -> (a substring of the message, {route: thunk}); "ext" is the route of the *_cuda modules cc, rs, cn."""
    fn = torch.ops.fn2b200
    img, flow, go, inp = _randn(B, C, H, W), _randn(B, 2, H, W), _randn(B, C, H, W), _randn(B, C, H, W)
    nrm, gn = _randn(B, 1, H, W), _randn(B, 1, H, W)
    small_img, small_nrm = _carve((1, C, H, W), (B, C, H, W)), _carve((1, 1, H, W), (B, 1, H, W))
    small_x, gcat = _carve((1, 2 * C, H, W), (B, 2 * C, H, W)), _randn(B, 12, H, W)
    a, b = _randn(1, 16, H, W), _randn(1, 16, H, W)
    small_go = _carve((1, 80, H, W), (1, 81, H, W))
    layout = (0, 6, 6, 9, -1, 11)
    e = lambda: img.new()  # noqa: E731  (the reference's empty out-parameters)
    return {
        # operands no route but the operator checked before
        "warp_concat_forward x batch": ("expected x", {
            "functional": lambda: F2.warp_concat_forward(small_x, flow),
            "op": lambda: fn.warp_concat_forward(small_x, flow, C, 0, 1.0, 1.0, 12, *layout)}),
        "warp_concat_backward x batch": ("expected x", {
            "functional": lambda: F2.warp_concat_backward(small_x, flow, gcat, need_x=False),
            "op": lambda: fn.warp_concat_backward(small_x, flow, gcat, C, 0, 1.0, 1.0, *layout, False, True)}),
        "channelnorm_backward output": ("do not match", {
            "functional": lambda: F2.channelnorm_backward(inp, small_nrm, small_nrm),
            "ext": lambda: cn.backward(inp, small_nrm, small_nrm, torch.empty_like(inp), 2),
            "op": lambda: fn.channelnorm_backward(inp, small_nrm, small_nrm, 2)}),
        "channelnorm_backward grad_output": ("do not match", {
            "functional": lambda: F2.channelnorm_backward(inp, nrm, small_nrm),
            "ext": lambda: cn.backward(inp, nrm, small_nrm, torch.empty_like(inp), 2),
            "op": lambda: fn.channelnorm_backward(inp, nrm, small_nrm, 2)}),
        "channelnorm_backward grad_input1": ("grad_input1 must be", {
            "functional": lambda: F2.channelnorm_backward(inp, nrm, gn, out=small_img),
            "ext": lambda: cn.backward(inp, nrm, gn, small_img, 2)}),
        "channelnorm_forward output": ("output must be", {
            "functional": lambda: F2.channelnorm_forward(inp, out=_carve((B, 1, H, W - 1), (B, 1, H, W))),
            "ext": lambda: cn.forward(inp, _carve((B, 1, H, W - 1), (B, 1, H, W)), 2)}),
        "resample2d_forward image batch": ("smaller than flow batch", {
            "functional": lambda: F2.resample2d_forward(small_img, flow, out=torch.empty_like(img)),
            "ext": lambda: rs.forward(small_img, flow, torch.empty_like(img), 1, True),
            "op": lambda: fn.resample2d_forward(small_img, flow, 1, True)}),
        "resample2d_backward image batch": ("smaller than flow batch", {
            "functional": lambda: F2.resample2d_backward(small_img, flow, go, out1=_carve((1, C, H, W), (B, C, H, W)),
                                                         out2=torch.empty_like(flow)),
            "ext": lambda: rs.backward(small_img, flow, go, _carve((1, C, H, W), (B, C, H, W)), torch.empty_like(flow), 1,
                                       True),
            "op": lambda: fn.resample2d_backward(small_img, flow, go, 1, True, False, True)}),
        "resample2d_backward grad_output": ("grad_output shape", {
            "functional": lambda: F2.resample2d_backward(img, flow, _carve((B, 2, H, W), (B, C, H, W))),
            "ext": lambda: rs.backward(img, flow, _carve((B, 2, H, W), (B, C, H, W)), torch.zeros_like(img),
                                       torch.empty_like(flow), 1, True),
            "op": lambda: fn.resample2d_backward(img, flow, _carve((B, 2, H, W), (B, C, H, W)), 1, True, True, True)}),
        "resample2d_backward grad_input1": ("grad_input1 must be", {
            "functional": lambda: F2.resample2d_backward(img, flow, go, out1=small_img, out2=torch.empty_like(flow)),
            "ext": lambda: rs.backward(img, flow, go, small_img, torch.empty_like(flow), 1, True)}),
        "resample2d_backward grad_input2": ("grad_input2 must be", {
            "functional": lambda: F2.resample2d_backward(img, flow, go, out2=_carve((1, 2, H, W), (B, 2, H, W))),
            "ext": lambda: rs.backward(img, flow, go, torch.zeros_like(img), _carve((1, 2, H, W), (B, 2, H, W)), 1, True)}),
        "correlation_backward grad_output": ("grad_output shape", {
            "functional": lambda: F2.correlation_backward(a, b, small_go, *PRM),
            "ext": lambda: cc.backward(a, b, e(), e(), small_go, e(), e(), *PRM, 1),
            "op": lambda: fn.correlation_backward(a, b, small_go, a.new_empty(0, dtype=torch.uint8), *PRM, 1, True, True)}),
        # one case of each refusal every route already made
        "out shape": ("output must be", {
            "functional": lambda: F2.resample2d_forward(img, flow, out=_carve((B, 2, H, W), (B, C, H, W))),
            "ext": lambda: rs.forward(img, flow, _carve((B, 2, H, W), (B, C, H, W)), 1, True)}),
        "out dtype": ("output must be", {
            "functional": lambda: F2.channelnorm_forward(inp, out=nrm.half()),
            "ext": lambda: cn.forward(inp, nrm.half(), 2)}),
        "out contiguity": ("grad_input2 must be", {
            "functional": lambda: F2.resample2d_backward(img, flow, go, out2=_randn(B, 2, H, 2 * W)[..., ::2]),
            "ext": lambda: rs.backward(img, flow, go, torch.zeros_like(img), _randn(B, 2, H, 2 * W)[..., ::2], 1, True)}),
        "empty correlation output": ("empty output", {
            "functional": lambda: F2.correlation_forward(a, b, *EMPTY),
            "ext": lambda: cc.forward(a, b, e(), e(), e(), *EMPTY, 1),
            "op": lambda: fn.correlation_forward(a, b, *EMPTY, 1)}),
    }


NAMES = ("warp_concat_forward x batch", "warp_concat_backward x batch", "channelnorm_backward output",
         "channelnorm_backward grad_output", "channelnorm_backward grad_input1", "channelnorm_forward output",
         "resample2d_forward image batch", "resample2d_backward image batch", "resample2d_backward grad_output",
         "resample2d_backward grad_input1", "resample2d_backward grad_input2", "correlation_backward grad_output",
         "out shape", "out dtype", "out contiguity", "empty correlation output")


def refusal(thunk):
    """(first line of the RuntimeError's message or None when the call went through, launches it issued)."""
    n0 = F2.launch_count()
    try:
        thunk()
        msg = None
    except RuntimeError as err:
        msg = str(err).splitlines()[0]
    torch.cuda.synchronize()
    return msg, F2.launch_count() - n0


def ext_refusals(cc, rs, cn):
    """What the "ext" route of every case gives with the modules cc, rs, cn: name -> (message, launches)."""
    return {name: refusal(routes["ext"]) for name, (_, routes) in _cases(cc, rs, cn).items() if "ext" in routes}


@pytest.fixture(scope="module")
def b1p():
    r = subprocess.run([sys.executable, os.path.join(HERE, "pybind_child.py"), "refusals"], capture_output=True,
                       text=True, timeout=900)
    assert r.returncode == 0, (r.stdout[-2000:], r.stderr[-4000:])
    return json.loads(r.stdout.splitlines()[-1])


def test_case_list_is_complete():
    from flownet2_b200.shims import channelnorm_cuda, correlation_cuda, resample2d_cuda
    assert tuple(_cases(correlation_cuda, resample2d_cuda, channelnorm_cuda)) == NAMES


@pytest.mark.parametrize("name", NAMES)
def test_every_route_refuses_with_one_message(name, b1p):
    from flownet2_b200.shims import channelnorm_cuda, correlation_cuda, resample2d_cuda
    expect, routes = _cases(correlation_cuda, resample2d_cuda, channelnorm_cuda)[name]
    got = {("B1" if route == "ext" else route): refusal(thunk) for route, thunk in routes.items()}
    if "ext" in routes:
        got["B1p"] = tuple(b1p[name])
    msgs = {route: msg for route, (msg, _) in got.items()}
    assert all(msg is not None and expect in msg for msg in msgs.values()), msgs
    assert len(set(msgs.values())) == 1, msgs
    assert all(n == 0 for _, n in got.values()), got
