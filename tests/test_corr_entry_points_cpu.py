"""CPU tests of the six correlation entry points: the plain and *_ws forms are the *_cat form with the identity placement
(cat_channels = D, ch_offset = 0, leaky_slope = 1), so every invalid call must fail the same way in all of them, with
the same message after the entry point's prefix, before anything touches the device."""
import ctypes

import pytest

P = ctypes.c_void_p
ONE = P(16)                          # never dereferenced: validation fails (or the call is a no-op) first
FLOWNETC = (20, 1, 20, 1, 2)         # pad, kernel_size, max_displacement, stride1, stride2 -> D = 441
WORKSPACES = [(P(0), 0), (P(256), 1 << 40)]   # none, and one large enough for the tensor cores


def _lib():
    from flownet2_b200._lib import LIB
    return LIB


def _depth(C, H, W, prm):
    D, oH, oW = ctypes.c_int(), ctypes.c_int(), ctypes.c_int()
    rc = _lib().fn2b200_correlation_out_shape(C, H, W, *prm, ctypes.byref(D), ctypes.byref(oH), ctypes.byref(oW))
    return D.value if rc == 0 else 1     # bad parameters: validation fails before the channel count matters


def _forward_forms(in1, in2, out, shape, prm):
    """(form, call) for the plain, *_ws and identity *_cat forwards."""
    L, D = _lib(), _depth(*shape[1:], prm)
    yield "plain", lambda: L.fn2b200_correlation_forward(in1, in2, out, *shape, *prm, 1, P(0))
    for ws, n in WORKSPACES:
        yield "ws", lambda ws=ws, n=n: L.fn2b200_correlation_forward_ws(in1, in2, out, *shape, *prm, 1, ws, n, P(0))
        yield "cat", lambda ws=ws, n=n: L.fn2b200_correlation_forward_cat(in1, in2, out, D, 0, 1.0, *shape, *prm, 1, ws, n,
                                                                          P(0))


def _backward_forms(in1, in2, gout, g1, g2, shape, prm):
    L, D = _lib(), _depth(*shape[1:], prm)
    yield "plain", lambda: L.fn2b200_correlation_backward(in1, in2, gout, g1, g2, *shape, *prm, 1, P(0))
    for ws, n in WORKSPACES:
        for split in (0, 1):
            yield "ws", lambda ws=ws, n=n, s=split: L.fn2b200_correlation_backward_ws(in1, in2, gout, g1, g2, *shape, *prm, 1,
                                                                                      ws, n, s, P(0))
            yield "cat", lambda ws=ws, n=n, s=split: L.fn2b200_correlation_backward_cat(in1, in2, gout, P(0), D, 0, 1.0, g1, g2,
                                                                                        *shape, *prm, 1, ws, n, s, P(0))


# (case, [B, C, H, W], (pad, kernel_size, max_displacement, stride1, stride2), directions, expected code)
INVALID = [
    ("negative batch", (-1, 4, 8, 8), FLOWNETC, "fb", -1),
    ("no channels", (1, 0, 8, 8), FLOWNETC, "fb", -1),
    ("no width", (1, 4, 8, 0), FLOWNETC, "fb", -1),
    ("negative pad", (1, 4, 8, 8), (-1, 1, 4, 1, 2), "fb", -1),
    ("kernel_size 0", (1, 4, 8, 8), (4, 0, 4, 1, 2), "fb", -1),
    ("stride2 0", (1, 4, 8, 8), (4, 1, 4, 1, 0), "fb", -1),
    ("empty output", (1, 4, 8, 8), (0, 1, 20, 1, 2), "fb", -1),
    ("input of 2^31 elements", (2048, 1024, 32, 32), (0, 1, 0, 1, 1), "fb", -1),
    ("output of 2^31 elements", (4096, 1, 40, 40), FLOWNETC, "fb", -1),
    ("stride1 2", (1, 4, 12, 13), (2, 1, 4, 2, 2), "b", -2),
]
NULLS = ["input1", "input2", "output"]


def _same_failure(forms, code, prefixes):
    L = _lib()
    rest = set()
    for form, call in forms:
        assert call() == code, form
        prefix, _, msg = L.fn2b200_last_error().decode().partition(": ")
        assert prefix in prefixes[form], (form, prefix)
        rest.add(msg)
    assert len(rest) == 1, rest
    return rest.pop()


FWD_PREFIXES = {"plain": ("correlation", "correlation_forward"), "ws": ("correlation", "correlation_forward"),
                "cat": ("correlation", "correlation_forward_cat")}
BWD_PREFIXES = {"plain": ("correlation", "correlation_backward"), "ws": ("correlation", "correlation_backward"),
                "cat": ("correlation", "correlation_backward_cat")}


@pytest.mark.parametrize("case,shape,prm,directions,code", INVALID, ids=[c[0] for c in INVALID])
def test_invalid_call_fails_alike_in_every_form(case, shape, prm, directions, code):
    if "f" in directions:
        _same_failure(_forward_forms(ONE, ONE, ONE, shape, prm), code, FWD_PREFIXES)
    msg = _same_failure(_backward_forms(ONE, ONE, ONE, ONE, ONE, shape, prm), code, BWD_PREFIXES)
    if case == "stride1 2":
        assert "stride1=2 unsupported" in msg


@pytest.mark.parametrize("which", NULLS)
def test_null_pointer_fails_alike_in_every_form(which):
    shape = (1, 64, 8, 8)
    ptrs = [P(0) if name == which else ONE for name in NULLS]
    assert _same_failure(_forward_forms(*ptrs, shape, FLOWNETC), -3, FWD_PREFIXES) == "null pointer"
    # backward: the third pointer is gradOutput
    assert _same_failure(_backward_forms(*ptrs, ONE, ONE, shape, FLOWNETC), -3, BWD_PREFIXES) == "null pointer"


def test_no_op_calls_return_before_touching_the_device():
    L = _lib()
    # B == 0, every pointer NULL
    empty = (0, 64, 8, 8)
    for form, call in list(_forward_forms(P(0), P(0), P(0), empty, FLOWNETC)) + list(
            _backward_forms(P(0), P(0), P(0), P(0), P(0), empty, FLOWNETC)):
        assert call() == 0, form
    # no gradient wanted: non-null inputs, both gradient pointers NULL (on a machine without a GPU, binding the device
    # would fail)
    for form, call in _backward_forms(ONE, ONE, ONE, P(0), P(0), (1, 64, 8, 8), FLOWNETC):
        assert call() == 0, form
    assert L.fn2b200_correlation_backward_cat(ONE, ONE, ONE, ONE, 473, 32, 0.1, P(0), P(0), 1, 64, 8, 8, *FLOWNETC, 1,
                                              P(0), 0, 0, P(0)) == 0
