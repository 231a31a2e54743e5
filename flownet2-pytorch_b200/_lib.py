"""The two native libraries: ``LIB``, the ctypes binding of libfn2b200.so (the C ABI declared in include/fn2b200.h,
used here for its scalar queries and by the tests of the C ABI), and ``OPS``, the operator library built from
pybind/fn2b200_ops.cc (torch.ops.fn2b200.* and the host-side glue of every op).

There is NO fallback: if a shared object is missing the import fails loudly, and every entry
point refuses non-CUDA tensors.  ``FN2B200_AUTOBUILD=1`` (default when nvcc is present) compiles the
libraries in-tree on first import.
"""
import ctypes
import importlib.util
import os
import sysconfig

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libfn2b200.so")

_c_int = ctypes.c_int
_c_ptr = ctypes.c_void_p


class Fn2B200Error(RuntimeError):
    """A libfn2b200 entry point returned a non-zero status (mirrors the reference's AT_ERROR)."""


def _run_build(script):
    spec = importlib.util.spec_from_file_location("_fn2b200_build", script)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    mod.build()


def _load():
    if not os.path.isfile(LIB_PATH):
        if os.environ.get("FN2B200_AUTOBUILD", "1") == "1":
            _run_build(os.path.join(_HERE, "build.py"))
        if not os.path.isfile(LIB_PATH):
            raise ImportError(
                "libfn2b200.so not found at %s -- build it with `python flownet2-pytorch_b200/build.py` "
                "(needs nvcc, sm_90a). There is no CPU/PyTorch fallback." % LIB_PATH)
    lib = ctypes.CDLL(LIB_PATH)
    lib.fn2b200_version.restype = _c_int
    lib.fn2b200_last_error.restype = ctypes.c_char_p
    lib.fn2b200_launch_count.restype = ctypes.c_uint64
    ip = ctypes.POINTER(_c_int)
    lp = ctypes.POINTER(ctypes.c_int64)
    lib.fn2b200_correlation_out_shape.argtypes = [_c_int] * 8 + [ip, ip, ip]
    lib.fn2b200_correlation_path.argtypes = [_c_int] * 8
    lib.fn2b200_correlation_forward.argtypes = [_c_ptr] * 3 + [_c_int] * 10 + [_c_ptr]
    lib.fn2b200_correlation_backward.argtypes = [_c_ptr] * 5 + [_c_int] * 10 + [_c_ptr]
    lib.fn2b200_correlation_forward_workspace.argtypes = [_c_int] * 9
    lib.fn2b200_correlation_forward_workspace.restype = ctypes.c_size_t
    lib.fn2b200_correlation_forward_ws.argtypes = [_c_ptr] * 3 + [_c_int] * 10 + [_c_ptr, ctypes.c_size_t, _c_ptr]
    lib.fn2b200_correlation_forward_ws.restype = _c_int
    lib.fn2b200_correlation_forward_cat.argtypes = ([_c_ptr] * 3 + [_c_int, _c_int, ctypes.c_float] + [_c_int] * 10
                                                    + [_c_ptr, ctypes.c_size_t, _c_ptr])
    lib.fn2b200_correlation_forward_cat.restype = _c_int
    lib.fn2b200_correlation_backward_workspace.argtypes = [_c_int] * 9
    lib.fn2b200_correlation_backward_workspace.restype = ctypes.c_size_t
    lib.fn2b200_correlation_backward_ws.argtypes = ([_c_ptr] * 5 + [_c_int] * 10 + [_c_ptr, ctypes.c_size_t, _c_int, _c_ptr])
    lib.fn2b200_correlation_backward_ws.restype = _c_int
    lib.fn2b200_correlation_backward_cat.argtypes = ([_c_ptr] * 4 + [_c_int, _c_int, ctypes.c_float] + [_c_ptr] * 2
                                                     + [_c_int] * 10 + [_c_ptr, ctypes.c_size_t, _c_int, _c_ptr])
    lib.fn2b200_correlation_backward_cat.restype = _c_int
    lib.fn2b200_resample2d_forward.argtypes = [_c_ptr, lp, _c_ptr, _c_ptr] + [_c_int] * 8 + [_c_ptr]
    lib.fn2b200_resample2d_forward_up.argtypes = [_c_ptr, lp, _c_ptr, _c_int, _c_int, _c_int, ctypes.c_float, _c_ptr] + [_c_int] * 4 + [_c_ptr]
    lib.fn2b200_resample2d_forward_up.restype = _c_int
    lib.fn2b200_warp_concat_forward.argtypes = ([_c_ptr, lp, _c_int, _c_ptr, _c_int, _c_int, _c_int, ctypes.c_float, _c_ptr]
                                                + [_c_int] * 5 + [ctypes.c_float] + [_c_int] * 5 + [_c_ptr])
    lib.fn2b200_warp_concat_forward.restype = _c_int
    lib.fn2b200_warp_concat_backward_workspace.argtypes = [_c_int] * 4
    lib.fn2b200_warp_concat_backward_workspace.restype = ctypes.c_size_t
    lib.fn2b200_warp_concat_backward.argtypes = ([_c_ptr, lp, _c_int, _c_ptr, _c_ptr] + [_c_int] * 5 + [ctypes.c_float] + [_c_int] * 2
                                                 + [_c_ptr, _c_ptr, _c_ptr, ctypes.c_size_t] + [_c_int] * 3 + [_c_ptr])
    lib.fn2b200_warp_concat_backward.restype = _c_int
    lib.fn2b200_warp_concat_backward_up_workspace.argtypes = [_c_int] * 6
    lib.fn2b200_warp_concat_backward_up_workspace.restype = ctypes.c_size_t
    lib.fn2b200_warp_concat_backward_up.argtypes = ([_c_ptr, lp, _c_int, _c_ptr, _c_int, _c_int, _c_int, ctypes.c_float, _c_ptr]
                                                    + [_c_int] * 5 + [ctypes.c_float] + [_c_int] * 2
                                                    + [_c_ptr, _c_ptr, _c_ptr, ctypes.c_size_t] + [_c_int] * 3 + [_c_ptr])
    lib.fn2b200_warp_concat_backward_up.restype = _c_int
    lib.fn2b200_resample2d_backward.argtypes = [_c_ptr, lp, _c_ptr, _c_ptr, _c_ptr, _c_ptr] + [_c_int] * 9 + [_c_ptr]
    lib.fn2b200_resample2d_backward_workspace.argtypes = [lp] + [_c_int] * 6
    lib.fn2b200_resample2d_backward_workspace.restype = ctypes.c_size_t
    lib.fn2b200_resample2d_backward_ws.argtypes = ([_c_ptr, lp, _c_ptr, _c_ptr, _c_ptr, _c_ptr] + [_c_int] * 9
                                                   + [_c_ptr, ctypes.c_size_t, _c_ptr])
    lib.fn2b200_resample2d_backward_ws.restype = _c_int
    lib.fn2b200_channelnorm_forward.argtypes = [_c_ptr, _c_ptr] + [_c_int] * 5 + [_c_ptr]
    lib.fn2b200_channelnorm_backward.argtypes = [_c_ptr] * 4 + [_c_int] * 5 + [_c_ptr]
    lib.fn2b200_channelnorm_forward_16.argtypes = [_c_ptr, _c_ptr] + [_c_int] * 6 + [_c_ptr]
    lib.fn2b200_channelnorm_forward_16.restype = _c_int
    lib.fn2b200_channelnorm_backward_16.argtypes = [_c_ptr] * 4 + [_c_int] * 6 + [_c_ptr]
    lib.fn2b200_channelnorm_backward_16.restype = _c_int
    for name in ("correlation_out_shape", "correlation_path", "correlation_forward",
                 "correlation_backward", "resample2d_forward", "resample2d_backward",
                 "channelnorm_forward", "channelnorm_backward"):
        getattr(lib, "fn2b200_" + name).restype = _c_int
    return lib


LIB = _load()

#: every symbol include/fn2b200.h declares (checked by tests/test_capi_symbols.py)
SYMBOLS = (
    "fn2b200_version", "fn2b200_last_error", "fn2b200_launch_count",
    "fn2b200_correlation_out_shape", "fn2b200_correlation_path",
    "fn2b200_correlation_forward", "fn2b200_correlation_backward",
    "fn2b200_correlation_forward_workspace", "fn2b200_correlation_forward_ws", "fn2b200_correlation_forward_cat",
    "fn2b200_correlation_backward_workspace", "fn2b200_correlation_backward_ws", "fn2b200_correlation_backward_cat",
    "fn2b200_resample2d_forward", "fn2b200_resample2d_backward",
    "fn2b200_resample2d_forward_up", "fn2b200_warp_concat_forward",
    "fn2b200_warp_concat_backward_workspace", "fn2b200_warp_concat_backward",
    "fn2b200_warp_concat_backward_up_workspace", "fn2b200_warp_concat_backward_up",
    "fn2b200_resample2d_backward_workspace", "fn2b200_resample2d_backward_ws",
    "fn2b200_channelnorm_forward", "fn2b200_channelnorm_backward",
    "fn2b200_channelnorm_forward_16", "fn2b200_channelnorm_backward_16",
)


OPS_LIBRARY_PATH = os.path.join(_HERE, "pybind", "fn2b200_ops" + (sysconfig.get_config_var("EXT_SUFFIX") or ".so"))


def _load_ops():
    """pybind/fn2b200_ops.cc, loaded as a Python module: importing it registers the torch.ops.fn2b200 operators, and
    the module's functions are the host-side glue of every op (what ``functional`` calls)."""
    if not os.path.isfile(OPS_LIBRARY_PATH) and os.environ.get("FN2B200_AUTOBUILD", "1") == "1":
        _run_build(os.path.join(_HERE, "pybind", "build_pybind.py"))
    if not os.path.isfile(OPS_LIBRARY_PATH):
        raise ImportError("%s not built: run python flownet2-pytorch_b200/pybind/build_pybind.py" % OPS_LIBRARY_PATH)
    import torch  # noqa: F401  (the module's tensor arguments need torch's bindings)
    spec = importlib.util.spec_from_file_location("fn2b200_ops", OPS_LIBRARY_PATH)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


OPS = _load_ops()


def check(rc, what):
    if rc != 0:
        msg = LIB.fn2b200_last_error().decode("utf-8", "replace")
        raise Fn2B200Error("%s failed (status %d): %s" % (what, rc, msg))
