"""ctypes binding of libfn2b200_test.so (flownet2-pytorch_b200/csrc_test/fn2b200_test.h): hardware self-tests
and micro-benchmarks.  Only tests/ load it -- the product package never does."""
import ctypes
import os

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB_PATH = os.path.join(ROOT, "flownet2-pytorch_b200", "libfn2b200_test.so")
HEADER = os.path.join(ROOT, "flownet2-pytorch_b200", "csrc_test", "fn2b200_test.h")

SYMBOLS = ("fn2b200_test_last_error", "fn2b200_test_wgmma_gemm_ss", "fn2b200_test_wgmma_gemm_mn", "fn2b200_test_wgmma_gemm_rs",
           "fn2b200_test_wgmma_gemm_rs_tma", "fn2b200_test_atomics_bench")


def load():
    if not os.path.isfile(LIB_PATH):
        raise ImportError("libfn2b200_test.so not built (python flownet2-pytorch_b200/build.py)")
    lib = ctypes.CDLL(LIB_PATH)
    p, i = ctypes.c_void_p, ctypes.c_int
    lib.fn2b200_test_last_error.restype = ctypes.c_char_p
    for s in SYMBOLS[1:5]:
        getattr(lib, s).argtypes = [p, p, p, i, p]
    lib.fn2b200_test_atomics_bench.argtypes = [p, p, i, i, i, i, p]
    for s in SYMBOLS[1:]:
        getattr(lib, s).restype = i
    return lib


def check(lib, rc, what):
    if rc != 0:
        raise RuntimeError("%s failed (status %d): %s" % (what, rc, lib.fn2b200_test_last_error().decode("utf-8", "replace")))
