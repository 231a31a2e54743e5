"""CPU tests of the drop-in boundary: the C-ABI library loads, exports every symbol that
include/fn2b200.h declares, and validates its arguments (no kernel is launched here)."""
import ctypes
import os
import re

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared_symbols():
    hdr = open(os.path.join(ROOT, "include", "fn2b200.h")).read()
    hdr = re.sub(r"/\*.*?\*/", "", hdr, flags=re.S)
    return sorted(set(re.findall(r"\b(fn2b200_\w+)\s*\(", hdr)))


def test_library_exports_every_declared_symbol():
    import flownet2_b200
    lib = ctypes.CDLL(flownet2_b200._lib.LIB_PATH)
    declared = _declared_symbols()
    assert len(declared) >= 11
    for name in declared:
        assert hasattr(lib, name), "libfn2b200.so does not export %s" % name
    assert sorted(flownet2_b200._lib.SYMBOLS) == declared
    assert lib.fn2b200_version() == 100


def test_library_is_sm90a_with_tma():
    import subprocess
    import flownet2_b200
    try:
        out = subprocess.run(["cuobjdump", "-lelf", flownet2_b200._lib.LIB_PATH], capture_output=True, text=True).stdout
    except FileNotFoundError:
        pytest.skip("cuobjdump not available")
    assert "sm_90a" in out


def test_argument_validation_without_gpu():
    from flownet2_b200._lib import LIB
    null = ctypes.c_void_p(0)
    one = ctypes.c_void_p(16)  # never dereferenced: validation fails first
    # stride1 != 1 in backward: the reference cannot run it either
    rc = LIB.fn2b200_correlation_backward(one, one, one, one, one, 1, 4, 8, 8, 4, 1, 4, 2, 2, 1, null)
    assert rc == -2 and b"stride1" in LIB.fn2b200_last_error()
    # empty output
    rc = LIB.fn2b200_correlation_forward(one, one, one, 1, 4, 8, 8, 0, 1, 20, 1, 2, 1, null)
    assert rc == -1
    # null pointers
    rc = LIB.fn2b200_correlation_forward(null, one, one, 1, 4, 8, 8, 4, 1, 4, 1, 2, 1, null)
    assert rc == -3
    # kernel_size > 1 for resample2d
    st = (ctypes.c_int64 * 4)(192, 64, 8, 1)
    rc = LIB.fn2b200_resample2d_forward(one, st, one, one, 1, 3, 8, 8, 8, 8, 2, 1, null)
    assert rc == -2 and b"kernel_size" in LIB.fn2b200_last_error()
    rc = LIB.fn2b200_channelnorm_forward(one, one, 1, 0, 8, 8, 2, null)
    assert rc == -1
    # B == 0 is a no-op success
    assert LIB.fn2b200_channelnorm_forward(null, null, 0, 3, 8, 8, 2, null) == 0


def test_out_shape_and_path_queries():
    from flownet2_b200 import functional as F2
    from flownet2_b200._lib import LIB
    assert F2.correlation_out_shape(256, 48, 64, 20, 1, 20, 1, 2) == (441, 48, 64)
    assert F2.correlation_out_shape(8, 12, 13, 2, 1, 4, 2, 2) == (25, 4, 5)
    assert LIB.fn2b200_correlation_path(256, 112, 256, 20, 1, 20, 1, 2) == 2   # FlowNetC -> tensor-core fwd + tiled bwd
    assert LIB.fn2b200_correlation_path(20, 112, 256, 20, 1, 20, 1, 2) == 1    # C % 64 != 0 -> TMA-tiled FMA kernels
    assert LIB.fn2b200_correlation_path(256, 111, 256, 20, 1, 20, 1, 2) == 1   # odd H -> FMA kernels
    assert LIB.fn2b200_correlation_forward_workspace(8, 256, 112, 256, 20, 1, 20, 1, 2) == 8 * 8 * 256 * 112 * 256
    assert LIB.fn2b200_correlation_forward_workspace(8, 20, 112, 256, 20, 1, 20, 1, 2) == 0
    assert LIB.fn2b200_correlation_path(256, 112, 256, 20, 3, 20, 1, 2) == 0   # kernel_size 3 -> generic
    assert LIB.fn2b200_correlation_path(256, 112, 250, 20, 1, 20, 1, 2) == 2   # even W is enough for the tc forward
    assert LIB.fn2b200_correlation_path(256, 112, 251, 20, 1, 20, 1, 2) == 0   # odd W -> generic
    assert LIB.fn2b200_correlation_path(256, 112, 256, 22, 1, 20, 1, 2) == 0   # (md-pad) % 4 != 0 -> generic
    assert LIB.fn2b200_correlation_path(256, 112, 256, 24, 1, 20, 1, 2) == 1


def test_no_cpu_fallback():
    import flownet2_b200 as f
    with pytest.raises(RuntimeError, match="CUDA tensors only"):
        f.Correlation(4, 1, 4, 1, 2, 1)(torch.zeros(1, 2, 8, 8), torch.zeros(1, 2, 8, 8))
    with pytest.raises(RuntimeError, match="CUDA tensors only"):
        f.Resample2d()(torch.zeros(1, 3, 8, 8), torch.zeros(1, 2, 8, 8))
    with pytest.raises(RuntimeError, match="CUDA tensors only"):
        f.ChannelNorm()(torch.zeros(1, 3, 8, 8))


def test_api_surface_matches_reference():
    """Constructor / Function signatures of SURVEY 8(b) level B2."""
    import inspect
    import flownet2_b200 as f
    assert list(inspect.signature(f.Correlation.__init__).parameters)[1:] == [
        "pad_size", "kernel_size", "max_displacement", "stride1", "stride2", "corr_multiply"]
    c = f.Correlation()
    assert (c.pad_size, c.kernel_size, c.max_displacement, c.stride1, c.stride2, c.corr_multiply) == (0, 0, 0, 1, 2, 1)
    sig = inspect.signature(f.CorrelationFunction.forward)
    assert [sig.parameters[k].default for k in ("pad_size", "kernel_size", "max_displacement", "stride1", "stride2",
                                                "corr_multiply")] == [3, 3, 20, 1, 2, 1]
    r = f.Resample2d()
    assert (r.kernel_size, r.bilinear) == (1, True)
    assert f.ChannelNorm().norm_deg == 2
    assert not list(c.parameters()) and not list(c.buffers()) and not c.state_dict()
    # B1 shim modules export exactly forward/backward
    from flownet2_b200 import compat
    import sys
    compat.install_extension_shims()
    try:
        for name in ("correlation_cuda", "resample2d_cuda", "channelnorm_cuda"):
            m = sys.modules[name]
            assert callable(m.forward) and callable(m.backward)
        assert list(inspect.signature(sys.modules["correlation_cuda"].forward).parameters) == [
            "input1", "input2", "rInput1", "rInput2", "output", "pad_size", "kernel_size", "max_displacement",
            "stride1", "stride2", "corr_type_multiply"]
    finally:
        compat.uninstall()


def test_pybind_extension_modules_build_and_export_the_reference_interface():
    """north_star: 'a thin C++/pybind extension'.  The three modules the reference imports by name are compiled in-tree
    (g++, no device code), export forward / backward like the reference's PYBIND11_MODULE blocks
    (correlation_cuda.cc:169-172, resample2d_cuda.cc:28-31, channelnorm_cuda.cc:27-30) and refuse CPU tensors."""
    import importlib.util
    spec = importlib.util.spec_from_file_location("_bp", os.path.join(ROOT, "flownet2-pytorch_b200", "pybind", "build_pybind.py"))
    bp = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(bp)
    for so in bp.build():
        assert os.path.isfile(so)
    # in a child interpreter: pybind11 caches extension modules by name, and an earlier test of this process may have
    # imported the reference's own correlation_cuda (oracle/_ref)
    import subprocess
    import sys
    code = (
        "import sys, torch; sys.path.insert(0, %r)\n"
        "from flownet2_b200 import compat\n"
        "compat.install('B1p')\n"
        "for name in ('correlation_cuda', 'resample2d_cuda', 'channelnorm_cuda'):\n"
        "    mod = sys.modules[name]\n"
        "    assert mod.__file__.endswith('.so') and '/pybind/' in mod.__file__ and callable(mod.forward) and callable(mod.backward)\n"
        "a = torch.zeros(1, 4, 8, 8)\n"
        "try:\n"
        "    sys.modules['correlation_cuda'].forward(a, a, a.new(), a.new(), a.new(), 4, 1, 4, 1, 2, 1)\n"
        "except RuntimeError as e:\n"
        "    assert 'CUDA tensor' in str(e), str(e)\n"
        "    print('OK')\n" % ROOT)
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and r.stdout.strip().endswith("OK"), (r.stdout[-1000:], r.stderr[-2000:])


def test_new_entry_points_validate_arguments_without_gpu():
    """Round-2 entry points (fused warp-concat, upsampled-flow resample, correlation-into-concat, workspace queries):
    argument errors are reported before anything touches the device."""
    import flownet2_b200
    L = flownet2_b200._lib.LIB
    P, I64 = ctypes.c_void_p, ctypes.c_int64 * 4
    st = I64(6 * 64, 64, 8, 1)
    # empty batch is a no-op, not an error
    assert L.fn2b200_warp_concat_forward(P(0), st, 3, P(0), 8, 8, 0, 1.0, P(0), 12, 0, 6, 6, 9, 20.0, -1, 11, 0, 8, 8, P(0)) != 0   # null flow
    assert b"null flow" in L.fn2b200_last_error()
    one = ctypes.c_float(0.0)
    pf = ctypes.cast(ctypes.pointer(one), P)
    assert L.fn2b200_warp_concat_forward(P(0), st, 3, pf, 8, 8, 0, 1.0, P(0), 12, 0, 6, 6, 9, 20.0, -1, 11, 0, 8, 8, P(0)) == 0      # B = 0
    assert L.fn2b200_warp_concat_forward(P(0), st, 3, pf, 8, 8, 0, 1.0, P(0), 12, 0, 6, 4, 9, 20.0, -1, 11, 1, 8, 8, P(0)) == -1     # warped overlaps x
    assert b"overlap" in L.fn2b200_last_error()
    assert L.fn2b200_warp_concat_forward(P(0), st, 3, pf, 8, 8, 0, 1.0, P(0), 12, 0, 6, 6, 9, 0.0, -1, 11, 1, 8, 8, P(0)) == -1      # flow_div = 0
    assert L.fn2b200_warp_concat_forward(P(0), st, 3, pf, 2, 3, 1, 1.0, P(0), 12, 0, 6, 6, 9, 20.0, -1, 11, 1, 8, 8, P(0)) == -1     # 4 * 3 != 8
    assert b"does not match" in L.fn2b200_last_error()
    assert L.fn2b200_warp_concat_forward(P(0), st, 3, pf, 8, 8, 3, 1.0, P(0), 12, 0, 6, 6, 9, 20.0, -1, 11, 1, 8, 8, P(0)) == -1     # bad mode
    assert L.fn2b200_warp_concat_backward_workspace(2, 3, 8, 8) == 2 * 8 * 8 * 16
    assert L.fn2b200_warp_concat_backward_workspace(2, 4, 8, 8) == 0
    assert L.fn2b200_warp_concat_backward(P(0), st, 4, pf, pf, 12, 0, 6, 6, 9, 20.0, -1, 11, pf, pf, P(0), 0, 1, 8, 8, P(0)) == -2    # C > 3
    assert L.fn2b200_resample2d_forward_up(P(0), st, pf, 2, 2, 1, 20.0, P(0), 0, 3, 8, 8, P(0)) == 0                              # B = 0
    assert L.fn2b200_resample2d_forward_up(P(0), st, pf, 2, 2, 2, 20.0, P(0), 1, 3, 8, 12, P(0)) == -1                            # 4 * 2 != 12
    # correlation into a concat buffer: the channel range must fit
    assert L.fn2b200_correlation_forward_cat(pf, pf, pf, 440, 0, 0.1, 1, 64, 8, 8, 20, 1, 20, 1, 2, 1, P(0), 0, P(0)) == -1
    assert b"do not fit" in L.fn2b200_last_error()
    assert L.fn2b200_correlation_forward_cat(pf, pf, pf, 473, 32, 0.1, 0, 64, 8, 8, 20, 1, 20, 1, 2, 1, P(0), 0, P(0)) == 0        # B = 0
    # Resample2d backward scratch: 16 bytes per image pixel for C <= 3, none for C > 3 or the planar scatter
    assert L.fn2b200_resample2d_backward_workspace(st, 2, 3, 8, 8, 8, 8) == 2 * 8 * 8 * 16
    assert L.fn2b200_resample2d_backward_workspace(st, 2, 5, 8, 8, 8, 8) == 0
    os.environ["FN2B200_RS_BWD"] = "planar"
    try:
        assert L.fn2b200_resample2d_backward_workspace(st, 2, 3, 8, 8, 8, 8) == 0
    finally:
        del os.environ["FN2B200_RS_BWD"]
