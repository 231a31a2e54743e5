"""CPU test: tests/kernel_manifest.py lists exactly the `__global__` instantiations compiled into libfn2b200.so, and
names for each one a case of tests/test_gpu_kernel_coverage.py (or says why none can reach it).  A new instantiation
without a test, or a stale manifest entry, fails here without a GPU."""
import importlib.util
import os
import subprocess
import sys

import pytest

from kernel_manifest import KERNELS

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GPU_FILE = os.path.join(ROOT, "tests", "test_gpu_kernel_coverage.py")


def _library():
    spec = importlib.util.spec_from_file_location("_fn2b200_build", os.path.join(ROOT, "flownet2-pytorch_b200", "build.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod.build()


def _kernel_symbols(lib):
    """Demangled `__global__` symbols without argument lists, as `cuobjdump -symbols | c++filt` prints them."""
    try:
        out = subprocess.run(["cuobjdump", "-symbols", lib], capture_output=True, text=True, check=True).stdout
        mangled = [line.split()[-1] for line in out.splitlines() if "STT_FUNC" in line and "STB_GLOBAL" in line]
        names = subprocess.run(["c++filt"], input="\n".join(mangled), capture_output=True, text=True, check=True).stdout
    except FileNotFoundError:
        pytest.skip("cuobjdump or c++filt not available")
    return {n.split("(")[0] for n in names.splitlines() if n}


def test_manifest_equals_the_compiled_kernels():
    compiled = _kernel_symbols(_library())
    assert len(compiled) > 100
    missing, stale = sorted(compiled - set(KERNELS)), sorted(set(KERNELS) - compiled)
    assert not missing, "instantiations without a manifest entry (add a case to %s): %s" % (GPU_FILE, missing)
    assert not stale, "manifest entries the library no longer has: %s" % stale


def test_manifest_values_name_gpu_cases():
    """Each value is a node of the GPU file (collected here; the cases themselves are skipped without a GPU)."""
    r = subprocess.run([sys.executable, "-m", "pytest", "--collect-only", "-q", "-p", "no:cacheprovider", GPU_FILE],
                       capture_output=True, text=True, cwd=ROOT, timeout=300)
    nodes = {line.split("::", 1)[1] for line in r.stdout.splitlines() if "::" in line}
    assert nodes, r.stdout[-2000:] + r.stderr[-2000:]
    for kernel, case in KERNELS.items():
        if case.startswith("unreachable:"):
            assert len(case) > len("unreachable: "), "%s: give the reason" % kernel
            continue
        assert case in nodes, "%s: no case %s in %s" % (kernel, case, GPU_FILE)
