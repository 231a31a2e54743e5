"""Build the three pybind extension modules the reference imports by name -- ``correlation_cuda``,
``resample2d_cuda``, ``channelnorm_cuda`` (correlation.py:4, resample2d.py:3, channelnorm.py:3) -- as thin ATen glue
over libfn2b200.so's C ABI (g++ only: no device code lives here).

    python flownet2-pytorch_b200/pybind/build_pybind.py [--force]

The .so files land next to this file (git-ignored; they travel to the GPU box with the gpurun snapshot) and find
libfn2b200.so through an $ORIGIN-relative rpath.  ``flownet2_b200.compat.install("B1p")`` puts them on sys.modules.
"""
import hashlib
import os
import subprocess
import sys
import sysconfig
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
PKG = os.path.dirname(HERE)
INCLUDE = os.path.join(os.path.dirname(PKG), "include")
NAMES = ("correlation_cuda", "resample2d_cuda", "channelnorm_cuda")
SUFFIX = sysconfig.get_config_var("EXT_SUFFIX") or ".so"


def target(name):
    return os.path.join(HERE, name + SUFFIX)


def _digest():
    h = hashlib.sha1()
    for f in sorted(os.listdir(HERE)):
        if f.endswith((".cc", ".h", ".py")):
            h.update(open(os.path.join(HERE, f), "rb").read())
    h.update(open(os.path.join(INCLUDE, "fn2b200.h"), "rb").read())
    import torch
    h.update(torch.__version__.encode())
    return h.hexdigest()


def build(force=False):
    stamp = os.path.join(HERE, "stamp.txt")
    digest = _digest()
    if not force and all(os.path.isfile(target(n)) for n in NAMES) and os.path.isfile(stamp) and open(stamp).read() == digest:
        return [target(n) for n in NAMES]
    from torch.utils import cpp_extension as ce
    inc = [INCLUDE, HERE] + ce.include_paths("cuda")
    libdirs = ce.library_paths("cuda")
    # the system g++ (the one nvcc and torch's own extensions use), NOT $CXX: this image's $CXX is a private GCC whose
    # libstdc++ is static-only -- linked into an extension it brings a second, uninitialised copy of the iostream locale
    # machinery and the first integer formatted into an error message segfaults
    cxx = os.environ.get("FN2B200_CXX", "g++")

    def one(name):
        cmd = [cxx, "-O2", "-std=c++17", "-fPIC", "-shared", "-DTORCH_EXTENSION_NAME=" + name, "-DTORCH_API_INCLUDE_EXTENSION_H",
               "-D_GLIBCXX_USE_CXX11_ABI=%d" % int(__import__("torch")._C._GLIBCXX_USE_CXX11_ABI)]
        cmd += ["-I" + sysconfig.get_paths()["include"]] + ["-I" + p for p in inc]
        cmd += [os.path.join(HERE, name + ".cc"), "-o", target(name) + ".tmp"]
        cmd += ["-L" + p for p in libdirs] + ["-L" + PKG, "-l:libfn2b200.so", "-Wl,-rpath,$ORIGIN/..",
                                              "-lc10", "-lc10_cuda", "-ltorch_cpu", "-ltorch_cuda", "-ltorch", "-ltorch_python", "-lcudart"]
        cmd += ["-Wl,-rpath," + p for p in libdirs]
        r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
        if r.returncode != 0:
            raise RuntimeError("building %s failed:\n%s" % (name, r.stdout[-4000:]))
        syms = subprocess.run(["nm", "-D", "--defined-only", target(name) + ".tmp"], stdout=subprocess.PIPE, text=True).stdout
        if "_ZNSo9_M_insert" in syms or "codecvt" in syms:
            raise RuntimeError("%s: libstdc++ was linked statically into the extension (compiler %s); use the system g++" % (name, cxx))
        os.replace(target(name) + ".tmp", target(name))
        return target(name)
    with ThreadPoolExecutor(max_workers=3) as ex:
        outs = list(ex.map(one, NAMES))
    open(stamp, "w").write(digest)
    return outs


if __name__ == "__main__":
    for p in build(force="--force" in sys.argv):
        print(p)
