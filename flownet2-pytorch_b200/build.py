"""Build libfn2b200.so (the product) and libfn2b200_test.so (micro-benchmarks, csrc_test/) for
sm_90a in-tree with nvcc -- no torch dependency, seconds per file.

    python flownet2-pytorch_b200/build.py [--force] [--verbose]

The shared objects land next to this file (git-ignored build products).  Sources are hashed so a rebuild only happens
when something changed.
"""
import hashlib
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
INCLUDE = os.path.join(os.path.dirname(HERE), "include")
CSRC_TEST = os.path.join(HERE, "csrc_test")
LIB = os.path.join(HERE, "libfn2b200.so")
LIB_TEST = os.path.join(HERE, "libfn2b200_test.so")
STAMP = os.path.join(HERE, "build", "stamp.txt")

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-std=c++17", "-lineinfo",
    "-Xcompiler", "-fPIC,-O3",
    "-Xptxas", "-v",
    "--expt-relaxed-constexpr",
]


def _sources():
    return sorted(f for f in os.listdir(CSRC) if f.endswith(".cu"))


def _test_sources():
    return sorted(f for f in os.listdir(CSRC_TEST) if f.endswith(".cu"))


def _digest():
    """sha1 over the sources and flags."""
    h = hashlib.sha1()
    for f in sorted(os.listdir(CSRC)) + ["../../include/fn2b200.h"]:
        h.update(open(os.path.join(CSRC, f), "rb").read())
    for f in sorted(os.listdir(CSRC_TEST)):
        h.update(open(os.path.join(CSRC_TEST, f), "rb").read())
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()


def nvcc_path():
    for cand in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if cand and (os.path.isfile(cand) or cand == "nvcc"):
            return cand
    return "nvcc"


def build(force=False, verbose=False):
    digest = _digest()
    if (not force and os.path.isfile(LIB) and os.path.isfile(LIB_TEST) and os.path.isfile(STAMP)
            and open(STAMP).read().strip() == digest):
        return LIB
    obj_dir = os.path.join(HERE, "build")
    os.makedirs(obj_dir, exist_ok=True)
    nvcc = nvcc_path()

    def compile_one(job):
        src_dir, src = job
        obj = os.path.join(obj_dir, src[:-3] + ".o")
        cmd = [nvcc] + NVCC_FLAGS + ["-I", INCLUDE, "-c", os.path.join(src_dir, src), "-o", obj]
        r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
        open(os.path.join(obj_dir, src[:-3] + ".ptxas.log"), "w").write(r.stdout)
        if r.returncode != 0:
            raise RuntimeError("nvcc failed for %s:\n%s" % (src, r.stdout[-6000:]))
        if verbose:
            print(r.stdout)
        return obj

    jobs = [(CSRC, f) for f in _sources()] + [(CSRC_TEST, f) for f in _test_sources()]
    with ThreadPoolExecutor(max_workers=os.cpu_count() or 4) as ex:
        objs = list(ex.map(compile_one, jobs))
    n = len(_sources())

    def link(out, objects):
        tmp = out + ".tmp%d" % os.getpid()
        cmd = [nvcc, "-shared", "-gencode", "arch=compute_90a,code=sm_90a", "-o", tmp] + objects + ["-cudart", "static"]
        r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
        if r.returncode != 0:
            raise RuntimeError("link failed:\n" + r.stdout[-4000:])
        os.replace(tmp, out)

    link(LIB, objs[:n])
    # the test library carries its own copy of the host plumbing (runtime.o) -- it never links the product kernels
    link(LIB_TEST, objs[n:] + [os.path.join(obj_dir, "runtime.o")])
    open(STAMP, "w").write(digest)
    return LIB


if __name__ == "__main__":
    path = build(force="--force" in sys.argv, verbose="--verbose" in sys.argv)
    print(path)
