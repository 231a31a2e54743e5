#!/usr/bin/env python3
"""Build recipe for ``oracle/_ref`` -- the REFERENCE's own CUDA kernels rebuilt for sm_90a.

TEST INFRASTRUCTURE ONLY.  Nothing under ``oracle/`` is on the product path; only ``tests/``,
``__graft_entry__.smoke()`` and ``bench.py``'s reference / cpu_baseline legs may load what this
script produces.

What it does (needs ``/root/reference``; the GPU box only ever sees the prebuilt outputs):

1. copies ``networks/{correlation,resample2d,channelnorm}_package`` to a scratch dir under /tmp
   (the reference tree is read-only and its sources must never enter this repository),
2. applies the two mechanical fixes the sources need to compile with torch 2.11 / nvcc 12.9
   (SURVEY.md section 8c): drop ``-std=c++11`` and the sm_50..sm_70 ``-gencode`` list from each
   ``setup.py``; ``tensor.type()`` -> ``tensor.scalar_type()`` inside the ``AT_DISPATCH_*`` macros
   (correlation_cuda_kernel.cu:386,393,403,495,507,524,541; channelnorm_kernel.cu:111,152),
3. builds each package with ``TORCH_CUDA_ARCH_LIST=9.0a`` and copies ONLY the resulting
   ``*_cuda*.so`` files into ``oracle/_ref/`` (git-ignored, not gpurun-ignored),
4. "installs" the reference's Python model code (models.py + networks/*.py, unmodified) into
   ``baseline/_ref/flownet2_pytorch/`` (git-ignored) so the end-to-end FlowNet2 / FlowNet2C
   harness can import the unmodified ``models.py`` on the GPU box, where /root/reference is absent.

No arithmetic is changed by the patch: the kernels are the reference's, byte for byte.
"""
import os
import re
import shutil
import subprocess
import sys
import tempfile

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.environ.get("FN2_REFERENCE", "/root/reference")
OUT_SO = os.path.join(REPO, "oracle", "_ref")
OUT_PY = os.path.join(REPO, "baseline", "_ref", "flownet2_pytorch")
PACKAGES = ("correlation", "resample2d", "channelnorm")


def _patch_setup(path):
    src = open(path).read()
    src = src.replace("cxx_args = ['-std=c++11']", "cxx_args = []")
    src = re.sub(r"nvcc_args = \[.*?\]", "nvcc_args = ['-lineinfo']", src, flags=re.S)
    open(path, "w").write(src)


def _patch_dispatch(path):
    src = open(path).read()
    src = re.sub(r"(AT_DISPATCH_[A-Z_]+\(\s*\w+)\.type\(\)", r"\1.scalar_type()", src)
    open(path, "w").write(src)


def build_extensions(force=False):
    os.makedirs(OUT_SO, exist_ok=True)
    have = [f for f in os.listdir(OUT_SO) if f.endswith(".so")]
    if not force and all(any(f.startswith(p + "_cuda") for f in have) for p in PACKAGES):
        return
    if not os.path.isdir(REF):
        raise RuntimeError("reference tree %s not present and oracle/_ref is not prebuilt" % REF)
    work = tempfile.mkdtemp(prefix="fn2ref_")
    env = dict(os.environ, TORCH_CUDA_ARCH_LIST="9.0a", MAX_JOBS=str(os.cpu_count() or 4))
    procs = []
    for p in PACKAGES:
        dst = os.path.join(work, p + "_package")
        shutil.copytree(os.path.join(REF, "networks", p + "_package"), dst, copy_function=shutil.copyfile)   # writable copies
        _patch_setup(os.path.join(dst, "setup.py"))
        for f in os.listdir(dst):
            if f.endswith(".cu"):
                _patch_dispatch(os.path.join(dst, f))
        log = open(os.path.join(work, p + ".log"), "w")
        procs.append((p, dst, log, subprocess.Popen(
            [sys.executable, "setup.py", "build_ext", "--inplace"], cwd=dst, env=env,
            stdout=log, stderr=subprocess.STDOUT)))
    for p, dst, log, proc in procs:
        rc = proc.wait()
        log.close()
        if rc != 0:
            sys.stderr.write(open(log.name).read()[-4000:])
            raise RuntimeError("reference package %s failed to build (log %s)" % (p, log.name))
        for f in os.listdir(dst):
            if f.endswith(".so"):
                shutil.copy2(os.path.join(dst, f), os.path.join(OUT_SO, f))
    shutil.rmtree(work, ignore_errors=True)


def install_python(force=False):
    if os.path.isfile(os.path.join(OUT_PY, "models.py")) and not force:
        return
    if not os.path.isdir(REF):
        return
    if os.path.isdir(OUT_PY):
        shutil.rmtree(OUT_PY)
    os.makedirs(os.path.join(OUT_PY, "networks"))
    for f in ("models.py", "__init__.py", "losses.py"):
        shutil.copy2(os.path.join(REF, f), os.path.join(OUT_PY, f))
    net = os.path.join(REF, "networks")
    for f in os.listdir(net):
        if f.endswith(".py"):
            shutil.copy2(os.path.join(net, f), os.path.join(OUT_PY, "networks", f))
    for p in PACKAGES:
        d = os.path.join(OUT_PY, "networks", p + "_package")
        os.makedirs(d)
        for f in ("__init__.py", p + ".py"):
            shutil.copy2(os.path.join(net, p + "_package", f), os.path.join(d, f))


def main():
    force = "--force" in sys.argv
    install_python(force)
    build_extensions(force)
    print("oracle/_ref:", sorted(os.listdir(OUT_SO)))


if __name__ == "__main__":
    main()
