"""Loader for ``oracle/_ref`` -- the reference's own CUDA extensions rebuilt for sm_90a
(TEST INFRASTRUCTURE ONLY; see oracle/build_ref.py).  Returns None when they are not built."""
import glob
import importlib.machinery
import importlib.util
import os
import sys

_HERE = os.path.dirname(os.path.abspath(__file__))
REF_SO = os.path.join(_HERE, "_ref")
REF_PY = os.path.join(os.path.dirname(_HERE), "baseline", "_ref", "flownet2_pytorch")
_CACHE = {}


def load_extension(name):
    """name in {'correlation_cuda', 'resample2d_cuda', 'channelnorm_cuda'} -> module or None."""
    if name in _CACHE:
        return _CACHE[name]
    import torch  # noqa: F401  (the extensions link against libtorch)
    hits = glob.glob(os.path.join(REF_SO, name + "*.so"))
    mod = None
    if hits:
        loader = importlib.machinery.ExtensionFileLoader(name, hits[0])
        spec = importlib.util.spec_from_file_location(name, hits[0], loader=loader)
        mod = importlib.util.module_from_spec(spec)
        loader.exec_module(mod)
    _CACHE[name] = mod
    return mod


def available():
    return all(load_extension(n) is not None for n in ("correlation_cuda", "resample2d_cuda", "channelnorm_cuda"))


def python_tree_available():
    return os.path.isfile(os.path.join(REF_PY, "models.py"))


def install_reference_extensions():
    """Put the reference's rebuilt extensions into sys.modules under their own names."""
    for n in ("correlation_cuda", "resample2d_cuda", "channelnorm_cuda"):
        m = load_extension(n)
        if m is None:
            raise RuntimeError("oracle/_ref/%s*.so missing -- run oracle/build_ref.py where /root/reference exists" % n)
        sys.modules[n] = m


def import_reference_models(fresh=True):
    """Import the unmodified reference ``models`` module from baseline/_ref (whatever ``*_cuda`` /
    ``networks.*`` entries are in sys.modules at this moment get bound)."""
    if not python_tree_available():
        raise RuntimeError("baseline/_ref/flownet2_pytorch missing -- run oracle/build_ref.py")
    if fresh:
        for k in [k for k in sys.modules if k == "models" or k == "networks" or k.startswith("networks.")]:
            # keep pre-seeded layer modules (B2) -- only drop what came from the reference tree
            mod = sys.modules[k]
            if getattr(mod, "__file__", "") and REF_PY in os.path.abspath(getattr(mod, "__file__", "")):
                del sys.modules[k]
        sys.modules.pop("models", None)
    if REF_PY not in sys.path:
        sys.path.insert(0, REF_PY)
    import importlib
    return importlib.import_module("models")
