"""Locate and import the UNMODIFIED reference package (TEST / BASELINE INFRASTRUCTURE ONLY).

Search order: $VQB_REFERENCE_ROOT (a directory that contains `vector_quantize_pytorch/`), then `oracle/_ref/` (git-ignored;
`install()` copies the reference package there, and `__graft_entry__.build()` calls it when $VQB_REFERENCE_SRC names a
checkout of the reference).  Used to (a) generate the golden fixtures under tests/golden/ (oracle/gen_golden*.py) and
(b) time the reference's own CPU forward in `bench.py --impl reference` / `cpu_baseline`.  No test needs it: the tests
compare against the stored fixtures.  `einx` is not a dependency of this project and is never called on the hot path:
oracle/einx_shim stands in for it.
"""
import importlib
import os
import shutil
import sys

_HERE = os.path.dirname(os.path.abspath(__file__))
_SHIM = os.path.join(_HERE, "einx_shim")
INSTALL_ROOT = os.path.join(_HERE, "_ref")


def reference_root():
    for c in (os.environ.get("VQB_REFERENCE_ROOT"), INSTALL_ROOT):
        if c and os.path.isdir(os.path.join(c, "vector_quantize_pytorch")):
            return c
    return None


def reference_available() -> bool:
    return reference_root() is not None


def install(src):
    """Copy the reference package (pure Python) from the checkout `src` into oracle/_ref/.  Returns False without it."""
    pkg = os.path.join(src, "vector_quantize_pytorch")
    if not os.path.isdir(pkg):
        return False
    dst = os.path.join(INSTALL_ROOT, "vector_quantize_pytorch")
    tmp = dst + ".tmp%d" % os.getpid()
    shutil.rmtree(tmp, ignore_errors=True)
    shutil.copytree(pkg, tmp, ignore=shutil.ignore_patterns("__pycache__"))
    shutil.rmtree(dst, ignore_errors=True)
    os.replace(tmp, dst)
    return True


def load_reference():
    """Returns the imported `vector_quantize_pytorch` reference module (einx shimmed)."""
    root = reference_root()
    if root is None:
        raise RuntimeError("reference not found ($VQB_REFERENCE_ROOT, oracle/_ref)")
    try:
        importlib.import_module("einx")
    except ImportError:
        sys.path.insert(0, _SHIM)
    if root not in sys.path:
        sys.path.insert(0, root)
    return importlib.import_module("vector_quantize_pytorch")
