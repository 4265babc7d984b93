"""TEST INFRASTRUCTURE ONLY — loads the UNMODIFIED reference build (oracle/_ref/toppra, made by
oracle/build_ref.sh) so tests / bench.py's cpu_baseline leg can run the reference's own
`TOPPRA(..., solver_wrapper="seidel")` path.  Nothing in toppra_b200/ may import this."""
import importlib
import os
import sys

_HERE = os.path.dirname(os.path.abspath(__file__))
REF_DIR = os.path.join(_HERE, "_ref")


def reference_available():
    return os.path.isdir(os.path.join(REF_DIR, "toppra"))


def load_reference():
    """Return the reference `toppra` package (imported from oracle/_ref)."""
    if not reference_available():
        raise ImportError("oracle/_ref/toppra missing: run oracle/build_ref.sh (TOPPRA_REFERENCE=<toppra checkout>, default /root/reference)")
    try:
        import matplotlib.pyplot  # noqa: F401
    except Exception:  # matplotlib absent -> stub (algorithm.py:14 imports pyplot unconditionally)
        stubs = os.path.join(_HERE, "stubs")
        if stubs not in sys.path:
            sys.path.insert(0, stubs)
    if REF_DIR not in sys.path:
        sys.path.insert(0, REF_DIR)
    mod = importlib.import_module("toppra")
    if not os.path.abspath(mod.__file__).startswith(REF_DIR):
        raise ImportError("a different `toppra` (%s) shadows oracle/_ref" % mod.__file__)
    importlib.import_module("toppra.algorithm")
    importlib.import_module("toppra.constraint")
    importlib.import_module("toppra.solverwrapper.cy_seidel_solverwrapper")
    return mod
