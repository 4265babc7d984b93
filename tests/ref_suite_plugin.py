"""pytest plugin (-p ref_suite_plugin) used by tests/test_reference_suite_dropin.py: makes `import toppra` resolve to
toppra_b200, so that the reference's OWN, unmodified test files (read in place from the reference checkout, never copied)
exercise this package's reference-facing API.  Without a GPU the kernels are replaced by the oracle-backed test double
(tests/cpu_engine.py) — what such a run proves is the API surface: names, argument meaning, return shapes, error
behaviour.  With TB_REF_SUITE_ENGINE=gpu the real engine is used."""
import importlib
import importlib.abc
import importlib.util
import os
import sys
import types

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for p in (ROOT, HERE):
    if p not in sys.path:
        sys.path.insert(0, p)


class _Alias(importlib.abc.MetaPathFinder, importlib.abc.Loader):
    """toppra[.x.y] -> toppra_b200[.x.y]; the alias module IS the toppra_b200 module object."""

    def find_spec(self, name, path=None, target=None):
        if name == "toppra" or name.startswith("toppra."):
            return importlib.util.spec_from_loader(name, self)
        return None

    def create_module(self, spec):
        return importlib.import_module("toppra_b200" + spec.name[len("toppra"):])

    def exec_module(self, module):
        pass


sys.meta_path.insert(0, _Alias())


class _Absent(types.ModuleType):
    """Stand-in for a third-party module the reference's tests import at module level but that is not installed here
    (matplotlib): importing works, USING it skips the test."""

    __path__ = []

    def __getattr__(self, name):
        if name.startswith("__"):
            raise AttributeError(name)
        import pytest
        pytest.skip("%s is not installed" % self.__name__)


try:
    importlib.import_module("cvxpy")
except ImportError:       # LP subset on scipy's HiGHS, so that the cvxpy-validated tests validate instead of skipping
    import mini_cvxpy
    sys.modules["cvxpy"] = mini_cvxpy

for _name in ("matplotlib", "matplotlib.pyplot"):
    try:
        importlib.import_module(_name)
    except ImportError:
        sys.modules[_name] = _Absent(_name)
        if "." in _name:   # `import a.b as c` reads the attribute b of a
            setattr(sys.modules[_name.rsplit(".", 1)[0]], _name.rsplit(".", 1)[1], sys.modules[_name])

import toppra_b200  # noqa: E402

if os.environ.get("TB_REF_SUITE_ENGINE", "cpu_double") != "gpu":
    import pytest  # noqa: E402
    import cpu_engine  # noqa: E402

    _mp = pytest.MonkeyPatch()
    cpu_engine.install(_mp)
