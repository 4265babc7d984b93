"""TEST INFRASTRUCTURE ONLY — ctypes front-end of tests/closure_model.c, the scalar model of the scan kernel's min-x
closure on top of the Seidel-shortcut model.  The library is compiled on first use into the temporary directory."""
import ctypes
import hashlib
import os
import subprocess
import tempfile

import numpy as np

from oracle import oracle as orc

_SRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "closure_model.c")
_ORACLE = os.path.join(os.path.dirname(os.path.dirname(_SRC)), "oracle")
_KEYS = ("lps", "mismatches", "resolves_ref", "resolves_model", "a_used", "a_declined", "b_used", "b_declined",
         "closed", "close_declined")


def build():
    """gcc with the oracle's flags -> <tmp>/tb_closure_model_<hash of the sources>.so; returns its path."""
    h = hashlib.sha256()
    for f in (_SRC, os.path.join(_ORACLE, "shortcut_model.c"), os.path.join(_ORACLE, "toppra_oracle.c")):
        with open(f, "rb") as fh:
            h.update(fh.read())
    so = os.path.join(tempfile.gettempdir(), "tb_closure_model_%s.so" % h.hexdigest()[:16])
    if not os.path.exists(so):
        tmp = "%s.%d" % (so, os.getpid())
        subprocess.check_call(["gcc", "-O2", "-ffp-contract=off", "-fno-fast-math", "-fPIC", "-shared", "-o", tmp, _SRC,
                               "-lm", "-lpthread"])
        os.replace(tmp, so)
    return so


class closure_model:
    """Context manager like oracle.shortcut_model: route the oracle through the closure model, which checks every
    2-variable LP bit for bit.  `margin(gap)` sets the closure's relative margin (default 1e-7, the kernel's);
    `stats()` adds `closed` and `close_declined` to the shortcut model's counters."""
    _lib = None

    def __enter__(self):
        if closure_model._lib is None:
            L = orc._setup(ctypes.CDLL(build()))
            L.orc_closure_model_margin.argtypes = [ctypes.c_double]
            closure_model._lib = L
        self._saved = orc._LIB
        orc._LIB = closure_model._lib
        orc._LIB.orc_closure_model_enable(1)
        self.stats(reset=True)
        return self

    def __exit__(self, *exc):
        closure_model._lib.orc_closure_model_enable(0)
        closure_model._lib.orc_closure_model_margin(1e-7)
        orc._LIB = self._saved

    def margin(self, gap):
        closure_model._lib.orc_closure_model_margin(gap)

    def stats(self, reset=False):
        out = np.zeros(len(_KEYS), dtype=np.int64)
        closure_model._lib.orc_closure_model_stats(out.ctypes.data_as(orc._lp), 1 if reset else 0)
        return dict(zip(_KEYS, (int(v) for v in out)))
