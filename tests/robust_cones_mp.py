"""TEST INFRASTRUCTURE ONLY — the 50-digit stage problem of tests/robust_mp.py with an ellipsoid per row and an optional
u box, for robust problems with several robust constraints.  No new mathematics: every row is evaluated by
robust_mp.Stage's own code, which reads the axes of the row it is working on; the u box enters as the two linear rows
u - uhi <= 0 and ulo - u <= 0 that ecosWrapper adds for a ubound (ecos_solverwrapper.py:138-150)."""
import contextlib

import numpy as np
from mpmath import mpf

import robust_mp as rmp


class RowStage(rmp.Stage):
    """rmp.Stage with axes [n, 3] (one ellipsoid per row; rows without the robust flag ignore theirs) and ubox
    (ulo, uhi) or None."""

    def __init__(self, a, b, c, conic, axes, xl, xh, xnext=None, ubox=None):
        a, b, c = (np.asarray(v, dtype=np.float64).ravel() for v in (a, b, c))
        conic = np.asarray(conic, dtype=bool).ravel()
        axes = np.asarray(axes, dtype=np.float64).reshape(len(a), 3)
        if ubox is not None:
            a = np.concatenate((a, [1.0, -1.0]))
            b = np.concatenate((b, [0.0, 0.0]))
            c = np.concatenate((c, [-float(ubox[1]), float(ubox[0])]))
            conic = np.concatenate((conic, [False, False]))
            axes = np.concatenate((axes, np.zeros((2, 3))))
        self._axes = [tuple(mpf(float(v)) for v in ax) for ax in axes] + [(mpf(0),) * 3] * 2   # + the x_next rows
        self._j = 0
        super(RowStage, self).__init__(a, b, c, conic, (0.0, 0.0, 0.0), xl, xh, xnext)
        # the inputs as given, axes per row (rmp.Stage's src holds its one ellipsoid there)
        self.src = (a, b, c, conic, tuple(map(tuple, axes)), float(xl), float(xh),
                    None if xnext is None else tuple(float(v) for v in xnext))

    # the axes of the row being evaluated (rmp.Stage reads self.ru / rx / rc inside its per-row methods)
    ru = property(lambda self: self._axes[self._j][0], lambda self, v: None)
    rx = property(lambda self: self._axes[self._j][1], lambda self, v: None)
    rc = property(lambda self: self._axes[self._j][2], lambda self, v: None)

    def f(self, j, u, x):
        self._j = j
        return super(RowStage, self).f(j, u, x)

    def _size(self, j, u, x):
        self._j = j
        return super(RowStage, self)._size(j, u, x)

    def row_set(self, j, x, certify=True):
        self._j = j
        return super(RowStage, self).row_set(j, x, certify)

    def _certify(self, j, x, s):
        self._j = j
        return super(RowStage, self)._certify(j, x, s)

    # rmp.Stage.flip_width / u_flip_width build perturbed copies as `Stage.__new__(Stage)` plus this stage's __dict__;
    # the copies must be RowStages, or they would lose the per-row axes
    def flip_width(self, direction, x_ref, eps=1e-16):
        with _copies_as(RowStage):
            return super(RowStage, self).flip_width(direction, x_ref, eps)

    def u_flip_width(self, x, end, eps=1e-16):
        with _copies_as(RowStage):
            return super(RowStage, self).u_flip_width(x, end, eps)


@contextlib.contextmanager
def _copies_as(cls):
    saved = rmp.Stage
    rmp.Stage = cls
    try:
        yield
    finally:
        rmp.Stage = saved
