"""Geometric paths — same public surface as the reference `toppra/interpolator.py`
(`AbstractGeometricPath` :125-192, `SplineInterpolator` :360-466, `propose_gridpoints` :49-122), with the spline
fit (scipy CubicSpline restated) and the piecewise-cubic evaluation running on the GPU
(csrc/tb_spline.cu: tb_spline_fit / tb_ppoly_eval).  `BatchSplineInterpolator` is the batched form used by
`toppra_b200.BatchTOPPRA` (B independent paths, one launch)."""
import logging
from typing import Union

import numpy as np

from . import _lib_poly, engine
from .utils import deprecated

logger = logging.getLogger(__name__)


def propose_gridpoints(path, max_err_threshold=1e-4, max_iteration=100, max_seg_length=0.05, min_nb_points=100,
                       max_points=4096):
    """Generate gridpoints that sufficiently cover the given path (reference interpolator.py:49-122): segments longer
    than `max_seg_length`, or whose estimated interpolation error 0.5 * max|q''(mid)| * d^2 exceeds
    `max_err_threshold`, are bisected pass after pass; then every segment is bisected until there are at least
    `min_nb_points` points.  Runs on the GPU (csrc/tb_frows.cu: tb_propose_gridpoints); this is the B = 1 case of
    `BatchSplineInterpolator.propose_gridpoints`.  Returns the list of gridpoints like the reference."""
    if not hasattr(path, "as_batch"):
        raise TypeError("toppra_b200.propose_gridpoints needs a path with a piecewise-polynomial device form "
                        "(SplineInterpolator, PPolyPath, PiecewisePolyPath, SimplePath, PolynomialPath); got %s"
                        % type(path).__name__)
    grid, glen = path.as_batch().propose_gridpoints(max_err_threshold, max_iteration, max_seg_length, min_nb_points,
                                                    max_points)
    return grid[0, :int(glen[0])].cpu().numpy().tolist()


class AbstractGeometricPath(object):
    """Abstract base class that represents geometric paths (reference interpolator.py:125-192)."""

    def __call__(self, path_positions: Union[float, np.ndarray], order: int = 0) -> np.ndarray:
        raise NotImplementedError

    @property
    def dof(self) -> int:
        raise NotImplementedError

    @property
    def path_interval(self):
        raise NotImplementedError

    @property
    def waypoints(self):
        return None

    def eval(self, ss_sam):
        return self(ss_sam, 0)

    def evald(self, ss_sam):
        return self(ss_sam, 1)

    def evaldd(self, ss_sam):
        return self(ss_sam, 2)


class _DevicePPoly(object):
    """Stand-in for the scipy PPoly objects the reference exposes as `.cspl/.cspld/.cspldd`:
    callable, with `.c` (coefficients of this derivative order, scipy layout [k, nseg, dof]) and `.x`."""

    def __init__(self, owner, order):
        self._owner = owner
        self._order = order

    def __call__(self, s, nu=0):
        return self._owner(s, self._order + nu)

    def derivative(self, nu=1):
        return _DevicePPoly(self._owner, self._order + nu)

    @property
    def x(self):
        return self._owner.ss_waypoints

    @property
    def c(self):
        c = self._owner._coefficients()
        for _ in range(self._order):  # scipy PPoly.derivative: c'[j] = c[j] * (k - j)
            k = c.shape[0] - 1
            c = c[:-1] * np.arange(k, 0, -1).reshape(-1, 1, 1)
        return c


class BatchSplineInterpolator(object):
    """B cubic-spline paths fitted and evaluated on the GPU.

    Parameters
    ----------
    ss_waypoints: (n,) shared by all paths, or (B, n)
    waypoints: (B, n, dof)
    bc_type: as scipy.interpolate.CubicSpline ('not-a-knot', 'clamped', 'natural', or a pair of
        (order, value) tuples with order in {1, 2}), or 'periodic' (closed curves: waypoints[:, 0] == waypoints[:, -1]).
    device: torch device (default: current CUDA device)

    `ss_waypoints` / `waypoints` may be numpy arrays (copied H2D here) or CUDA tensors (used in place)."""

    def __init__(self, ss_waypoints, waypoints, bc_type="not-a-knot", device=None, validate=True):
        torch = engine.torch_mod()
        self.device = engine.default_device(device if device is not None else
                                            (waypoints.device if isinstance(waypoints, torch.Tensor) else None))
        self.d_wp = engine.as_device(waypoints, self.device)
        if self.d_wp.dim() != 3:
            raise ValueError("waypoints must have shape (B, n, dof)")
        self.B, self.n, self._dof = self.d_wp.shape
        self.d_ss = engine.as_device(ss_waypoints, self.device)
        if self.d_ss.shape[-1] != self.n or self.d_ss.dim() not in (1, 2) or (self.d_ss.dim() == 2 and
                                                                           self.d_ss.shape[0] != self.B):
            raise ValueError("ss_waypoints must have shape (n,) or (B, n)")
        if self.n < 2:
            raise ValueError("at least 2 waypoints are needed")
        self.ss_host = engine.host_view(ss_waypoints)  # None when the knots were given as a CUDA tensor
        if validate:
            # scipy CubicSpline raises "`x` must be strictly increasing sequence."; dx = 0 would give inf/NaN here.
            # Host inputs are checked on the host (no device synchronisation); CUDA tensors with one small reduction.
            if self.ss_host is None:
                increasing = not bool((self.d_ss[..., 1:] <= self.d_ss[..., :-1]).any())
            else:
                increasing = bool(np.all(np.diff(self.ss_host, axis=-1) > 0))
            if not increasing:
                raise ValueError("`ss_waypoints` must be a strictly increasing sequence.")
        self.bc_type = bc_type
        bc = engine.parse_bc(bc_type, self.B, self._dof, self.device)
        if validate and isinstance(bc_type, str) and bc_type == "periodic":
            # scipy _validate_bc: np.allclose(y[0], y[-1], rtol=1e-15, atol=1e-15)
            wp_host = engine.host_view(waypoints)
            if wp_host is not None:
                closed = bool(np.allclose(wp_host[:, 0], wp_host[:, -1], rtol=1e-15, atol=1e-15))
            else:
                first, last = self.d_wp[:, 0], self.d_wp[:, -1]
                closed = bool(((first - last).abs() <= 1e-15 + 1e-15 * last.abs()).all())
            if not closed:
                raise ValueError("The first and last `y` point along axis 0 must be identical (within machine precision) "
                                 "when bc_type='periodic'.")
        self.d_ppoly = engine.spline_fit(self.d_ss, self.d_wp, bc)

    @classmethod
    def from_ppoly(cls, breaks, coeffs, device=None):
        """Paths given directly as piecewise cubics in scipy's PPoly layout ("PPoly in", SURVEY §8 f4): any path type
        that has such a form (CubicSpline / PPoly objects, cubic Hermite paths, polynomials up to degree 3) goes to the
        kernels without a fit.

        breaks: (nseg + 1,) shared or (B, nseg + 1), strictly increasing.
        coeffs: (B, k, nseg, dof) with k <= 4, highest power first, local power basis
                sum_j c[j] (s - breaks[i]) ** (k - 1 - j) like `scipy.interpolate.PPoly.c`; k < 4 is zero-padded."""
        torch = engine.torch_mod()
        self = object.__new__(cls)
        self.device = engine.default_device(device if device is not None else
                                            (coeffs.device if isinstance(coeffs, torch.Tensor) else None))
        c = engine.as_device(coeffs, self.device)
        if c.dim() != 4 or not 1 <= c.shape[1] <= 4:
            raise ValueError("coeffs must have shape (B, k, nseg, dof) with k <= 4 (cubic pieces at most)")
        if c.shape[1] < 4:
            pad = torch.zeros((c.shape[0], 4 - c.shape[1]) + tuple(c.shape[2:]), dtype=c.dtype, device=c.device)
            c = torch.cat((pad, c), dim=1).contiguous()
        self._set_pieces(breaks, c)
        return self

    def _set_pieces(self, breaks, c):
        """Device form of pieces c [B, k, nseg, dof] (CUDA fp64) over `breaks`; checks the breaks."""
        self.B, _, nseg, self._dof = c.shape
        self.n = nseg + 1
        self.d_ss = engine.as_device(breaks, self.device)
        if self.d_ss.shape[-1] != self.n or self.d_ss.dim() not in (1, 2) or (self.d_ss.dim() == 2 and
                                                                           self.d_ss.shape[0] != self.B):
            raise ValueError("breaks must have shape (nseg + 1,) or (B, nseg + 1)")
        if bool((self.d_ss[..., 1:] <= self.d_ss[..., :-1]).any()):
            raise ValueError("breaks must be strictly increasing")
        self.bc_type = None
        self.ss_host = engine.host_view(breaks)
        self.d_ppoly = c
        self.d_wp = engine.ppoly_eval(self.d_ppoly, self.d_ss, self.d_ss, 0)  # positions at the breaks

    @property
    def dof(self):
        return self._dof

    @property
    def nseg(self):
        return self.n - 1

    def eval_device(self, s, order=0):
        """s: CUDA tensor [G] (shared) or [B, G] -> CUDA tensor [B, G, dof]."""
        if order not in (0, 1, 2):
            raise ValueError("Invalid order %s" % order)
        if isinstance(self.bc_type, str) and self.bc_type == "periodic":
            # scipy sets extrapolate='periodic' for these splines: PPoly.__call__ first maps
            # x -> xmin + (x - xmin) % (xmax - xmin), so the end of the interval evaluates at its start
            torch = engine.torch_mod()
            x0, x1 = self.d_ss[..., :1], self.d_ss[..., -1:]
            s = (x0 + torch.remainder(s - x0, x1 - x0)).contiguous()
        return engine.ppoly_eval(self.d_ppoly, self.d_ss, s, order)

    def __call__(self, path_positions, order=0):
        s = np.atleast_1d(np.asarray(path_positions, dtype=np.float64))
        out = self.eval_device(engine.as_device(s, self.device), order)
        return out.cpu().numpy()

    def propose_gridpoints(self, max_err_threshold=1e-4, max_iteration=100, max_seg_length=0.05, min_nb_points=100,
                           max_points=4096):
        """Adaptive gridpoints for every path of the batch (reference propose_gridpoints, interpolator.py:49-122; one
        warp per path, tb_propose_gridpoints).  The grids are RAGGED: returns (grid [B, Gmax] CUDA tensor padded with
        the path end, glen [B] int32 CUDA tensor); Gmax = longest grid of the batch.  Pass both to
        `BatchTOPPRA(..., gridpoints=grid, glen=glen)`.  Raises ValueError like the reference when a path finds no
        good grid within `max_iteration` passes (or needs more than `max_points` points)."""
        grid, glen, status = engine.propose_gridpoints(self.d_ppoly, self.d_ss, max_err_threshold, max_iteration,
                                                       max_seg_length, min_nb_points, max_points)
        st = status.cpu().numpy()          # one small D2H: the error behaviour of the reference needs the host
        if (st == 1).any():
            raise ValueError("Unable to find a good gridpoint for this path.")
        if (st != 0).any():
            raise ValueError("propose_gridpoints: more than max_points=%d gridpoints needed" % max_points)
        gmax = int(glen.max().item())
        return grid[:, :gmax].contiguous(), glen

    def chunk(self, lo, hi):
        """View of paths [lo, hi) sharing this object's device buffers (used by chunked batch solves)."""
        view = object.__new__(BatchSplineInterpolator)
        view.device, view.n, view._dof, view.bc_type = self.device, self.n, self._dof, self.bc_type
        view.B = hi - lo
        view.d_wp = self.d_wp[lo:hi]
        view.d_ss = self.d_ss if self.d_ss.dim() == 1 else self.d_ss[lo:hi]
        view.ss_host = None if self.ss_host is None else (self.ss_host if self.ss_host.ndim == 1 else self.ss_host[lo:hi])
        view.d_ppoly = self.d_ppoly[lo:hi]
        return view


class BatchPiecewisePolyPath(BatchSplineInterpolator):
    """B paths given as piecewise polynomials with up to 8 coefficients per piece (degree <= 7) in scipy's PPoly layout.

    breaks: (nseg + 1,) shared or (B, nseg + 1), strictly increasing.
    coeffs: (B, k, nseg, dof), 1 <= k <= 8, highest power first, local power basis
            sum_j c[j] (s - breaks[i]) ** (k - 1 - j) like `scipy.interpolate.PPoly.c`.
    device: torch device (default: that of a CUDA `coeffs`, else the current CUDA device)

    Derivatives are those of scipy's derivative objects, `PPoly(c, x).derivative()` and `.derivative().derivative()`,
    bit for bit.  k <= 4 is zero-padded to the cubic form exactly like `BatchSplineInterpolator.from_ppoly` and runs on
    the cubic kernels; 5 <= k <= 8 runs on libtoppra_b200_poly.so (evaluate q', q'' at the gridpoints, build the stage
    records from them, then the record scan).  `BatchTOPPRA` / `BatchTOPPRAsd` accept both; the fused vel+acc scan is
    cubic only.  `order` is k."""

    def __init__(self, breaks, coeffs, device=None):
        torch = engine.torch_mod()
        self.device = engine.default_device(device if device is not None else
                                            (coeffs.device if isinstance(coeffs, torch.Tensor) else None))
        c = engine.as_device(coeffs, self.device)
        if c.dim() != 4 or not 1 <= c.shape[1] <= _lib_poly.MAX_COEFFS:
            raise ValueError("coeffs must have shape (B, k, nseg, dof) with 1 <= k <= %d; got %s"
                             % (_lib_poly.MAX_COEFFS, tuple(c.shape)))
        self.order = int(c.shape[1])
        if self.order <= 4:
            self.__dict__.update(BatchSplineInterpolator.from_ppoly(breaks, c, device=self.device).__dict__)
            return
        self._set_pieces(breaks, c)

    def chunk(self, lo, hi):
        view = object.__new__(BatchPiecewisePolyPath)
        view.__dict__.update(BatchSplineInterpolator.chunk(self, lo, hi).__dict__)
        view.order = self.order
        return view


class SplineInterpolator(AbstractGeometricPath):
    """Interpolate the given waypoints by cubic spline — drop-in for the reference class
    (interpolator.py:360-466): same constructor, `__call__(s, order)`, `.dof`, `.path_interval`, `.duration`,
    `.waypoints`, `.cspl/.cspld/.cspldd` (objects exposing `.c`, `.x` and `__call__`).

    The fit (scipy CubicSpline restated) and every evaluation run on the GPU."""

    def __init__(self, ss_waypoints, waypoints, bc_type="not-a-knot", device=None) -> None:
        super(SplineInterpolator, self).__init__()
        self.ss_waypoints = np.array(ss_waypoints, dtype=np.float64)
        self._q_waypoints = np.array(waypoints, dtype=np.float64)
        assert self.ss_waypoints.shape[0] == self._q_waypoints.shape[0]
        self._scalar_dof = self._q_waypoints.ndim == 1
        self._batch = None
        self._c_host = None
        if len(self.ss_waypoints) > 1:
            wp = self._q_waypoints.reshape(len(self.ss_waypoints), -1)
            self._batch = BatchSplineInterpolator(self.ss_waypoints, wp[None], bc_type=bc_type, device=device)
        self.cspl = _DevicePPoly(self, 0)
        self.cspld = _DevicePPoly(self, 1)
        self.cspldd = _DevicePPoly(self, 2)

    def _coefficients(self):
        if self._batch is None:
            raise ValueError("a single-waypoint path has no polynomial coefficients")
        if self._c_host is None:
            self._c_host = self._batch.d_ppoly[0].cpu().numpy()
        c = self._c_host
        return c[:, :, 0] if self._scalar_dof else c

    def __call__(self, path_positions, order=0):
        scalar_in = np.ndim(path_positions) == 0
        s = np.atleast_1d(np.asarray(path_positions, dtype=np.float64))
        if self._batch is None:
            # single waypoint: constant path (reference interpolator.py:398-417)
            if order == 0:
                out = np.zeros((len(s), self.dof))
                out[:, :] = self._q_waypoints[0]
            elif order in (1, 2):
                out = np.zeros((len(s), self.dof))
            else:
                raise ValueError(f"Invalid order {order}")
        else:
            if order not in (0, 1, 2):
                raise ValueError(f"Invalid order {order}")
            out = self._batch(s.reshape(-1), order)[0].reshape(s.shape + (self._batch.dof,))
        if self._scalar_dof:
            out = out[..., 0]
        if scalar_in:
            out = np.asarray(out[0])   # scipy returns a 0-d ndarray for a scalar path at a scalar position
        return out

    @property
    def waypoints(self):
        """Tuple[np.ndarray, np.ndarray]: positions and waypoints."""
        return self.ss_waypoints, self._q_waypoints

    def get_duration(self):
        return self.duration

    @property
    def duration(self):
        return self.ss_waypoints[-1] - self.ss_waypoints[0]

    @property
    def path_interval(self):
        return np.array([self.ss_waypoints[0], self.ss_waypoints[-1]])

    def get_path_interval(self):
        return self.path_interval

    @property
    def dof(self):
        if np.isscalar(self._q_waypoints[0]):
            return 1
        return self._q_waypoints[0].shape[0]

    # device view used by the constraints / algorithms
    def as_batch(self):
        if self._batch is None:
            raise ValueError("single-waypoint paths cannot be parameterised")
        return self._batch


class PPolyPath(AbstractGeometricPath):
    """A single path given as a piecewise cubic in scipy's PPoly layout ("PPoly in", SURVEY §8 f4): the way other path
    types of the reference (scipy CubicSpline / PPoly objects, the cubic-Hermite `SimplePath`, polynomials up to degree
    3) reach the GPU solver.  `ppoly`: an object with `.c` (k, nseg[, dof]) and `.x` (nseg + 1,), or the pair (c, x)."""

    def __init__(self, ppoly, x=None, device=None):
        super(PPolyPath, self).__init__()
        c = np.asarray(ppoly.c if x is None else ppoly, dtype=np.float64)
        self._x = np.asarray(ppoly.x if x is None else x, dtype=np.float64)
        self._scalar_dof = c.ndim == 2
        if self._scalar_dof:
            c = c[:, :, None]
        if c.ndim != 3:
            raise ValueError("PPoly coefficients must have shape (k, nseg) or (k, nseg, dof)")
        self._batch = self._device_form(self._x, c[None], device)

    @staticmethod
    def _device_form(x, c, device):
        return BatchSplineInterpolator.from_ppoly(x, c, device=device)

    def __call__(self, path_positions, order=0):
        if order not in (0, 1, 2):
            raise ValueError(f"Invalid order {order}")
        scalar_in = np.ndim(path_positions) == 0
        s = np.atleast_1d(np.asarray(path_positions, dtype=np.float64))
        out = self._batch(s.reshape(-1), order)[0].reshape(s.shape + (self._batch.dof,))
        if self._scalar_dof:
            out = out[..., 0]
        return out[0] if scalar_in else out

    @property
    def dof(self):
        return self._batch.dof

    @property
    def path_interval(self):
        return np.array([self._x[0], self._x[-1]])

    @property
    def duration(self):
        return self._x[-1] - self._x[0]

    @property
    def waypoints(self):
        """Breakpoints and the positions there."""
        return self._x, self(self._x)

    def as_batch(self):
        return self._batch


class PiecewisePolyPath(PPolyPath):
    """A single path given as a piecewise polynomial with up to 8 coefficients per piece (degree <= 7) in scipy's PPoly
    layout — the reference's C++ `PiecewisePolyPath` in Python form.  Same surface as `PPolyPath`; `ppoly` is an object
    with `.c` (k, nseg[, dof]) and `.x` (nseg + 1,), or the pair (c, x).  Values and derivatives equal scipy's
    `PPoly(c, x)`, `.derivative()` and `.derivative().derivative()` bit for bit, so `TOPPRA(constraints, path)` gives
    the reference's result for a path object with that convention.

    Quintic paths from scipy::

        from scipy.interpolate import BPoly, PPoly, make_interp_spline
        path = PiecewisePolyPath(PPoly.from_spline(make_interp_spline(ss, qs, k=5)))
        # quintic Hermite through positions, velocities and accelerations; yi[i] = [q_i, qd_i, qdd_i] per joint
        path = PiecewisePolyPath(PPoly.from_bernstein_basis(BPoly.from_derivatives(ss, yi)))

    `PPoly.from_spline` keeps the B-spline's full knot vector, whose outer pieces have zero length; pass
    `(pp.c[:, k:-k], pp.x[k:-k])` (k = 5 here) to keep the pieces inside the interval, where the breaks increase
    strictly."""

    @staticmethod
    def _device_form(x, c, device):
        return BatchPiecewisePolyPath(x, c, device=device)

    @property
    def order(self):
        """Coefficients per piece (degree + 1)."""
        return self._batch.order


class PolynomialPath(PPolyPath):
    """Polynomial path coeff[i, 0] + coeff[i, 1] s + coeff[i, 2] s^2 + ... on [s_start, s_end] — public surface of the
    reference's `PolynomialPath` (interpolator.py:584-686).  The GPU evaluation works on cubic pieces, so the degree is
    limited to 3 here; the polynomial is re-expanded about `s_start` (one piece), values agree with the reference to
    rounding."""

    def __init__(self, coeff, s_start=0.0, s_end=1.0, device=None):
        self.s_start, self.s_end = s_start, s_end
        scalar = np.isscalar(coeff[0])
        polys = [np.polynomial.Polynomial(np.asarray(c, dtype=np.float64)) for c in ([coeff] if scalar else coeff)]
        if max(p.degree() for p in polys) > 3:
            raise NotImplementedError("toppra_b200: PolynomialPath is limited to degree 3 (cubic pieces on the GPU)")
        self.coeff = np.array(coeff).reshape(1, -1) if scalar else coeff
        self.poly = polys
        cols = []
        for p in polys:  # Taylor coefficients at s_start, highest power first
            cols.append([p.deriv(3)(s_start) / 6.0, p.deriv(2)(s_start) / 2.0, p.deriv(1)(s_start), p(s_start)])
        c = np.array(cols, dtype=np.float64).T[:, None, :]          # (4, 1 piece, dof)
        super(PolynomialPath, self).__init__(c, np.array([s_start, s_end], dtype=np.float64), device=device)
        self._flat = scalar

    def __call__(self, path_positions, order=0):
        out = super(PolynomialPath, self).__call__(path_positions, order)
        if self._flat:  # 1-D coefficient list: the reference returns flattened arrays (interpolator.py:666-686)
            return np.atleast_1d(out[..., 0])
        return out

    @property
    def duration(self):
        return self.s_end - self.s_start

    # deprecated accessors the reference still carries (interpolator.py:652-665)
    @deprecated
    def get_path_interval(self):
        return self.path_interval

    @deprecated
    def get_duration(self):
        return self.duration

    @deprecated
    def get_dof(self):
        return self.dof


class UnivariateSplineInterpolator(PPolyPath):
    """Waypoints smoothed by one cubic smoothing spline per joint — public surface of the reference's
    `UnivariateSplineInterpolator` (interpolator.py:508-581).

    The smoothing fit is scipy's `UnivariateSpline` (FITPACK), exactly the call the reference makes; it is one-off host
    data preparation.  The fitted splines are cubic, so they reach the GPU as "PPoly in": each joint's B-spline is converted
    to piecewise-cubic form, the joints' knot sets are merged (FITPACK places knots per joint), and solving / evaluation
    run on the device like for any other path.  Values agree with the reference to rounding (the conversion re-expands
    each piece about its left breakpoint)."""

    def __init__(self, ss_waypoints, waypoints, device=None):
        from scipy.interpolate import PPoly, UnivariateSpline
        assert ss_waypoints[0] == 0, "First index must equals zero."
        self.ss_waypoints = np.array(ss_waypoints, dtype=np.float64)
        q = np.array(waypoints, dtype=np.float64)
        self._q_waypoints = q
        cols = q.reshape(-1, 1) if q.ndim == 1 else q
        assert self.ss_waypoints.shape[0] == cols.shape[0]
        self.uspl = [UnivariateSpline(self.ss_waypoints, cols[:, i]) for i in range(cols.shape[1])]
        pieces = [PPoly.from_spline(spl._eval_args) for spl in self.uspl]
        lo, hi = self.ss_waypoints[0], self.ss_waypoints[-1]
        knots = np.unique(np.concatenate([p.x for p in pieces] + [[lo, hi]]))
        knots = knots[(knots >= lo) & (knots <= hi)]
        c = np.empty((4, len(knots) - 1, cols.shape[1]))
        for k, p in enumerate(pieces):      # Taylor coefficients at each left breakpoint (PPoly evaluates the right piece)
            left = knots[:-1]
            c[0, :, k], c[1, :, k] = p(left, 3) / 6.0, p(left, 2) / 2.0
            c[2, :, k], c[3, :, k] = p(left, 1), p(left)
        super(UnivariateSplineInterpolator, self).__init__(c, knots, device=device)

    @property
    def waypoints(self):
        return self.ss_waypoints, self._q_waypoints
