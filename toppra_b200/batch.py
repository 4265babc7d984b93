"""Batched TOPP-RA: B independent paths per launch.  There is no reference equivalent (the reference solves one
path per Python object); the per-path semantics are exactly those of
`TOPPRA(constraints, path, gridpoints, solver_wrapper="seidel").compute_parameterization(sd_start, sd_end)`
(reference reachability_algorithm.py:240-376), see csrc/tb_scan.cu."""
import numpy as np

from . import engine
from .constraint import (ConstraintType, JointAccelerationConstraint, JointVelocityConstraint, RecordContext)
from .exceptions import BadInputVelocities
from .interpolator import BatchSplineInterpolator


def conic_info(ctx, constraints):
    """(row0, nrows, ellipsoid) of the robust constraint of the list, or None."""
    row0 = 0
    for c in constraints:
        n = c.num_rows(ctx)
        if c.get_constraint_type() == ConstraintType.CanonicalConic:
            return row0, n, c.ellipsoid()
        row0 += n
    return None


def ragged(glen):
    """Keyword arguments that make an engine call ragged: none on a common grid length, so those calls stay as they are."""
    return {} if glen is None else {"glen": glen}


def scan_any(records, R, grid, conic, sd_start=None, sd_end=None, sd_end_hi=None, backward_only=False,
             counters=False, fast_lower=False, glen=None):
    """K2 for purely linear problems, K2r when a robust constraint is present."""
    if conic is None:
        return engine.scan(records, R, grid, sd_start, sd_end, sd_end_hi, backward_only, counters,
                           fast_lower=fast_lower, glen=glen)
    if sd_end_hi is not None:
        raise NotImplementedError("robust problems: compute_controllable_sets needs sdmin == sdmax")
    return engine.scan_robust(records, R, conic[0], conic[1], conic[2], grid, sd_start, sd_end, backward_only, counters,
                              **ragged(glen))


def build_records(ctx, constraints, out=None):
    """Stage records [B, G, W] for a list of CanonicalLinear constraints (= seidelWrapper.__init__,
    cy_seidel_solverwrapper.pyx:425-531).  Returns (records, R).  `out`: optional preallocated buffer whose first
    ctx.B records are (re)used (chunked solves)."""
    conic = [c for c in constraints if c.get_constraint_type() == ConstraintType.CanonicalConic]
    if len(conic) > 1:
        raise NotImplementedError("toppra_b200: at most one robust (conic) constraint per problem")
    for c in constraints:
        if c.get_constraint_type() not in (ConstraintType.CanonicalLinear, ConstraintType.CanonicalConic):
            raise NotImplementedError("constraint type %s cannot be turned into stage rows" % c.get_constraint_type())
    rows = [c.num_rows(ctx) for c in constraints]
    R = int(sum(rows))
    ubound = any(getattr(c, "has_ubound", lambda _ctx: False)(ctx) for c in constraints)
    if ubound and conic:
        raise NotImplementedError("toppra_b200: a constraint with a ubound next to a robust (conic) constraint")
    if out is not None:
        records = out[:ctx.B]
    else:
        records, _ = engine.alloc_records(ctx.B, ctx.G, R, ctx.device, ubound=ubound)
    kinds = [type(c) for c in constraints]
    fused_pair = ()
    if kinds.count(JointVelocityConstraint) == 1 and kinds.count(JointAccelerationConstraint) == 1:
        # one K1 launch writes the velocity bound AND the acceleration rows (wherever the two sit in the list); it also
        # initialises the bound slots and the padding, so no separate init pass is needed
        iv, ia = kinds.index(JointVelocityConstraint), kinds.index(JointAccelerationConstraint)
        vel, acc = constraints[iv], constraints[ia]
        for c in (vel, acc):
            if ctx.bpath.dof != c.get_dof():
                raise ValueError("Wrong dimension: constraint dof ({:d}) not equal to path dof ({:d})".format(
                    c.get_dof(), ctx.bpath.dof))
        if ubound:
            engine.init_bounds(records, R)     # the u-bound pair is not written by K1
        engine.coeff_velacc(ctx.bpath.d_ppoly, ctx.bpath.d_ss, ctx.d_grid, ctx.limits(vel.device_limits(ctx.device)),
                            ctx.limits(acc.device_limits(ctx.device)), acc.interpolation, records, R, int(sum(rows[:ia])), 1)
        fused_pair = (iv, ia)
        if len(constraints) == 2:
            return records, R
    else:
        engine.init_bounds(records, R)
    row0 = 0
    for i, (c, n) in enumerate(zip(constraints, rows)):
        if i not in fused_pair:
            c.append_records(ctx, records, R, row0)
        row0 += n
    return records, R


_COPY_STREAMS = {}


def copy_stream(device):
    """One device-to-host copy stream per device, shared by every solve: copies of consecutive solves stay ordered."""
    torch = engine.torch_mod()
    key = str(device)
    if key not in _COPY_STREAMS:
        _COPY_STREAMS[key] = torch.cuda.Stream(device)
    return _COPY_STREAMS[key]


class BatchResult(object):
    """Device-resident result of BatchTOPPRA.compute_parameterization.

    K [B,G,2] controllable sets, sd [B,G] path velocities, sdd [B,G-1] path accelerations (u),
    status [B] int32 (toppra_b200.algorithm.STATUS_CODES order), fail_stage [B] int32."""

    def __init__(self, out):
        self.K = out["K"]
        self.sd = out["sd"]
        self.sdd = out["u"]
        self.status = out["status"]
        self.fail_stage = out["fail_stage"]
        self.counters = out.get("counters")

    def to_host(self, pinned=None):
        """Copy to host.  `pinned`: optional dict of preallocated pinned tensors with the same keys."""
        torch = engine.torch_mod()
        host = {}
        for key in ("K", "sd", "sdd", "status", "fail_stage"):
            t = getattr(self, key)
            if pinned is not None and key in pinned:
                pinned[key].copy_(t, non_blocking=True)
                host[key] = pinned[key]
            else:
                host[key] = t.to("cpu", non_blocking=False)
        torch.cuda.current_stream().synchronize()
        return {k: v.numpy() for k, v in host.items()}


class BatchTOPPRA(object):
    """Time-optimal parameterisation of B independent paths on one GPU.

    Parameters
    ----------
    constraint_list: list of toppra_b200.constraint objects (limits shared by all paths, or batched
        (B, dof, 2) limits).
    path: BatchSplineInterpolator (or BatchPiecewisePolyPath)
    gridpoints: (G,) shared by all paths, or (B, G); must start/end at the path interval.
    """

    def __init__(self, constraint_list, path, gridpoints=None, max_record_bytes=32 << 30, exact=True, validate=True,
                 fused=None, glen=None, gridpt_max_err_threshold=1e-3, gridpt_min_nb_points=100):
        if not isinstance(path, BatchSplineInterpolator):
            raise TypeError("BatchTOPPRA needs a BatchSplineInterpolator")
        torch = engine.torch_mod()
        self.constraints = constraint_list
        self.path = path
        self.device = path.device
        if gridpoints is None:
            # reference algorithm.py:100-106: gridpoints proposed per path (interpolator.propose_gridpoints) -> RAGGED
            # grids [B, Gmax] + lengths, solved in one launch (tb_scan_ragged / tb_scan_velacc_ragged)
            gridpoints, glen = path.propose_gridpoints(max_err_threshold=gridpt_max_err_threshold,
                                                       min_nb_points=gridpt_min_nb_points)
            validate = False   # the proposed grids span the path interval and increase by construction
        self.glen = None if glen is None else engine.as_device(glen, self.device, dtype=torch.int32)
        gp = engine.host_view(gridpoints)  # None for CUDA tensors
        grid_host = gp if (gp is not None and gp.ndim == 1) else None
        self.d_grid = engine.as_device(gridpoints, self.device)
        if self.d_grid.dim() not in (1, 2) or (self.d_grid.dim() == 2 and self.d_grid.shape[0] != path.B):
            raise ValueError("gridpoints must have shape (G,) or (B, G)")
        if self.glen is not None:
            engine.check_glen(self.glen, path.B, self.d_grid)
        if validate and self.glen is not None:
            # ragged grids: the last REAL gridpoint of every path must be the end of its interval; padding is ignored
            g, ss = self.d_grid, path.d_ss
            last = torch.gather(g, 1, (self.glen.to(torch.int64) - 1).clamp(min=0).unsqueeze(1))[:, 0]
            col = torch.arange(g.shape[1], device=g.device).unsqueeze(0)
            real = col[:, 1:] < self.glen.unsqueeze(1)
            t = ((g[:, 0] != ss[..., 0]).any() | (last != ss[..., -1]).any()).to(torch.int32)
            t = t + 2 * ((g[:, 1:] <= g[:, :-1]) & real).any().to(torch.int32)
            code = int(t)
            if code & 1:
                raise ValueError("Invalid manually supplied gridpoints.")
            if code & 2:
                raise ValueError("Bad input gridpoints.")
        elif validate:
            # reference algorithm.py:107-120: gridpoints must span exactly the path interval ("Invalid manually supplied
            # gridpoints.") and increase strictly ("Bad input gridpoints.").  Host data is checked on the host (no
            # device synchronisation); CUDA tensors with one small reduction.
            ss_host = getattr(path, "ss_host", None)
            if gp is not None and ss_host is not None:
                code = int(np.any(gp[..., 0] != ss_host[..., 0]) or np.any(gp[..., -1] != ss_host[..., -1]))
                code += 2 * int(np.any(np.diff(gp, axis=-1) <= 0))
            else:
                g, ss = self.d_grid, path.d_ss
                t = ((g[..., 0] != ss[..., 0]).any() | (g[..., -1] != ss[..., -1]).any()).to(torch.int32)
                if g.shape[-1] > 1:
                    t = t + 2 * (g[..., 1:] <= g[..., :-1]).any().to(torch.int32)
                code = int(t)
            if code & 1:
                raise ValueError("Invalid manually supplied gridpoints.")
            if code & 2:
                raise ValueError("Bad input gridpoints.")
        for c in constraint_list:  # per-path limit arrays must cover exactly this batch (raw pointers go to the kernels)
            for name in ("vlim", "alim"):
                lim = getattr(c, name, None)
                if isinstance(lim, np.ndarray) and (lim.shape[-2] != path.dof or (lim.ndim == 3 and lim.shape[0] != path.B)):
                    raise ValueError("%s.%s has shape %s; expected (%d, 2) or (%d, %d, 2)"
                                     % (type(c).__name__, name, lim.shape, path.dof, path.B, path.dof))
        self.ctx = RecordContext(path, self.d_grid, grid_host, None)
        self.records = None
        try:  # static LP rows per stage (nC = R + 2); user-defined constraints report theirs at setup()
            self.R = int(sum(c.num_rows(self.ctx) for c in constraint_list))
        except NotImplementedError:
            self.R = None
        # Stage records cost 8 * (3R + 2) * G bytes per path (138 KB at 7-DOF / 200 gridpoints): batches whose
        # records exceed `max_record_bytes` are solved in chunks through one reused record buffer.
        self.max_record_bytes = int(max_record_bytes)
        # exact=True (default): bit-identical to the reference's seidelWrapper.  exact=False: the min-x LP of the
        # backward pass takes the shortcut TB_SCAN_FAST_LOWER (include/toppra_b200.h): same LP optimum, deviations
        # from the reference's rounding noise <= ~1e-15, about 1.7x faster.
        self.exact = bool(exact)
        self._grid_host = grid_host
        self.conic = conic_info(self.ctx, self.constraints)
        # JointVelocity (optional) + JointAcceleration: the scan builds the LP rows itself from the spline
        # (tb_scan_velacc, K1 fused into K2): no stage records, no chunking.  fused=False forces the record path.
        kinds = [type(c) for c in constraint_list]
        self.fused = (fused is not False and sorted(k.__name__ for k in kinds) in
                      (["JointAccelerationConstraint"], ["JointAccelerationConstraint", "JointVelocityConstraint"])
                      and engine.is_cubic(path.d_ppoly)
                      and engine.velacc_fused_supported(path.nseg, path.dof,
                                                        constraint_list[kinds.index(JointAccelerationConstraint)].interpolation))
        if fused and not self.fused:
            raise ValueError("fused=True needs a [JointVelocityConstraint,] JointAccelerationConstraint problem on a "
                             "piecewise-cubic path that fits one LP row per lane (see tb_scan_velacc)")
        self.xbound = None

    @property
    def B(self):
        return self.path.B

    @property
    def G(self):
        return self.d_grid.shape[-1]

    def setup(self):
        """K1: constraint coefficients -> stage records (done once; reused by every solve).  Fused vel+acc problems
        only need the velocity bound xbound [B, G, 2]."""
        if self.fused:
            kinds = [type(c) for c in self.constraints]
            acc = self.constraints[kinds.index(JointAccelerationConstraint)]
            vel = self.constraints[kinds.index(JointVelocityConstraint)] if JointVelocityConstraint in kinds else None
            for c in self.constraints:
                if self.path.dof != c.get_dof():
                    raise ValueError("Wrong dimension: constraint dof ({:d}) not equal to path dof ({:d})".format(
                        c.get_dof(), self.path.dof))
            self._alim = acc.device_limits(self.device)
            self._interp = acc.interpolation
            self.R = acc.num_rows(self.ctx)
            self.xbound = engine.xbound_velocity(self.path.d_ppoly, self.path.d_ss, self.d_grid,
                                                 None if vel is None else vel.device_limits(self.device))
            return self.xbound
        self.records, self.R = build_records(self.ctx, self.constraints)
        return self.records

    def _ready(self):
        if (self.xbound if self.fused else self.records) is None:
            self.setup()

    def _scan(self, s0, s1, sd_end_hi=None, **kw):
        """One scan launch over the whole batch on whatever row source this problem uses."""
        self._ready()
        if self.fused:
            return engine.scan_velacc(self.path.d_ppoly, self.path.d_ss, self.d_grid, self._alim, self._interp,
                                      self.xbound, s0, s1, sd_end_hi, fast_lower=not self.exact, glen=self.glen, **kw)
        if self.conic is None:
            return engine.scan(self.records, self.R, self.d_grid, s0, s1, sd_end_hi, fast_lower=not self.exact,
                               glen=self.glen, **kw)
        if sd_end_hi is not None:
            raise NotImplementedError("robust problems: compute_controllable_sets needs sdmin == sdmax")
        kw.pop("forward_from", None)
        return engine.scan_robust(self.records, self.R, self.conic[0], self.conic[1], self.conic[2], self.d_grid, s0, s1,
                                  kw.get("backward_only", False), kw.get("counters", False), **ragged(self.glen))

    def _vel_tensor(self, v):
        if v is None:
            return None
        torch = engine.torch_mod()
        if isinstance(v, torch.Tensor):
            t = engine.as_device(v, self.device)
            if t.dim() == 0:
                t = t.expand(self.B).contiguous()
            if tuple(t.shape) != (self.B,):
                raise ValueError("boundary velocities must be scalars or have shape (B,)")
            if bool((t < 0).any()):
                raise BadInputVelocities("Negative path velocities: path velocities must be positive")
            return t
        arr = np.broadcast_to(np.asarray(v, dtype=np.float64), (self.B,))
        if np.any(arr < 0):
            raise BadInputVelocities("Negative path velocities: path velocities must be positive")
        if not np.any(arr != 0):
            return None  # kernels treat NULL as zeros
        return engine.as_device(np.ascontiguousarray(arr), self.device)

    def _pinned_outputs(self, pinned):
        """Complete `pinned` (a dict, possibly empty / None) to the full set of pinned result tensors."""
        torch = engine.torch_mod()
        B, G = self.B, self.G
        shapes = {"K": ((B, G, 2), torch.float64), "sd": ((B, G), torch.float64), "sdd": ((B, G - 1), torch.float64),
                  "status": ((B,), torch.int32), "fail_stage": ((B,), torch.int32)}
        pinned = {} if pinned is None else pinned
        for key, (shape, dt) in shapes.items():
            if key not in pinned:
                pinned[key] = torch.empty(shape, dtype=dt).pin_memory()
        return pinned

    def solve_to_host(self, sd_start=0.0, sd_end=0.0, pinned=None, sync=True):
        """compute_parameterization + copy of (K, sd, sdd, status, fail_stage) to pinned host memory, with the D2H
        copy of K overlapped with the forward pass: the scan runs as a backward-only and a forward-only launch and K
        leaves on a second stream in between.  Returns the dict of pinned host TENSORS (same keys and types for every
        problem kind: chunked and robust problems take the plain path).  sync=True (default): the host waits for the
        copies, the buffers are valid on return.  sync=False (pipelined callers): nothing is waited for and all copies
        run on the package's copy stream (`batch.copy_stream(device)`), so the next solve's kernels overlap them; the
        buffers are valid once `self.host_ready` (a CUDA event recorded after the last copy) has completed —
        `inst.host_ready.synchronize()`."""
        torch = engine.torch_mod()
        pinned = self._pinned_outputs(pinned)
        main = torch.cuda.current_stream(self.device)
        if self.conic is not None or self.chunk_size() < self.B:
            res = self.compute_parameterization(sd_start, sd_end)
            for key in pinned:
                pinned[key].copy_(getattr(res, key), non_blocking=True)
            self.last_result = res
            self.host_ready = torch.cuda.Event()
            self.host_ready.record(main)
            if sync:
                self.host_ready.synchronize()
            return pinned
        s0, s1 = self._vel_tensor(sd_start), self._vel_tensor(sd_end)
        copy = copy_stream(self.device)
        self._copy_stream = copy
        back = self._scan(s0, s1, backward_only=True)
        ev = torch.cuda.Event()
        ev.record(main)
        with torch.cuda.stream(copy):
            copy.wait_event(ev)
            pinned["K"].copy_(back["K"], non_blocking=True)
        back["K"].record_stream(copy)
        fwd = self._scan(s0, s1, forward_from=back)
        self.last_result = BatchResult(fwd)
        if sync:
            # the host waits for this solve: the small results follow the forward launch on the caller's stream
            pinned["sd"].copy_(fwd["sd"], non_blocking=True)
            pinned["sdd"].copy_(fwd["u"], non_blocking=True)
            pinned["status"].copy_(fwd["status"], non_blocking=True)
            pinned["fail_stage"].copy_(fwd["fail_stage"], non_blocking=True)
            main.wait_stream(copy)            # the step is complete (for events / callers) when K has landed too
            self.host_ready = torch.cuda.Event()
            self.host_ready.record(main)
            self.host_ready.synchronize()     # host-visible: every copy above has landed
            return pinned
        # pipelined caller: EVERY device-to-host copy goes to the copy stream, so the caller's stream is free for the next
        # solve at once (its kernels overlap these copies); the buffers are valid at `self.host_ready`.  Callers that keep
        # more than one solve in flight alternate between two sets of pinned buffers.
        done = torch.cuda.Event()
        done.record(main)
        with torch.cuda.stream(copy):
            copy.wait_event(done)
            pinned["sd"].copy_(fwd["sd"], non_blocking=True)
            pinned["sdd"].copy_(fwd["u"], non_blocking=True)
            pinned["status"].copy_(fwd["status"], non_blocking=True)
            pinned["fail_stage"].copy_(fwd["fail_stage"], non_blocking=True)
            self.host_ready = torch.cuda.Event()
            self.host_ready.record(copy)
        for key in ("sd", "u", "status", "fail_stage"):
            fwd[key].record_stream(copy)
        return pinned

    def chunk_size(self):
        """Paths per chunk so that the record buffer stays within max_record_bytes."""
        if self.fused:
            return self.B  # no stage records
        return self.record_chunk_size()

    def record_chunk_size(self):
        """Paths per chunk of the methods that always read stage records (feasible and reachable sets), fused or not."""
        rows = sum(c.num_rows(self.ctx) for c in self.constraints)
        per_path = 8 * engine.record_doubles(rows) * self.G
        return max(1, min(self.B, self.max_record_bytes // per_path))

    def _chunked(self, nchunk, shapes, solve):
        """Solve the batch in chunks of `nchunk` paths through ONE record buffer.  Per chunk [lo, hi): its records are built
        (K1) into the buffer, then solve(lo, hi, records, grid, glen) returns a dict of that chunk's results, which are
        written into full-batch tensors.  shapes: {key: (shape, dtype)} of those tensors."""
        torch = engine.torch_mod()
        out = {key: torch.empty(shape, dtype=dt, device=self.device) for key, (shape, dt) in shapes.items()}
        buf = None
        for lo in range(0, self.B, nchunk):
            hi = min(self.B, lo + nchunk)
            grid = self.d_grid if self.d_grid.dim() == 1 else self.d_grid[lo:hi]
            glen = None if self.glen is None else self.glen[lo:hi].contiguous()   # ragged grids: the chunk's lengths
            ctx = RecordContext(self.path.chunk(lo, hi), grid, self._grid_host, None, lo, hi, self.B)
            if buf is None:
                buf, self.R = build_records(ctx, self.constraints)
                rec = buf
            else:
                rec, _ = build_records(ctx, self.constraints, out=buf)
            part = solve(lo, hi, rec, grid, glen)
            for key in out:
                out[key][lo:hi] = part[key]
        return out

    def _shapes(self, *keys):
        """{key: (shape, dtype)} of full-batch results."""
        torch = engine.torch_mod()
        B, G = self.B, self.G
        table = {"K": ((B, G, 2), torch.float64), "X": ((B, G, 2), torch.float64), "L": ((B, G, 2), torch.float64),
                 "sd": ((B, G), torch.float64), "u": ((B, G - 1), torch.float64), "info": ((B, 4), torch.float64),
                 "status": ((B,), torch.int32), "fail_stage": ((B,), torch.int32), "counters": ((B, 4), torch.int32)}
        return {key: table[key] for key in keys}

    def _records(self):
        """The whole batch's stage records, built once (also for problems whose scan is fused)."""
        if self.records is None:
            self.records, self.R = build_records(self.ctx, self.constraints)
        return self.records

    def compute_parameterization(self, sd_start=0.0, sd_end=0.0, counters=False):
        """Backward + forward pass for all paths (K1 + K2).  Returns a BatchResult (device tensors).
        Large batches run in chunks of `chunk_size()` paths (K1 -> K2 per chunk, one record buffer)."""
        s0, s1 = self._vel_tensor(sd_start), self._vel_tensor(sd_end)
        nchunk = self.chunk_size()
        if nchunk >= self.B:
            return BatchResult(self._scan(s0, s1, counters=counters))
        keys = ("K", "sd", "u", "status", "fail_stage") + (("counters",) if counters else ())
        return BatchResult(self._chunked(nchunk, self._shapes(*keys), lambda lo, hi, rec, grid, glen: scan_any(
            rec, self.R, grid, self.conic, _rows(s0, lo, hi), _rows(s1, lo, hi), counters=counters,
            fast_lower=not self.exact, glen=glen)))

    def compute_controllable_sets(self, sdmin, sdmax):
        """K[B,G,2] with K[N] = [sdmin^2, sdmax^2] (reference reachability_algorithm.py:166-202) and status."""
        lo = np.ascontiguousarray(np.broadcast_to(np.asarray(sdmin, dtype=np.float64), (self.B,)))
        hi = np.ascontiguousarray(np.broadcast_to(np.asarray(sdmax, dtype=np.float64), (self.B,)))
        assert np.all(lo <= hi) and np.all(0 <= lo)
        same = bool(np.all(lo == hi))
        s1, s1_hi = engine.as_device(lo, self.device), None if same else engine.as_device(hi, self.device)
        nchunk = self.chunk_size()
        if nchunk >= self.B:
            out = self._scan(None, s1, s1_hi, backward_only=True)
        else:
            out = self._chunked(nchunk, self._shapes("K", "status"), lambda a, b, rec, grid, glen: scan_any(
                rec, self.R, grid, self.conic, None, s1[a:b], _rows(s1_hi, a, b), backward_only=True,
                fast_lower=not self.exact, glen=glen))
        return out["K"], out["status"]

    def compute_reachable_sets(self, sdmin, sdmax):
        """Reachable sets L [B, G, 2] of every path (reference compute_reachable_sets, reachability_algorithm.py:378-431)
        in one launch of tb_reachable_sets (feasible-set pass + forward recursion) per record chunk.
        Returns (L, X, fail_stage)."""
        if self.conic is not None:
            raise NotImplementedError("compute_reachable_sets: linear problems only")
        lo = np.ascontiguousarray(np.broadcast_to(np.asarray(sdmin, dtype=np.float64), (self.B,)))
        hi = np.ascontiguousarray(np.broadcast_to(np.asarray(sdmax, dtype=np.float64), (self.B,)))
        assert np.all(lo <= hi) and np.all(0 <= lo)
        lo, hi = engine.as_device(lo, self.device), engine.as_device(hi, self.device)
        nchunk = self.record_chunk_size()
        if nchunk >= self.B:
            out = engine.reachable_sets(self._records(), self.R, self.d_grid, lo, hi, **ragged(self.glen))
        else:
            out = self._chunked(nchunk, self._shapes("L", "X", "fail_stage"), lambda a, b, rec, grid, glen:
                                engine.reachable_sets(rec, self.R, grid, lo[a:b], hi[a:b], **ragged(glen)))
        return out["L"], out["X"], out["fail_stage"]

    def compute_feasible_sets(self):
        """Feasible sets X [B, G, 2] of every path (reference compute_feasible_sets, reachability_algorithm.py:131-164),
        per record chunk."""
        def solve(lo, hi, rec, grid, glen):
            if self.conic is not None:
                return engine.scan_robust(rec, self.R, self.conic[0], self.conic[1], self.conic[2], grid,
                                          feasible_sets=True, **ragged(glen))
            return dict(K=engine.feasible_sets(rec, self.R, grid, **ragged(glen)))

        nchunk = self.record_chunk_size()
        if nchunk >= self.B:
            return solve(0, self.B, self._records(), self.d_grid, self.glen)["K"]
        return self._chunked(nchunk, self._shapes("K"), solve)["K"]


class BatchTOPPRAsd(BatchTOPPRA):
    """TOPPRAsd (reference desired_duration_algorithm.py:20-234) for B paths: every path gets the convex combination of
    its fastest and slowest parameterisation whose duration is `desired_duration` (scalar or [B]); unachievable
    durations return the fastest / slowest one.  Three launches: two scans (TB_SCAN_SD_FORWARD [| TB_SCAN_SD_SLOW]) and
    the per-path bisection tb_sd_bisect (csrc/tb_frows.cu).  Problems with a robust (conic) constraint run the conic
    backward pass once (tb_scan_robust, backward only), both forward passes in one launch of tbr_sd_forward_robust
    (csrc/tb_conic.cu), then tb_sd_bisect."""

    def set_desired_duration(self, desired_duration):
        self.desired_duration = desired_duration

    def compute_parameterization(self, sd_start=0.0, sd_end=0.0, atol=1e-5):
        s0, s1 = self._vel_tensor(sd_start), self._vel_tensor(sd_end)
        want = np.ascontiguousarray(np.broadcast_to(np.asarray(self.desired_duration, dtype=np.float64), (self.B,)))
        want = engine.as_device(want, self.device)

        def solve(lo, hi, rec, grid, glen):
            a, b = _rows(s0, lo, hi), _rows(s1, lo, hi)
            if self.conic is not None:
                fast, slow = sd_passes_robust(self._records() if rec is None else rec, self.R, self.conic, grid, a, b,
                                              glen)
            elif rec is None:   # the whole batch on this problem's own row source
                fast, slow = self._scan(a, b, sd_forward="fast"), self._scan(a, b, sd_forward="slow")
            else:
                fast, slow = (engine.scan(rec, self.R, grid, a, b, sd_forward=mode, fast_lower=not self.exact,
                                          **ragged(glen)) for mode in ("fast", "slow"))
            out = engine.sd_bisect(fast["sd"], fast["u"], slow["sd"], slow["u"], grid, want[lo:hi], atol,
                                   status_in=fast["status"], **ragged(glen))
            return dict(K=fast["K"], sd=out["sd"], u=out["u"], status=out["status"], fail_stage=fast["fail_stage"],
                        info=out["info"])

        nchunk = self.chunk_size()
        if nchunk >= self.B:
            out = solve(0, self.B, None, self.d_grid, self.glen)
        else:
            out = self._chunked(nchunk, self._shapes("K", "sd", "u", "status", "fail_stage", "info"), solve)
        res = BatchResult(out)
        res.alpha, res.duration_fast, res.duration_slow = out["info"][:, 0], out["info"][:, 1], out["info"][:, 2]
        return res


def _rows(t, lo, hi):
    """Rows [lo, hi) of a per-path tensor, or None."""
    return None if t is None else t[lo:hi]


def sd_passes_robust(records, R, conic, grid, sd_start, sd_end, glen=None):
    """TOPPRAsd's fastest and slowest pass of robust problems: the conic backward pass once (tb_scan_robust, backward
    only), then both forward passes in one tbr_sd_forward_robust launch.  Returns (fast, slow) in the form of
    engine.scan(..., sd_forward=...): K, sd (= x = sd^2), u, status, fail_stage (K / status / fail_stage in `fast`)."""
    back = engine.scan_robust(records, R, conic[0], conic[1], conic[2], grid, None, sd_end, backward_only=True,
                              **ragged(glen))
    fwd = engine.sd_forward_robust(records, R, conic[0], conic[1], conic[2], grid, back["K"], back["status"], sd_start,
                                   **ragged(glen))
    fast = dict(K=back["K"], sd=fwd["x_fast"], u=fwd["u_fast"], status=fwd["status"], fail_stage=fwd["fail_stage"])
    return fast, dict(sd=fwd["x_slow"], u=fwd["u_slow"])


def solve_batch(ss_waypoints, waypoints, gridpoints, vlim, alim, sd_start=0.0, sd_end=0.0,
                discretization_scheme=1, device=None):
    """One-call convenience: fit B splines, build vel+acc records, scan.  Inputs numpy or tensors."""
    path = BatchSplineInterpolator(ss_waypoints, waypoints, device=device)
    cons = [JointVelocityConstraint(vlim), JointAccelerationConstraint(alim, discretization_scheme)]
    inst = BatchTOPPRA(cons, path, gridpoints)
    return inst.compute_parameterization(sd_start, sd_end)
