"""Thin tensor-level front-end of the C-ABI (toppra_b200/_lib.py -> libtoppra_b200.so).

PyTorch is used for storage (device tensors), streams and H2D/D2H copies only; every number is computed by the
hand-written sm_90a kernels in toppra_b200/csrc.  No function here has a CPU fallback."""
import ctypes

import numpy as np

from . import _lib, _lib_cones, _lib_poly, _lib_reach, _lib_robust

BC_KINDS = {"not-a-knot": 0, "clamped": 1, "natural": 2, "periodic": 3}


def torch_mod():
    return _lib.require_cuda()


def as_device(x, device, dtype=None):
    """numpy / tensor -> contiguous fp64 CUDA tensor."""
    torch = torch_mod()
    dtype = dtype or torch.float64
    if isinstance(x, torch.Tensor):
        return x.to(device=device, dtype=dtype, non_blocking=True).contiguous()
    arr = np.ascontiguousarray(x)
    if not arr.flags.writeable:  # e.g. broadcast views: torch wants a writable buffer
        arr = arr.copy()
    return torch.as_tensor(arr, dtype=dtype).to(device, non_blocking=True).contiguous()


def host_view(x):
    """numpy view of host data (numpy array, sequence, or CPU tensor); None for CUDA tensors (no sync here)."""
    torch = torch_mod()
    if isinstance(x, torch.Tensor):
        return None if x.is_cuda else x.detach().numpy()
    return np.asarray(x, dtype=np.float64)


def default_device(device=None):
    torch = torch_mod()
    if device is None:
        return torch.device("cuda", torch.cuda.current_device())
    return torch.device(device)


def parse_bc(bc_type, B, dof, device):
    """scipy CubicSpline bc_type -> ((kind0, val0), (kind1, val1)) with device value tensors [B, dof] or None."""
    if isinstance(bc_type, str):
        if bc_type not in BC_KINDS:
            raise ValueError("bc_type=%r not understood" % (bc_type,))
        return (BC_KINDS[bc_type], None), (BC_KINDS[bc_type], None)
    out = []
    for side in bc_type:
        if isinstance(side, str):
            if side == "periodic":   # scipy _validate_bc
                raise ValueError("'periodic' `bc_type` is defined for both curve ends and cannot be used with other "
                                 "boundary conditions.")
            if side not in BC_KINDS:
                raise ValueError("bc_type=%r not understood" % (side,))
            out.append((BC_KINDS[side], None))
        else:
            order, val = side
            if order not in (1, 2):
                raise ValueError("The specified derivative order must be 1 or 2.")
            if isinstance(val, torch_mod().Tensor):   # boundary values already on the device: [B, dof]
                out.append((int(order), as_device(val.reshape(B, dof).contiguous(), device)))
                continue
            val = np.asarray(val, dtype=np.float64)
            val = np.broadcast_to(val, (B, dof)) if val.ndim <= 1 else val.reshape(B, dof)
            out.append((int(order), as_device(np.ascontiguousarray(val), device)))
    return tuple(out)


def spline_fit(ss, wp, bc=((0, None), (0, None))):
    """ss: [n] or [B, n]; wp: [B, n, dof] (CUDA fp64) -> ppoly [B, 4, n-1, dof]."""
    torch = torch_mod()
    lib = _lib.load()
    B, n, dof = wp.shape
    ppoly = torch.empty((B, 4, n - 1, dof), dtype=torch.float64, device=wp.device)
    (k0, v0), (k1, v1) = bc
    nws = lib.tb_spline_fit_workspace_doubles(B, n, dof)
    if nws < 0:
        raise ValueError("spline_fit: batch too large for one call (B=%d, n=%d, dof=%d)" % (B, n, dof))
    ws = torch.empty((nws,), dtype=torch.float64, device=wp.device) if nws > 0 else None
    with torch.cuda.device(wp.device):
        rc = lib.tb_spline_fit(_lib.ptr(ss), 1 if ss.dim() == 1 else 0, _lib.ptr(wp), B, n, dof, k0, _lib.ptr(v0), k1,
                               _lib.ptr(v1), _lib.ptr(ppoly), _lib.ptr(ws), _lib.stream_ptr())
    _lib.check(rc, "tb_spline_fit")
    return ppoly


def is_cubic(ppoly):
    """Paths with 4 coefficients per piece take libtoppra_b200's kernels; 1..8 otherwise take libtoppra_b200_poly's
    (the order-k path: evaluate, build records from the samples, record scan)."""
    return ppoly.shape[1] == 4


def require_cubic(ppoly, what):
    if not is_cubic(ppoly):
        raise NotImplementedError("%s needs piecewise-cubic paths; this path has order %d (%d coefficients per piece)"
                                  % (what, ppoly.shape[1], ppoly.shape[1]))


def ppoly_eval(ppoly, breaks, s, order):
    """ppoly [B,k,nseg,dof], breaks [nseg+1] or [B,nseg+1], s [G] or [B,G] -> [B,G,dof]."""
    torch = torch_mod()
    B, kc, nseg, dof = ppoly.shape
    G = s.shape[-1]
    out = torch.empty((B, G, dof), dtype=torch.float64, device=ppoly.device)
    if not is_cubic(ppoly):
        with torch.cuda.device(ppoly.device):
            rc = _lib_poly.load().tbp_ppoly_eval(_lib.ptr(ppoly), _lib.ptr(breaks), 1 if breaks.dim() == 1 else 0, B, kc,
                                                 nseg, dof, _lib.ptr(s), 1 if s.dim() == 1 else 0, G, int(order),
                                                 _lib.ptr(out), _lib.stream_ptr())
        _lib.check(rc, "tbp_ppoly_eval")
        return out
    lib = _lib.load()
    with torch.cuda.device(ppoly.device):
        rc = lib.tb_ppoly_eval(_lib.ptr(ppoly), _lib.ptr(breaks), 1 if breaks.dim() == 1 else 0, B, nseg, dof,
                               _lib.ptr(s), 1 if s.dim() == 1 else 0, G, int(order), _lib.ptr(out), _lib.stream_ptr())
    _lib.check(rc, "tb_ppoly_eval")
    return out


def record_doubles(R):
    return int(_lib.load().tb_record_doubles(int(R)))


def alloc_records(B, G, R, device, ubound=False):
    """Stage records [B, G, W]: a[R] | b[R] | c[R] | xlo | xhi (W = 3R+2 rounded to even); with ubound=True the record
    also carries ulo | uhi (W = 3R+4 rounded to even; the scans are told by TB_SCAN_UBOUND, inferred from W)."""
    torch = torch_mod()
    W = record_doubles(R)
    if ubound:
        W = (3 * R + 4 + 1) & ~1
    return torch.empty((B, G, W), dtype=torch.float64, device=device), W


def has_ubound(records, R):
    return records.shape[-1] >= 3 * int(R) + 4


def init_bounds(records, R):
    torch = torch_mod()
    B, G, W = records.shape
    with torch.cuda.device(records.device):
        rc = _lib.load().tb_init_bounds(_lib.ptr(records), B, G, W, R, _lib.stream_ptr())
    _lib.check(rc, "tb_init_bounds")


def check_grid_shapes(B, breaks, nbreaks, grid, G):
    """Per-path arrays must have the batch's leading dimension (the kernels index them with the path number)."""
    if breaks.dim() not in (1, 2) or breaks.shape[-1] != nbreaks or (breaks.dim() == 2 and breaks.shape[0] != B):
        raise ValueError("breakpoints must have shape (%d,) or (%d, %d); got %s" % (nbreaks, B, nbreaks, tuple(breaks.shape)))
    if grid.dim() not in (1, 2) or grid.shape[-1] != G or (grid.dim() == 2 and grid.shape[0] != B):
        raise ValueError("gridpoints must have shape (G,) or (%d, G); got %s" % (B, tuple(grid.shape)))


def check_grid(grid, B, G):
    """gridpoints: (G,) shared by the batch or (B, G)."""
    if grid.dim() not in (1, 2) or grid.shape[-1] != G or (grid.dim() == 2 and grid.shape[0] != B):
        raise ValueError("gridpoints must have shape (%d,) or (%d, %d); got %s" % (G, B, G, tuple(grid.shape)))


def check_shape(t, shape, what):
    if t is not None and tuple(t.shape) != tuple(shape):
        raise ValueError("%s must have shape %s; got %s" % (what, tuple(shape), tuple(t.shape)))


def check_path_vector(t, B, what):
    if t is not None and tuple(t.shape) != (B,):
        raise ValueError("%s must have shape (%d,); got %s" % (what, B, tuple(t.shape)))


def velacc_limits(vlim, alim, B, dof):
    """(vlim, alim, shared) for the records of coeff_velacc / rows_velacc_sampled: each limit array (dof, 2) or
    (B, dof, 2), either may be None.  When one is per path, the other is expanded to (B, dof, 2) and shared is False."""
    lims = [t for t in (vlim, alim) if t is not None]
    for t in lims:  # raw pointers go to the kernels: a short limit array would be read out of bounds on the device
        if t.dim() not in (2, 3) or tuple(t.shape[-2:]) != (dof, 2) or (t.dim() == 3 and t.shape[0] != B):
            raise ValueError("limits must have shape (dof, 2) or (B, dof, 2) with B = %d, dof = %d; got %s"
                             % (B, dof, tuple(t.shape)))
    shared = all(t.dim() == 2 for t in lims)
    if not shared:
        vlim = None if vlim is None else (vlim if vlim.dim() == 3 else vlim.expand(B, dof, 2).contiguous())
        alim = None if alim is None else (alim if alim.dim() == 3 else alim.expand(B, dof, 2).contiguous())
    return vlim, alim, shared


def check_vlim_grid(vlim_grid, B, G, dof):
    """Per-gridpoint velocity limits: (G, dof, 2) shared by the batch or (B, G, dof, 2)."""
    if tuple(vlim_grid.shape[-3:]) != (G, dof, 2) or vlim_grid.dim() not in (3, 4) or (vlim_grid.dim() == 4 and vlim_grid.shape[0] != B):
        raise ValueError("varying velocity limits must have shape (G, dof, 2) or (B, G, dof, 2); got %s" % (tuple(vlim_grid.shape),))


def coeff_velacc(ppoly, breaks, grid, vlim, alim, interp, records, R_total, row0=0, write_xbound=1):
    """K1.  vlim/alim: [dof,2] or [B,dof,2] device tensors (either may be None, not both).  Order-k paths: q' and q''
    at the gridpoints (tbp_ppoly_eval), then the records from those samples (rows_velacc_sampled)."""
    torch = torch_mod()
    B, _, nseg, dof = ppoly.shape
    G = grid.shape[-1]
    W = records.shape[-1]
    vlim, alim, shared = velacc_limits(vlim, alim, B, dof)
    check_grid_shapes(B, breaks, nseg + 1, grid, G)
    if not is_cubic(ppoly):
        qd, qdd = ppoly_eval(ppoly, breaks, grid, 1), ppoly_eval(ppoly, breaks, grid, 2)
        rows_velacc_sampled(qd, qdd, grid, vlim, alim, interp, records, R_total, row0, write_xbound)
        return
    with torch.cuda.device(records.device):
        rc = _lib.load().tb_coeff_velacc(_lib.ptr(ppoly), _lib.ptr(breaks), 1 if breaks.dim() == 1 else 0, B, nseg, dof,
                                         _lib.ptr(grid), 1 if grid.dim() == 1 else 0, G, _lib.ptr(vlim),
                                         _lib.ptr(alim), 1 if shared else 0, 1 if interp else 0, _lib.ptr(records), W,
                                         int(R_total), int(row0), int(write_xbound), _lib.stream_ptr())
    _lib.check(rc, "tb_coeff_velacc")


def rows_velacc_sampled(qd, qdd, grid, vlim, alim, interp, records, R_total, row0=0, write_xbound=1):
    """K1's records from sampled path derivatives qd = q'(grid), qdd = q''(grid), both [B, G, dof]
    (tbp_rows_velacc_sampled).  Every other argument as coeff_velacc."""
    torch = torch_mod()
    B, G, dof = qd.shape
    W = records.shape[-1]
    check_shape(qdd, (B, G, dof), "qdd")
    check_grid(grid, B, G)
    if tuple(records.shape[:2]) != (B, G):
        raise ValueError("records must have shape (%d, %d, W); got %s" % (B, G, tuple(records.shape)))
    vlim, alim, shared = velacc_limits(vlim, alim, B, dof)
    with torch.cuda.device(records.device):
        rc = _lib_poly.load().tbp_rows_velacc_sampled(_lib.ptr(qd), _lib.ptr(qdd), B, dof, _lib.ptr(grid),
                                                      1 if grid.dim() == 1 else 0, G, _lib.ptr(vlim), _lib.ptr(alim),
                                                      1 if shared else 0, 1 if interp else 0, _lib.ptr(records), W,
                                                      int(R_total), int(row0), int(write_xbound), _lib.stream_ptr())
    _lib.check(rc, "tbp_rows_velacc_sampled")


DEVICE_MODELS = {"coupled_cosine": 0, "pendulums": 1}  # TB_INVDYN_* of include/toppra_b200.h


def coeff_second_order(model, params, ppoly, breaks, grid, taulim, friction, interp, records, R_total, row0):
    """Joint-torque rows of a SecondOrderConstraint whose inverse dynamics is a DEVICE MODEL (tb_coeff_second_order):
    evaluated on the GPU from the spline, written straight into `records`.  taulim [dof,2] or [B,dof,2] (device),
    friction [dof] device tensor or None.  Returns the number of rows written."""
    torch = torch_mod()
    require_cubic(ppoly, "SecondOrderConstraint with a device model (tb_coeff_second_order)")
    B, _, nseg, dof = ppoly.shape
    G = grid.shape[-1]
    W = records.shape[-1]
    check_grid_shapes(B, breaks, nseg + 1, grid, G)
    if taulim.dim() not in (2, 3) or tuple(taulim.shape[-2:]) != (dof, 2) or (taulim.dim() == 3 and taulim.shape[0] != B):
        raise ValueError("torque limits must have shape (dof, 2) or (B, dof, 2); got %s" % (tuple(taulim.shape),))
    if friction is not None and tuple(friction.shape) != (dof,):
        raise ValueError("joint friction must have shape (dof,)")
    prm = as_device(np.asarray(params, dtype=np.float64).reshape(-1), records.device)
    with torch.cuda.device(records.device):
        rc = _lib.load().tb_coeff_second_order(int(DEVICE_MODELS[model]), _lib.ptr(prm), int(prm.numel()), _lib.ptr(ppoly),
                                               _lib.ptr(breaks), 1 if breaks.dim() == 1 else 0, B, nseg, dof,
                                               _lib.ptr(grid), 1 if grid.dim() == 1 else 0, G, _lib.ptr(taulim),
                                               1 if taulim.dim() == 2 else 0, _lib.ptr(friction), 1 if interp else 0,
                                               _lib.ptr(records), W, int(R_total), int(row0), _lib.stream_ptr())
    _lib.check(rc, "tb_coeff_second_order")
    return (4 if interp else 2) * dof


def rows_canlinear(a, b, c, F, g, F_mode, grid, interp, records, R_total, row0):
    """Generic CanonicalLinear rows.  a,b,c: [B,G,m]; F/g per F_mode (see include/toppra_b200.h)."""
    torch = torch_mod()
    B, G, m = a.shape
    W = records.shape[-1]
    if F_mode == 0:
        k = F.shape[0]
    elif F_mode == 1:
        k = F.shape[2]
    else:
        k = 2 * m
    # shapes per include/toppra_b200.h: raw pointers go to the kernel, a short array would be read out of bounds
    check_shape(b, (B, G, m), "b")
    check_shape(c, (B, G, m), "c")
    check_grid(grid, B, G)
    if F_mode not in (0, 1, 2, 3):
        raise ValueError("F_mode must be 0..3; got %r" % (F_mode,))
    check_shape(F, {0: (k, m), 1: (B, G, k, m)}.get(F_mode, None if F is None else tuple(F.shape)), "F")
    check_shape(g, {0: (k,), 1: (B, G, k), 2: (k,), 3: (B, k)}[F_mode], "g")
    if tuple(records.shape[:2]) != (B, G):
        raise ValueError("records must have shape (%d, %d, W); got %s" % (B, G, tuple(records.shape)))
    with torch.cuda.device(records.device):
        rc = _lib.load().tb_rows_canlinear(_lib.ptr(a), _lib.ptr(b), _lib.ptr(c), _lib.ptr(F), _lib.ptr(g), int(F_mode),
                                           B, G, m, k, _lib.ptr(grid), 1 if grid.dim() == 1 else 0, 1 if interp else 0,
                                           _lib.ptr(records), W, int(R_total), int(row0), _lib.stream_ptr())
    _lib.check(rc, "tb_rows_canlinear")
    return 2 * k if interp else k


def scan(records, R, grid, sd_start=None, sd_end=None, sd_end_hi=None, backward_only=False, counters=False,
         sd_forward=None, forward_from=None, fast_lower=False, glen=None):
    """K2.  Returns dict(K [B,G,2], sd [B,G], u [B,G-1], status [B] int32, fail_stage [B] int32[, counters [B,4]]).
    glen: optional int32 [B] gridpoints per path (ragged batch, grid [B, G] padded)."""
    torch = torch_mod()
    B, G, W = records.shape
    dev = records.device
    check_grid(grid, B, G)
    for t, what in ((sd_start, "sd_start"), (sd_end, "sd_end"), (sd_end_hi, "sd_end_hi")):
        check_path_vector(t, B, what)
    out, u_arg = _scan_outputs(B, G, dev, backward_only, counters, forward_from)
    check_glen(glen, B, grid)
    ub = has_ubound(records, R)
    flags = _scan_flags(backward_only, sd_forward, forward_from, fast_lower and not ub, ub)
    with torch.cuda.device(dev):
        rc = _lib.load().tb_scan_ragged(_lib.ptr(records), W, int(R), _lib.ptr(grid), 1 if grid.dim() == 1 else 0, B, G,
                                        _lib.ptr(glen), _lib.ptr(sd_start), _lib.ptr(sd_end), _lib.ptr(sd_end_hi), flags,
                                        _lib.ptr(out["K"]), _lib.ptr(out["sd"]), _lib.ptr(u_arg), _lib.ptr(out["status"]),
                                        _lib.ptr(out["fail_stage"]), _lib.ptr(out.get("counters")), _lib.stream_ptr())
    _lib.check(rc, "tb_scan")
    return out


SCAN_FLAGS = dict(backward_only=1, sd_fast=4, sd_slow=12, forward_only=16, fast_lower=32, ubound=64)


def _scan_flags(backward_only, sd_forward, forward_from, fast_lower, ubound=False):
    """TB_SCAN_* flags word of a scan launch; forward_from (an earlier backward-only result) means forward only."""
    return ((SCAN_FLAGS["backward_only"] if backward_only else 0)
            | {None: 0, "fast": SCAN_FLAGS["sd_fast"], "slow": SCAN_FLAGS["sd_slow"]}[sd_forward]
            | (SCAN_FLAGS["forward_only"] if forward_from is not None else 0)
            | (SCAN_FLAGS["fast_lower"] if fast_lower else 0)
            | (SCAN_FLAGS["ubound"] if ubound else 0))


def _scan_outputs(B, G, dev, backward_only, counters, forward_from=None):
    """Output dict of a scan: K [B,G,2], sd [B,G], u [B,G-1], status / fail_stage [B] int32[, counters [B,4] zeroed].
    forward_from: reuse K / status / fail_stage of an earlier backward-only launch.  sd and u are None when
    backward_only.  Also returns the tensor to pass as u: a one-element stand-in when G = 1 leaves u empty."""
    torch = torch_mod()
    if forward_from is not None:
        K, status, fail_stage = forward_from["K"], forward_from["status"], forward_from["fail_stage"]
    else:
        K = torch.empty((B, G, 2), dtype=torch.float64, device=dev)
        status = torch.empty((B,), dtype=torch.int32, device=dev)
        fail_stage = torch.empty((B,), dtype=torch.int32, device=dev)
    sd = None if backward_only else torch.empty((B, G), dtype=torch.float64, device=dev)
    u = None if backward_only else torch.empty((B, max(G - 1, 0)), dtype=torch.float64, device=dev)
    u_arg = u if (u is None or u.numel() > 0) else torch.empty((1,), dtype=torch.float64, device=dev)
    out = dict(K=K, sd=sd, u=u, status=status, fail_stage=fail_stage)
    if counters:
        out["counters"] = torch.zeros((B, 4), dtype=torch.int32, device=dev)
    return out, u_arg


def check_glen(glen, B, grid):
    if glen is None:
        return
    torch = torch_mod()
    if glen.dtype != torch.int32 or tuple(glen.shape) != (B,):
        raise ValueError("glen must be an int32 tensor of shape (%d,)" % B)
    if grid.dim() != 2:
        raise ValueError("ragged batches (glen) need per-path gridpoints of shape (B, G)")


def velacc_fused_supported(nseg, dof, interp):
    """tb_scan_velacc holds one LP row per lane and the spline's derivative coefficients in 16 KB of shared memory."""
    return (4 if interp else 2) * dof + 2 <= 32 and 8 * ((nseg * dof * 6 + nseg + 2) & ~1) <= 16 * 1024


def xbound_velocity(ppoly, breaks, grid, vlim, out=None):
    """Velocity bound alone: xbound [B, G, 2] clipped to the solver box (+-1e8 when vlim is None) = K1 with no rows."""
    torch = torch_mod()
    require_cubic(ppoly, "xbound_velocity (the fused scan's velocity bound)")
    B = ppoly.shape[0]
    xb = torch.empty((B, grid.shape[-1], 2), dtype=torch.float64, device=ppoly.device) if out is None else out
    if vlim is None:
        init_bounds(xb, 0)
    else:
        xbound_constant(ppoly, breaks, grid, vlim, xb, 0, 1)
    return xb


def xbound_constant(ppoly, breaks, grid, vlim, records, R_total, write_xbound):
    """JointVelocityConstraint alone into the xbound slots of `records` (tb_xbound_velocity, thread per gridpoint)."""
    torch = torch_mod()
    require_cubic(ppoly, "xbound_constant")
    B, _, nseg, dof = ppoly.shape
    G = grid.shape[-1]
    W = records.shape[-1]
    check_grid_shapes(B, breaks, nseg + 1, grid, G)
    if vlim.dim() not in (2, 3) or tuple(vlim.shape[-2:]) != (dof, 2) or (vlim.dim() == 3 and vlim.shape[0] != B):
        raise ValueError("velocity limits must have shape (dof, 2) or (B, dof, 2); got %s" % (tuple(vlim.shape),))
    with torch.cuda.device(records.device):
        rc = _lib.load().tb_xbound_velocity(_lib.ptr(ppoly), _lib.ptr(breaks), 1 if breaks.dim() == 1 else 0, B, nseg, dof,
                                            _lib.ptr(grid), 1 if grid.dim() == 1 else 0, G, _lib.ptr(vlim),
                                            1 if vlim.dim() == 2 else 0, _lib.ptr(records), W, int(R_total),
                                            int(write_xbound), _lib.stream_ptr())
    _lib.check(rc, "tb_xbound_velocity")


def scan_velacc(ppoly, breaks, grid, alim, interp, xbound, sd_start=None, sd_end=None, sd_end_hi=None,
                backward_only=False, counters=False, sd_forward=None, forward_from=None, fast_lower=False, glen=None):
    """K2 fused with K1 for JointVelocity + JointAcceleration (tb_scan_velacc): rows are built inside the scan from
    the spline; `xbound` [B, G, 2] from xbound_velocity().  Same outputs as scan()."""
    torch = torch_mod()
    require_cubic(ppoly, "scan_velacc (the fused vel+acc scan)")
    B, _, nseg, dof = ppoly.shape
    G = grid.shape[-1]
    dev = ppoly.device
    check_grid_shapes(B, breaks, nseg + 1, grid, G)
    if alim.dim() not in (2, 3) or tuple(alim.shape[-2:]) != (dof, 2) or (alim.dim() == 3 and alim.shape[0] != B):
        raise ValueError("acceleration limits must have shape (dof, 2) or (B, dof, 2); got %s" % (tuple(alim.shape),))
    if tuple(xbound.shape) != (B, G, 2):
        raise ValueError("xbound must have shape (B, G, 2)")
    for t, what in ((sd_start, "sd_start"), (sd_end, "sd_end"), (sd_end_hi, "sd_end_hi")):
        check_path_vector(t, B, what)
    out, u_arg = _scan_outputs(B, G, dev, backward_only, counters, forward_from)
    flags = _scan_flags(backward_only, sd_forward, forward_from, fast_lower)
    check_glen(glen, B, grid)
    with torch.cuda.device(dev):
        rc = _lib.load().tb_scan_velacc_ragged(_lib.ptr(ppoly), _lib.ptr(breaks), 1 if breaks.dim() == 1 else 0, nseg, dof,
                                        _lib.ptr(grid), 1 if grid.dim() == 1 else 0, B, G, _lib.ptr(glen), _lib.ptr(alim),
                                        1 if alim.dim() == 2 else 0, 1 if interp else 0, _lib.ptr(xbound),
                                        _lib.ptr(sd_start), _lib.ptr(sd_end), _lib.ptr(sd_end_hi), flags,
                                        _lib.ptr(out["K"]), _lib.ptr(out["sd"]), _lib.ptr(u_arg), _lib.ptr(out["status"]),
                                        _lib.ptr(out["fail_stage"]), _lib.ptr(out.get("counters")), _lib.stream_ptr())
    _lib.check(rc, "tb_scan_velacc")
    return out


def scan_robust(records, R, conic_row0, conic_rows, ellipsoid, grid, sd_start=None, sd_end=None, backward_only=False,
                counters=False, feasible_sets=False, glen=None, sd_end_hi=None):
    """K2r: like scan() with rows [conic_row0, conic_row0+conic_rows) robustified by the ellipsoid (ru, rx, rc).
    glen: optional int32 [B] gridpoints per path (ragged batch, tb_scan_robust_ragged).  sd_end_hi: optional [B] upper
    terminal velocity, K[N] = [sd_end^2, sd_end_hi^2] (compute_controllable_sets(sdmin, sdmax), tb_scan_robust_ex)."""
    torch = torch_mod()
    B, G, W = records.shape
    dev = records.device
    backward_only = backward_only or feasible_sets
    out, u_arg = _scan_outputs(B, G, dev, backward_only, counters)
    ell = np.ascontiguousarray(ellipsoid, dtype=np.float64)
    assert ell.shape == (3,)
    lib = _lib.load()
    args = (_lib.ptr(records), W, int(R), int(conic_row0), int(conic_rows), ctypes.c_void_p(ell.ctypes.data),
            _lib.ptr(grid), 1 if grid.dim() == 1 else 0, B, G)
    rest = (2 if feasible_sets else (1 if backward_only else 0),
            _lib.ptr(out["K"]), _lib.ptr(out["sd"]), _lib.ptr(u_arg), _lib.ptr(out["status"]),
            _lib.ptr(out["fail_stage"]), _lib.ptr(out.get("counters")), _lib.stream_ptr())
    ends = (_lib.ptr(sd_start), _lib.ptr(sd_end))
    if glen is not None:
        check_grid(grid, B, G)
        check_glen(glen, B, grid)
    check_path_vector(sd_end_hi, B, "sd_end_hi")
    with torch.cuda.device(dev):
        if sd_end_hi is not None:
            name = "tb_scan_robust_ex"
            rc = lib.tb_scan_robust_ex(*args, _lib.ptr(glen), *ends, _lib.ptr(sd_end_hi), *rest)
        elif glen is not None:
            name = "tb_scan_robust_ragged"
            rc = lib.tb_scan_robust_ragged(*args, _lib.ptr(glen), *ends, *rest)
        else:
            name = "tb_scan_robust"
            rc = lib.tb_scan_robust(*args, *ends, *rest)
    _lib.check(rc, name)
    return out


def sd_forward_robust(records, R, conic_row0, conic_rows, ellipsoid, grid, K, status_in, sd_start=None, glen=None):
    """The fastest and the slowest TOPPRAsd forward pass of robust problems in one launch (tbr_sd_forward_robust), on K
    and status of a backward-only scan_robust over the same records.  Returns dict(x_fast, x_slow [B,G] = sd^2,
    u_fast, u_slow [B,G-1], status [B], fail_stage [B] int32 of the fastest pass).  glen: optional int32 [B] gridpoints
    per path (ragged batch)."""
    torch = torch_mod()
    B, G, W = records.shape
    dev = records.device
    check_grid(grid, B, G)
    check_glen(glen, B, grid)
    check_path_vector(sd_start, B, "sd_start")
    check_shape(K, (B, G, 2), "K")
    if status_in.dtype != torch.int32 or tuple(status_in.shape) != (B,):
        raise ValueError("status_in must be an int32 tensor of shape (%d,)" % B)
    ell = np.ascontiguousarray(ellipsoid, dtype=np.float64)
    assert ell.shape == (3,)
    out = {key: torch.empty((B, G), dtype=torch.float64, device=dev) for key in ("x_fast", "x_slow")}
    out.update({key: torch.empty((B, max(G - 1, 0)), dtype=torch.float64, device=dev) for key in ("u_fast", "u_slow")})
    out["status"] = torch.empty((B,), dtype=torch.int32, device=dev)
    out["fail_stage"] = torch.empty((B,), dtype=torch.int32, device=dev)
    u_fast, u_slow = (out[k] if G > 1 else None for k in ("u_fast", "u_slow"))
    with torch.cuda.device(dev):
        rc = _lib_robust.load().tbr_sd_forward_robust(
            _lib.ptr(records), W, int(R), int(conic_row0), int(conic_rows), ctypes.c_void_p(ell.ctypes.data),
            _lib.ptr(grid), 1 if grid.dim() == 1 else 0, B, G, _lib.ptr(glen), _lib.ptr(K), _lib.ptr(status_in),
            _lib.ptr(sd_start), _lib.ptr(out["x_fast"]), _lib.ptr(u_fast), _lib.ptr(out["x_slow"]), _lib.ptr(u_slow),
            _lib.ptr(out["status"]), _lib.ptr(out["fail_stage"]), _lib.stream_ptr())
    _lib.check(rc, "tbr_sd_forward_robust")
    return out


def socp_stage_batch(g, a, b, c, conic_row0, conic_rows, ellipsoid, xbox, xnext=None):
    """Batched robust stage problems on device (tbr_socp_stage_batch): min g0 u + g1 x over the rows a, b, c [B, n]
    (robust on [conic_row0, conic_row0 + conic_rows)), xbox [B, 2] and the optional x_next rows xnext [B, 3] =
    (delta, lo, hi) (NaN delta = none).  Inputs numpy or tensors.  Returns numpy optvar [B, 2] = (u, x), NaN if
    infeasible."""
    torch = torch_mod()
    dev = default_device()
    g = as_device(g, dev).reshape(-1, 2)
    B = g.shape[0]
    a, b, c = (as_device(t, dev).reshape(B, -1) for t in (a, b, c))
    n = a.shape[1]
    xbox = as_device(xbox, dev).reshape(B, 2)
    xnext = None if xnext is None else as_device(xnext, dev).reshape(B, 3)
    ell = np.ascontiguousarray(ellipsoid, dtype=np.float64)
    assert ell.shape == (3,)
    optvar = torch.empty((B, 2), dtype=torch.float64, device=dev)
    with torch.cuda.device(dev):
        rc = _lib_robust.load().tbr_socp_stage_batch(
            _lib.ptr(g), _lib.ptr(a) if n else None, _lib.ptr(b) if n else None, _lib.ptr(c) if n else None, n,
            int(conic_row0), int(conic_rows), ctypes.c_void_p(ell.ctypes.data), _lib.ptr(xbox), _lib.ptr(xnext), B,
            _lib.ptr(optvar), _lib.stream_ptr())
    _lib.check(rc, "tbr_socp_stage_batch")
    return optvar.cpu().numpy()


def feasible_sets(records, R, grid, glen=None):
    """compute_feasible_sets for B paths: X [B,G,2].  glen: optional int32 [B] gridpoints per path (ragged batch,
    tb_feasible_sets_ragged; X past a path's own gridpoints is NaN)."""
    torch = torch_mod()
    B, G, W = records.shape
    check_grid(grid, B, G)
    check_glen(glen, B, grid)
    X = torch.empty((B, G, 2), dtype=torch.float64, device=records.device)
    lib = _lib.load()
    args = (_lib.ptr(records), W, int(R), _lib.ptr(grid), 1 if grid.dim() == 1 else 0, B, G)
    flags = SCAN_FLAGS["ubound"] if has_ubound(records, R) else 0
    with torch.cuda.device(records.device):
        if glen is None:
            rc = lib.tb_feasible_sets_ex(*args, flags, _lib.ptr(X), _lib.stream_ptr())
        else:
            rc = lib.tb_feasible_sets_ragged(*args, _lib.ptr(glen), flags, _lib.ptr(X), _lib.stream_ptr())
    _lib.check(rc, "tb_feasible_sets")
    return X


def reachable_sets(records, R, grid, sdmin=None, sdmax=None, glen=None):
    """compute_reachable_sets for B paths in one launch (tb_reachable_sets).  sdmin / sdmax: [B] tensors or None.
    Returns dict(X [B,G,2] feasible sets, L [B,G,2] reachable sets, fail_stage [B] int32).  glen: optional int32 [B]
    gridpoints per path (ragged batch, tb_reachable_sets_ragged; X and L past a path's own gridpoints are NaN)."""
    torch = torch_mod()
    B, G, W = records.shape
    dev = records.device
    check_grid(grid, B, G)
    check_glen(glen, B, grid)
    for t, what in ((sdmin, "sdmin"), (sdmax, "sdmax")):
        check_path_vector(t, B, what)
    X = torch.empty((B, G, 2), dtype=torch.float64, device=dev)
    L = torch.empty((B, G, 2), dtype=torch.float64, device=dev)
    fs = torch.empty((B,), dtype=torch.int32, device=dev)
    lib = _lib.load()
    args = (_lib.ptr(records), W, int(R), _lib.ptr(grid), 1 if grid.dim() == 1 else 0, B, G)
    rest = (_lib.ptr(sdmin), _lib.ptr(sdmax), SCAN_FLAGS["ubound"] if has_ubound(records, R) else 0, _lib.ptr(X),
            _lib.ptr(L), _lib.ptr(fs), _lib.stream_ptr())
    with torch.cuda.device(dev):
        if glen is None:
            rc = lib.tb_reachable_sets(*args, *rest)
        else:
            rc = lib.tb_reachable_sets_ragged(*args, _lib.ptr(glen), *rest)
    _lib.check(rc, "tb_reachable_sets")
    return dict(X=X, L=L, fail_stage=fs)


def reachable_sets_robust(records, R, conic_row0, conic_rows, ellipsoid, grid, sdmin=None, sdmax=None, glen=None):
    """compute_reachable_sets of robust problems: the feasible sets X of one tb_scan_robust[_ragged]
    (TB_SCAN_FEASIBLE_SETS) launch, then the forward recursion in one tbr_reachable_sets_robust launch.  Same arguments
    and result as reachable_sets(): dict(X [B,G,2], L [B,G,2], fail_stage [B] int32)."""
    torch = torch_mod()
    B, G, W = records.shape
    dev = records.device
    check_grid(grid, B, G)
    check_glen(glen, B, grid)
    for t, what in ((sdmin, "sdmin"), (sdmax, "sdmax")):
        check_path_vector(t, B, what)
    X = scan_robust(records, R, conic_row0, conic_rows, ellipsoid, grid, feasible_sets=True, glen=glen)["K"]
    ell = np.ascontiguousarray(ellipsoid, dtype=np.float64)
    L = torch.empty((B, G, 2), dtype=torch.float64, device=dev)
    fs = torch.empty((B,), dtype=torch.int32, device=dev)
    with torch.cuda.device(dev):
        rc = _lib_reach.load().tbr_reachable_sets_robust(
            _lib.ptr(records), W, int(R), int(conic_row0), int(conic_rows), ctypes.c_void_p(ell.ctypes.data),
            _lib.ptr(grid), 1 if grid.dim() == 1 else 0, B, G, _lib.ptr(glen), _lib.ptr(X), _lib.ptr(sdmin),
            _lib.ptr(sdmax), _lib.ptr(L), _lib.ptr(fs), _lib.stream_ptr())
    _lib.check(rc, "tbr_reachable_sets_robust")
    return dict(X=X, L=L, fail_stage=fs)


def _cone_table(cones, R):
    """The host cone table [R][4] = (robust flag 0/1, ru, rx, rc) per row, C-contiguous float64."""
    t = np.ascontiguousarray(cones, dtype=np.float64)
    if t.shape != (int(R), 4):
        raise ValueError("cone table must have shape (%d, 4); got %s" % (int(R), t.shape))
    return t


def scan_cones(records, R, cones, grid, sd_start=None, sd_end=None, backward_only=False, counters=False,
               feasible_sets=False, glen=None, sd_end_hi=None):
    """scan_robust() on the cone table cones [R, 4] (tbc_scan): every row its own robust flag and axes; records with a
    u-bound pair (W >= 3R+4) add the u box (TB_SCAN_UBOUND).  Same arguments otherwise, same result."""
    torch = torch_mod()
    B, G, W = records.shape
    dev = records.device
    backward_only = backward_only or feasible_sets
    out, u_arg = _scan_outputs(B, G, dev, backward_only, counters)
    table = _cone_table(cones, R)
    if glen is not None:
        check_grid(grid, B, G)
        check_glen(glen, B, grid)
    check_path_vector(sd_end_hi, B, "sd_end_hi")
    flags = ((2 if feasible_sets else (1 if backward_only else 0))
             | (SCAN_FLAGS["ubound"] if has_ubound(records, R) else 0))
    with torch.cuda.device(dev):
        rc = _lib_cones.load().tbc_scan(
            _lib.ptr(records), W, int(R), ctypes.c_void_p(table.ctypes.data), _lib.ptr(grid), 1 if grid.dim() == 1 else 0,
            B, G, _lib.ptr(glen), _lib.ptr(sd_start), _lib.ptr(sd_end), _lib.ptr(sd_end_hi), flags, _lib.ptr(out["K"]),
            _lib.ptr(out["sd"]), _lib.ptr(u_arg), _lib.ptr(out["status"]), _lib.ptr(out["fail_stage"]),
            _lib.ptr(out.get("counters")), _lib.stream_ptr())
    _lib.check(rc, "tbc_scan")
    return out


def sd_forward_cones(records, R, cones, grid, K, status_in, sd_start=None, glen=None):
    """sd_forward_robust() on the cone table cones [R, 4] (tbc_sd_forward), with the u box of records that carry one."""
    torch = torch_mod()
    B, G, W = records.shape
    dev = records.device
    check_grid(grid, B, G)
    check_glen(glen, B, grid)
    check_path_vector(sd_start, B, "sd_start")
    check_shape(K, (B, G, 2), "K")
    if status_in.dtype != torch.int32 or tuple(status_in.shape) != (B,):
        raise ValueError("status_in must be an int32 tensor of shape (%d,)" % B)
    table = _cone_table(cones, R)
    out = {key: torch.empty((B, G), dtype=torch.float64, device=dev) for key in ("x_fast", "x_slow")}
    out.update({key: torch.empty((B, max(G - 1, 0)), dtype=torch.float64, device=dev) for key in ("u_fast", "u_slow")})
    out["status"] = torch.empty((B,), dtype=torch.int32, device=dev)
    out["fail_stage"] = torch.empty((B,), dtype=torch.int32, device=dev)
    u_fast, u_slow = (out[k] if G > 1 else None for k in ("u_fast", "u_slow"))
    with torch.cuda.device(dev):
        rc = _lib_cones.load().tbc_sd_forward(
            _lib.ptr(records), W, int(R), ctypes.c_void_p(table.ctypes.data),
            SCAN_FLAGS["ubound"] if has_ubound(records, R) else 0, _lib.ptr(grid), 1 if grid.dim() == 1 else 0, B, G,
            _lib.ptr(glen), _lib.ptr(K), _lib.ptr(status_in), _lib.ptr(sd_start), _lib.ptr(out["x_fast"]),
            _lib.ptr(u_fast), _lib.ptr(out["x_slow"]), _lib.ptr(u_slow), _lib.ptr(out["status"]),
            _lib.ptr(out["fail_stage"]), _lib.stream_ptr())
    _lib.check(rc, "tbc_sd_forward")
    return out


def socp_stage_batch_cones(g, a, b, c, cones, xbox, xnext=None, ubox=None):
    """socp_stage_batch() on the cone table cones [n, 4] (tbc_socp_stage_batch), with the optional u box ubox [B, 2].
    Returns numpy optvar [B, 2] = (u, x), NaN if infeasible."""
    torch = torch_mod()
    dev = default_device()
    g = as_device(g, dev).reshape(-1, 2)
    B = g.shape[0]
    a, b, c = (as_device(t, dev).reshape(B, -1) for t in (a, b, c))
    n = a.shape[1]
    xbox = as_device(xbox, dev).reshape(B, 2)
    xnext = None if xnext is None else as_device(xnext, dev).reshape(B, 3)
    ubox = None if ubox is None else as_device(ubox, dev).reshape(B, 2)
    table = _cone_table(cones, n)
    optvar = torch.empty((B, 2), dtype=torch.float64, device=dev)
    with torch.cuda.device(dev):
        rc = _lib_cones.load().tbc_socp_stage_batch(
            _lib.ptr(g), _lib.ptr(a) if n else None, _lib.ptr(b) if n else None, _lib.ptr(c) if n else None, n,
            ctypes.c_void_p(table.ctypes.data), _lib.ptr(xbox), _lib.ptr(xnext), _lib.ptr(ubox), B, _lib.ptr(optvar),
            _lib.stream_ptr())
    _lib.check(rc, "tbc_socp_stage_batch")
    return optvar.cpu().numpy()


def reachable_sets_cones(records, R, cones, grid, sdmin=None, sdmax=None, glen=None):
    """reachable_sets_robust() on the cone table cones [R, 4]: the feasible sets of one tbc_scan
    (TB_SCAN_FEASIBLE_SETS) launch, then one tbc_reachable_sets launch.  Same result: dict(X, L, fail_stage)."""
    torch = torch_mod()
    B, G, W = records.shape
    dev = records.device
    check_grid(grid, B, G)
    check_glen(glen, B, grid)
    for t, what in ((sdmin, "sdmin"), (sdmax, "sdmax")):
        check_path_vector(t, B, what)
    X = scan_cones(records, R, cones, grid, feasible_sets=True, glen=glen)["K"]
    table = _cone_table(cones, R)
    L = torch.empty((B, G, 2), dtype=torch.float64, device=dev)
    fs = torch.empty((B,), dtype=torch.int32, device=dev)
    with torch.cuda.device(dev):
        rc = _lib_cones.load().tbc_reachable_sets(
            _lib.ptr(records), W, int(R), ctypes.c_void_p(table.ctypes.data),
            SCAN_FLAGS["ubound"] if has_ubound(records, R) else 0, _lib.ptr(grid), 1 if grid.dim() == 1 else 0, B, G,
            _lib.ptr(glen), _lib.ptr(X), _lib.ptr(sdmin), _lib.ptr(sdmax), _lib.ptr(L), _lib.ptr(fs),
            _lib.stream_ptr())
    _lib.check(rc, "tbc_reachable_sets")
    return dict(X=X, L=L, fail_stage=fs)


def propose_gridpoints(ppoly, breaks, max_err_threshold=1e-4, max_iteration=100, max_seg_length=0.05, min_nb_points=100,
                       max_points=2048):
    """propose_gridpoints for B paths (tb_propose_gridpoints).  Returns (grid [B, max_points] padded with the path end,
    glen [B] int32, status [B] int32: 0 ok, 1 = no good grid within max_iteration passes, < 0 = max_points exceeded)."""
    torch = torch_mod()
    B, kc, nseg, dof = ppoly.shape
    dev = ppoly.device
    check_grid_shapes(B, breaks, nseg + 1, breaks, nseg + 1)
    grid = torch.empty((B, int(max_points)), dtype=torch.float64, device=dev)
    scratch = torch.empty_like(grid)
    glen = torch.empty((B,), dtype=torch.int32, device=dev)
    status = torch.empty((B,), dtype=torch.int32, device=dev)
    if not is_cubic(ppoly):
        with torch.cuda.device(dev):
            rc = _lib_poly.load().tbp_propose_gridpoints(_lib.ptr(ppoly), _lib.ptr(breaks), 1 if breaks.dim() == 1 else 0, B,
                                                         kc, nseg, dof, float(max_err_threshold), int(max_iteration),
                                                         float(max_seg_length), int(min_nb_points), int(max_points),
                                                         _lib.ptr(grid), _lib.ptr(scratch), _lib.ptr(glen),
                                                         _lib.ptr(status), _lib.stream_ptr())
        _lib.check(rc, "tbp_propose_gridpoints")
        return grid, glen, status
    with torch.cuda.device(dev):
        rc = _lib.load().tb_propose_gridpoints(_lib.ptr(ppoly), _lib.ptr(breaks), 1 if breaks.dim() == 1 else 0, B, nseg,
                                               dof, float(max_err_threshold), int(max_iteration), float(max_seg_length),
                                               int(min_nb_points), int(max_points), _lib.ptr(grid), _lib.ptr(scratch),
                                               _lib.ptr(glen), _lib.ptr(status), _lib.stream_ptr())
    _lib.check(rc, "tb_propose_gridpoints")
    return grid, glen, status


def sd_bisect(x_fast, u_fast, x_slow, u_slow, grid, desired, atol=1e-5, status_in=None, max_iter=200, glen=None):
    """TOPPRAsd blend (tb_sd_bisect).  Returns dict(sd [B,G], u [B,G-1], info [B,4] = (alpha, fastest, slowest duration,
    bisection steps), status [B]).  glen: optional int32 [B] gridpoints per path (ragged batch, tb_sd_bisect_ragged)."""
    torch = torch_mod()
    B, G = x_fast.shape
    dev = x_fast.device
    check_grid(grid, B, G)
    check_glen(glen, B, grid)
    check_path_vector(desired, B, "desired_duration")
    check_shape(x_slow, (B, G), "x_slow")
    for t, what in ((u_fast, "u_fast"), (u_slow, "u_slow")):
        check_shape(t, (B, G - 1), what)
    if status_in is not None and (status_in.dtype != torch.int32 or tuple(status_in.shape) != (B,)):
        raise ValueError("status_in must be an int32 tensor of shape (%d,)" % B)
    sd = torch.empty((B, G), dtype=torch.float64, device=dev)
    u = torch.empty((B, G - 1), dtype=torch.float64, device=dev)
    info = torch.empty((B, 4), dtype=torch.float64, device=dev)
    status = torch.empty((B,), dtype=torch.int32, device=dev)
    lib = _lib.load()
    args = (_lib.ptr(x_fast), _lib.ptr(u_fast), _lib.ptr(x_slow), _lib.ptr(u_slow), _lib.ptr(grid),
            1 if grid.dim() == 1 else 0, B, G)
    rest = (_lib.ptr(desired), float(atol), int(max_iter), _lib.ptr(status_in), _lib.ptr(sd), _lib.ptr(u), _lib.ptr(info),
            _lib.ptr(status), _lib.stream_ptr())
    with torch.cuda.device(dev):
        if glen is None:
            rc = lib.tb_sd_bisect(*args, *rest)
        else:
            rc = lib.tb_sd_bisect_ragged(*args, _lib.ptr(glen), *rest)
    _lib.check(rc, "tb_sd_bisect")
    return dict(sd=sd, u=u, info=info, status=status)


def spline_time_stamps(sd, grid, glen=None):
    """ParametrizeSpline knots (tb_spline_time_stamps).  Returns (t [B,G], s [B,G] compacted + padded, nkeep [B] int32)."""
    torch = torch_mod()
    B, G = sd.shape
    dev = sd.device
    check_grid(grid, B, G)
    check_glen(glen, B, grid)
    t = torch.empty((B, G), dtype=torch.float64, device=dev)
    s = torch.empty((B, G), dtype=torch.float64, device=dev)
    nkeep = torch.empty((B,), dtype=torch.int32, device=dev)
    with torch.cuda.device(dev):
        rc = _lib.load().tb_spline_time_stamps(_lib.ptr(sd), _lib.ptr(grid), 1 if grid.dim() == 1 else 0, _lib.ptr(glen), B,
                                               G, _lib.ptr(t), _lib.ptr(s), _lib.ptr(nkeep), _lib.stream_ptr())
    _lib.check(rc, "tb_spline_time_stamps")
    return t, s, nkeep


def solve_velacc_host(ss, wp, grid, vlim, alim, interp=True, sd_start=None, sd_end=None, device=0):
    """Pure C-ABI pipeline with HOST (numpy) buffers: tb_solve_velacc_host.  No torch involved."""
    lib = _lib.load()
    ss = np.ascontiguousarray(ss, dtype=np.float64)
    wp = np.ascontiguousarray(wp, dtype=np.float64)
    grid = np.ascontiguousarray(grid, dtype=np.float64)
    B, n, dof = wp.shape
    G = grid.shape[0]
    alim = np.ascontiguousarray(alim, dtype=np.float64)
    shared = alim.ndim == 2
    if vlim is not None:
        vlim = np.ascontiguousarray(vlim, dtype=np.float64)
        if (vlim.ndim == 2) != shared:
            vlim = np.ascontiguousarray(np.broadcast_to(vlim, (B, dof, 2)))
            alim = np.ascontiguousarray(np.broadcast_to(alim, (B, dof, 2)))
            shared = False
    K = np.empty((B, G, 2))
    sd = np.empty((B, G))
    u = np.empty((B, max(G - 1, 1)))
    status = np.empty((B,), dtype=np.int32)

    def hp(arr):
        return None if arr is None else ctypes.c_void_p(arr.ctypes.data)

    s0 = None if sd_start is None else np.ascontiguousarray(np.broadcast_to(sd_start, (B,)), dtype=np.float64)
    s1 = None if sd_end is None else np.ascontiguousarray(np.broadcast_to(sd_end, (B,)), dtype=np.float64)
    rc = lib.tb_solve_velacc_host(int(device), hp(ss), hp(wp), B, n, dof, hp(grid), G, hp(vlim), hp(alim),
                                  1 if shared else 0, 1 if interp else 0, hp(s0), hp(s1), hp(K), hp(sd), hp(u),
                                  hp(status))
    _lib.check(rc, "tb_solve_velacc_host")
    return dict(K=K, sd=sd, u=u[:, :G - 1], status=status)


def lp2d_batch(v, a, b, c, low, high, active_c=None):
    """Batched 2-variable LPs on device (tb_lp2d_batch).  Inputs numpy or tensors: v [B,3], a/b/c [B,n],
    low/high [B,2], active_c [B,2] int.  Returns numpy (result [B], optval [B], optvar [B,2], active [B,2])."""
    torch = torch_mod()
    dev = default_device()
    v = as_device(v, dev)
    B = v.shape[0]
    a, b, c = (as_device(t, dev).reshape(B, -1) for t in (a, b, c))
    n = a.shape[1]
    low, high = as_device(low, dev), as_device(high, dev)
    act = None if active_c is None else as_device(np.asarray(active_c), dev, torch.int32)
    result = torch.empty((B,), dtype=torch.int32, device=dev)
    optval = torch.empty((B,), dtype=torch.float64, device=dev)
    optvar = torch.empty((B, 2), dtype=torch.float64, device=dev)
    active = torch.empty((B, 2), dtype=torch.int32, device=dev)
    with torch.cuda.device(dev):
        rc = _lib.load().tb_lp2d_batch(_lib.ptr(v), _lib.ptr(a) if n else None, _lib.ptr(b) if n else None,
                                       _lib.ptr(c) if n else None, _lib.ptr(low), _lib.ptr(high), _lib.ptr(act), B, n,
                                       _lib.ptr(result), _lib.ptr(optval), _lib.ptr(optvar), _lib.ptr(active),
                                       _lib.stream_ptr())
    _lib.check(rc, "tb_lp2d_batch")
    return result.cpu().numpy(), optval.cpu().numpy(), optvar.cpu().numpy(), active.cpu().numpy()


def lp1d_batch(v, a, b, low, high):
    """Batched 1-variable LPs on device (tb_lp1d_batch).  v [B,2], a/b [B,n], low/high [B]."""
    torch = torch_mod()
    dev = default_device()
    v = as_device(v, dev)
    B = v.shape[0]
    a, b = (as_device(t, dev).reshape(B, -1) for t in (a, b))
    n = a.shape[1]
    low, high = as_device(low, dev), as_device(high, dev)
    result = torch.empty((B,), dtype=torch.int32, device=dev)
    optval = torch.empty((B,), dtype=torch.float64, device=dev)
    optvar = torch.empty((B,), dtype=torch.float64, device=dev)
    active = torch.empty((B,), dtype=torch.int32, device=dev)
    with torch.cuda.device(dev):
        rc = _lib.load().tb_lp1d_batch(_lib.ptr(v), _lib.ptr(a) if n else None, _lib.ptr(b) if n else None,
                                       _lib.ptr(low), _lib.ptr(high), B, n, _lib.ptr(result), _lib.ptr(optval),
                                       _lib.ptr(optvar), _lib.ptr(active), _lib.stream_ptr())
    _lib.check(rc, "tb_lp1d_batch")
    return result.cpu().numpy(), optval.cpu().numpy(), optvar.cpu().numpy(), active.cpu().numpy()


def time_grid(sd, grid):
    """K3: const-accel time stamps.  sd [B,G], grid [G] or [B,G] -> (t_grid [B,G], us [B,G-1])."""
    torch = torch_mod()
    B, G = sd.shape
    t = torch.empty((B, G), dtype=torch.float64, device=sd.device)
    us = torch.empty((B, G - 1), dtype=torch.float64, device=sd.device)
    with torch.cuda.device(sd.device):
        rc = _lib.load().tb_time_grid(_lib.ptr(sd), _lib.ptr(grid), 1 if grid.dim() == 1 else 0, B, G, _lib.ptr(t),
                                      _lib.ptr(us), _lib.stream_ptr())
    _lib.check(rc, "tb_time_grid")
    return t, us


def constaccel_eval(ppoly, breaks, grid, sd, t_grid, us, ts, order):
    """K3: q / qd / qdd at times ts ([M] shared or [B,M]) -> [B,M,dof]."""
    torch = torch_mod()
    B, kc, nseg, dof = ppoly.shape
    G = sd.shape[1]
    M = ts.shape[-1]
    out = torch.empty((B, M, dof), dtype=torch.float64, device=sd.device)
    if not is_cubic(ppoly):
        with torch.cuda.device(sd.device):
            rc = _lib_poly.load().tbp_constaccel_eval(_lib.ptr(ppoly), _lib.ptr(breaks), 1 if breaks.dim() == 1 else 0, kc,
                                                      nseg, dof, _lib.ptr(grid), 1 if grid.dim() == 1 else 0,
                                                      _lib.ptr(sd), _lib.ptr(t_grid), _lib.ptr(us), B, G, _lib.ptr(ts),
                                                      1 if ts.dim() == 1 else 0, M, int(order), _lib.ptr(out),
                                                      _lib.stream_ptr())
        _lib.check(rc, "tbp_constaccel_eval")
        return out
    with torch.cuda.device(sd.device):
        rc = _lib.load().tb_constaccel_eval(_lib.ptr(ppoly), _lib.ptr(breaks), 1 if breaks.dim() == 1 else 0, nseg, dof,
                                            _lib.ptr(grid), 1 if grid.dim() == 1 else 0, _lib.ptr(sd), _lib.ptr(t_grid),
                                            _lib.ptr(us), B, G, _lib.ptr(ts), 1 if ts.dim() == 1 else 0, M, int(order),
                                            _lib.ptr(out), _lib.stream_ptr())
    _lib.check(rc, "tb_constaccel_eval")
    return out


def xbound_varying(ppoly, breaks, grid, vlim_grid, records, R_total, write_xbound):
    """Velocity bound with per-gridpoint limits vlim_grid [G,dof,2] or [B,G,dof,2] into the xbound slots."""
    torch = torch_mod()
    B, _, nseg, dof = ppoly.shape
    G = grid.shape[-1]
    W = records.shape[-1]
    check_grid_shapes(B, breaks, nseg + 1, grid, G)
    check_vlim_grid(vlim_grid, B, G, dof)
    if not is_cubic(ppoly):
        xbound_varying_sampled(ppoly_eval(ppoly, breaks, grid, 1), vlim_grid, records, R_total, write_xbound)
        return
    with torch.cuda.device(records.device):
        rc = _lib.load().tb_xbound_varying(_lib.ptr(ppoly), _lib.ptr(breaks), 1 if breaks.dim() == 1 else 0, B, nseg, dof,
                                           _lib.ptr(grid), 1 if grid.dim() == 1 else 0, G, _lib.ptr(vlim_grid),
                                           1 if vlim_grid.dim() == 3 else 0, _lib.ptr(records), W, int(R_total),
                                           int(write_xbound), _lib.stream_ptr())
    _lib.check(rc, "tb_xbound_varying")


def xbound_varying_sampled(qd, vlim_grid, records, R_total, write_xbound):
    """xbound_varying from sampled qd = q'(grid) [B, G, dof] (tbp_xbound_varying_sampled)."""
    torch = torch_mod()
    B, G, dof = qd.shape
    W = records.shape[-1]
    check_vlim_grid(vlim_grid, B, G, dof)
    if tuple(records.shape[:2]) != (B, G):
        raise ValueError("records must have shape (%d, %d, W); got %s" % (B, G, tuple(records.shape)))
    with torch.cuda.device(records.device):
        rc = _lib_poly.load().tbp_xbound_varying_sampled(_lib.ptr(qd), B, dof, G, _lib.ptr(vlim_grid),
                                                         1 if vlim_grid.dim() == 3 else 0, _lib.ptr(records), W,
                                                         int(R_total), int(write_xbound), _lib.stream_ptr())
    _lib.check(rc, "tbp_xbound_varying_sampled")
