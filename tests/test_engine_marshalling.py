"""CPU: the ctypes layer between the Python host and the C-ABI, checked without a GPU.

1. Every prototype in toppra_b200/_lib.py agrees with the declaration in include/toppra_b200.h (argument count and kind:
   pointer / int / double) — a mismatch there would be undefined behaviour on the GPU, not an exception.
2. Every tensor-level function of toppra_b200/engine.py is run on CPU tensors against a RECORDING library: no kernel runs,
   but the call each function would make is checked against its prototype (count, ints are ints, pointers are tensors'
   data pointers or NULL), the launch flags are checked for the modes that have them, and the shape / dtype validation is
   shown to raise before anything reaches the library.
The numbers come from the `-m gpu` tests; this file pins the plumbing in front of them."""
import contextlib
import ctypes
import os
import re

import numpy as np
import pytest
import torch

from toppra_b200 import _lib, engine

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ---- 1. header <-> prototypes ------------------------------------------------------------------------------------
def header_prototypes():
    """{name: (kinds, return kind)} with kind in {"ptr", "int", "double"} parsed from the declarations."""
    text = open(os.path.join(ROOT, "include", "toppra_b200.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    text = re.sub(r"//[^\n]*", "", text)
    out = {}
    for ret, name, args in re.findall(r"\b(int|const char \*)\s*(tb_[a-z0-9_]+)\s*\(([^)]*)\)\s*;", text):
        kinds, names = [], []
        for arg in [a.strip() for a in args.split(",")]:
            if arg in ("", "void"):
                continue
            if "*" in arg:
                kinds.append("ptr")
            elif re.match(r"(const\s+)?double\b", arg):
                kinds.append("double")
            elif re.match(r"(const\s+)?int\b", arg):
                kinds.append("int")
            else:
                raise AssertionError("unparsed argument %r of %s" % (arg, name))
            names.append(re.findall(r"[A-Za-z_][A-Za-z_0-9]*", arg)[-1])
        out[name] = (kinds, "ptr" if "*" in ret else "int")
        PARAM_NAMES[name] = names
    return out


PARAM_NAMES = {}     # {entry point: parameter names of the header declaration}, filled by header_prototypes()


def named_args(name, args):
    """{parameter name: value} of one recorded call, by the header's parameter names."""
    if not PARAM_NAMES:
        header_prototypes()
    return dict(zip(PARAM_NAMES[name], args))


def _kind(ctype):
    if ctype is ctypes.c_int:
        return "int"
    if ctype is ctypes.c_double:
        return "double"
    if ctype in (ctypes.c_void_p, ctypes.c_char_p) or hasattr(ctype, "contents") or issubclass(ctype, ctypes._Pointer):
        return "ptr"
    raise AssertionError("unexpected ctypes type %r" % (ctype,))


def test_ctypes_prototypes_match_the_header():
    declared = header_prototypes()
    assert len(declared) >= 30
    for name, (argtypes, restype) in _lib._PROTOS.items():
        kinds, ret = declared[name]
        assert [_kind(t) for t in argtypes] == kinds, name
        assert _kind(restype) == ret, name


# ---- 2. engine.py against a recording library ----------------------------------------------------------------------
class RecordingLib(object):
    """Stands in for the loaded shared library: every entry point records its arguments, checks them against the ctypes
    prototype and reports success."""

    # the two size queries answer like the library does (toppra_b200.h: W = 3R + 2 rounded up to even)
    RESULTS = {"tb_record_doubles": lambda R: (3 * R + 2 + 1) & ~1,
               "tb_spline_fit_workspace_doubles": lambda B, n, dof: 7 * B * n * dof}

    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        if name not in _lib._PROTOS:
            raise AttributeError(name)
        argtypes, _ = _lib._PROTOS[name]

        def entry(*args):
            assert len(args) == len(argtypes), "%s: %d arguments, prototype has %d" % (name, len(args), len(argtypes))
            for k, (a, t) in enumerate(zip(args, argtypes)):
                kind = _kind(t)
                if kind == "int":
                    assert isinstance(a, (int, np.integer)) and not isinstance(a, bool), (name, k, a)
                elif kind == "double":
                    assert isinstance(a, float), (name, k, a)
                else:
                    assert a is None or isinstance(a, (ctypes.c_void_p, int)), (name, k, a)
            self.calls.append((name, args))
            return self.RESULTS.get(name, lambda *a: 0)(*args)

        return entry

    def last(self, name):
        for n, args in reversed(self.calls):
            if n == name:
                return args
        raise AssertionError("no call of " + name)


@pytest.fixture
def lib(monkeypatch):
    rec = RecordingLib()
    monkeypatch.setattr(_lib, "require_cuda", lambda: torch)
    monkeypatch.setattr(_lib, "load", lambda: rec)
    monkeypatch.setattr(_lib, "stream_ptr", lambda: ctypes.c_void_p(0))
    monkeypatch.setattr(torch.cuda, "device", lambda dev: contextlib.nullcontext())
    monkeypatch.setattr(engine, "default_device", lambda device=None: torch.device("cpu"))
    return rec


B, G, DOF, NSEG = 3, 11, 2, 4


def _path():
    ppoly = torch.zeros((B, 4, NSEG, DOF), dtype=torch.float64)
    breaks = torch.linspace(0, 1, NSEG + 1, dtype=torch.float64)
    grid = torch.linspace(0, 1, G, dtype=torch.float64)
    return ppoly, breaks, grid


def _lims():
    return torch.ones((DOF, 2), dtype=torch.float64), torch.ones((DOF, 2), dtype=torch.float64)


def test_every_engine_entry_marshals_its_prototype(lib):
    ppoly, breaks, grid = _path()
    vlim, alim = _lims()
    vec = torch.zeros(B, dtype=torch.float64)
    c = engine.spline_fit(breaks, torch.zeros((B, NSEG + 1, DOF), dtype=torch.float64))
    assert tuple(c.shape) == (B, 4, NSEG, DOF)
    assert tuple(engine.ppoly_eval(ppoly, breaks, grid, 1).shape) == (B, G, DOF)
    R = 2 * DOF * 2
    records, W = engine.alloc_records(B, G, R, torch.device("cpu"))
    assert W == engine.record_doubles(R) and not engine.has_ubound(records, R)
    engine.coeff_velacc(ppoly, breaks, grid, vlim, alim, True, records, R)
    out = engine.scan(records, R, grid, vec, vec)
    assert set(out) == {"K", "sd", "u", "status", "fail_stage"} and tuple(out["u"].shape) == (B, G - 1)
    flags = lib.last("tb_scan_ragged")[11]
    assert flags == 0
    engine.scan(records, R, grid, vec, vec, backward_only=True, counters=True)
    assert lib.last("tb_scan_ragged")[11] == engine.SCAN_FLAGS["backward_only"]
    engine.scan(records, R, grid, vec, vec, sd_forward="slow", fast_lower=True)
    assert lib.last("tb_scan_ragged")[11] == engine.SCAN_FLAGS["sd_slow"] | engine.SCAN_FLAGS["fast_lower"]
    rec_ub, _ = engine.alloc_records(B, G, R, torch.device("cpu"), ubound=True)
    assert engine.has_ubound(rec_ub, R)
    engine.scan(rec_ub, R, grid, vec, vec, fast_lower=True)       # fast_lower is dropped when u-bounds are present
    assert lib.last("tb_scan_ragged")[11] == engine.SCAN_FLAGS["ubound"]
    ragged = grid.expand(B, G).contiguous()
    glen = torch.full((B,), G, dtype=torch.int32)
    engine.scan(records, R, ragged, vec, vec, glen=glen)
    assert lib.last("tb_scan_ragged")[7] is not None
    xb = engine.xbound_velocity(ppoly, breaks, grid, vlim)
    assert tuple(xb.shape) == (B, G, 2)
    out = engine.scan_velacc(ppoly, breaks, grid, alim, True, xb, vec, vec)
    assert tuple(out["K"].shape) == (B, G, 2)
    engine.scan_velacc(ppoly, breaks, ragged, alim, True, xb, vec, vec, glen=glen)
    assert tuple(engine.feasible_sets(records, R, grid).shape) == (B, G, 2)
    assert lib.last("tb_feasible_sets_ex")[7] == 0
    engine.feasible_sets(rec_ub, R, grid)
    assert lib.last("tb_feasible_sets_ex")[7] == engine.SCAN_FLAGS["ubound"]
    out = engine.reachable_sets(records, R, grid, vec, vec)
    assert tuple(out["L"].shape) == (B, G, 2) and out["fail_stage"].dtype == torch.int32
    out = engine.scan_robust(records, R, 0, R, np.array([0.1, 0.1, 0.1]), grid, vec, vec)
    assert tuple(out["sd"].shape) == (B, G)
    engine.scan_robust(records, R, 0, R, np.array([0.1, 0.1, 0.1]), grid, feasible_sets=True)
    gridp, glen2, status = engine.propose_gridpoints(ppoly, breaks, max_points=64)
    assert tuple(gridp.shape) == (B, 64) and glen2.dtype == torch.int32 and status.dtype == torch.int32
    x = torch.zeros((B, G), dtype=torch.float64)
    u = torch.zeros((B, G - 1), dtype=torch.float64)
    out = engine.sd_bisect(x, u, x, u, grid, vec)
    assert tuple(out["info"].shape) == (B, 4)
    t, s, nkeep = engine.spline_time_stamps(x, grid)
    assert tuple(t.shape) == (B, G) and nkeep.dtype == torch.int32
    tg, us = engine.time_grid(x, grid)
    assert tuple(us.shape) == (B, G - 1)
    q = engine.constaccel_eval(ppoly, breaks, grid, x, tg, us, torch.zeros(5, dtype=torch.float64), 0)
    assert tuple(q.shape) == (B, 5, DOF)
    engine.init_bounds(records, R)
    # sizes and the main arrays land in the parameters the header NAMES for them (catches swapped arguments of one kind)
    sizes = {"B": B, "G": G, "dof": DOF, "nseg": NSEG}
    arrays = {"ppoly": (ppoly.data_ptr(), c.data_ptr()), "breaks": (breaks.data_ptr(),)}   # c: the fit's OUTPUT
    for name, args in lib.calls:
        named = named_args(name, args)
        for key, want in sizes.items():
            if key in named and name != "tb_propose_gridpoints":
                assert named[key] == want, (name, key, named[key])
        for key, want in arrays.items():
            if key in named:
                assert named[key].value in want, (name, key)
        if "grid" in named and named.get("grid_shared") == 1:
            assert named["grid"].value == grid.data_ptr(), name
        if "records" in named and "W" in named and name != "tb_xbound_velocity":      # that one writes a [B, G, 2] array
            assert named["records"].value in (records.data_ptr(), rec_ub.data_ptr()) and \
                named["W"] in (records.shape[-1], rec_ub.shape[-1]), name
    seen = {name for name, _ in lib.calls}
    assert {"tb_spline_fit", "tb_ppoly_eval", "tb_coeff_velacc", "tb_scan_ragged", "tb_scan_velacc_ragged",
            "tb_xbound_velocity", "tb_feasible_sets_ex", "tb_reachable_sets", "tb_scan_robust", "tb_propose_gridpoints",
            "tb_sd_bisect", "tb_spline_time_stamps", "tb_time_grid", "tb_constaccel_eval", "tb_init_bounds"} <= seen


def test_row_builders_and_host_entry_marshal(lib):
    ppoly, breaks, grid = _path()
    vlim, alim = _lims()
    m, k = DOF, 3
    R = 2 * k + 4 * DOF + 2 * DOF
    records, _ = engine.alloc_records(B, G, R, torch.device("cpu"))
    a = torch.zeros((B, G, m), dtype=torch.float64)
    F0, g0 = torch.zeros((k, m), dtype=torch.float64), torch.zeros(k, dtype=torch.float64)
    assert engine.rows_canlinear(a, a, a, F0, g0, 0, grid, True, records, R, 0) == 2 * k
    F1, g1 = torch.zeros((B, G, k, m), dtype=torch.float64), torch.zeros((B, G, k), dtype=torch.float64)
    assert engine.rows_canlinear(a, a, a, F1, g1, 1, grid, False, records, R, 0) == k
    assert engine.rows_canlinear(a, a, a, None, torch.zeros(2 * m, dtype=torch.float64), 2, grid, True, records, R, 2 * k) == 4 * m
    assert lib.last("tb_rows_canlinear")[3] is None and lib.last("tb_rows_canlinear")[9] == 2 * m
    assert engine.rows_canlinear(a, a, a, None, torch.zeros((B, 2 * m), dtype=torch.float64), 3, grid, False, records, R, 0) == 2 * m
    taulim = torch.ones((DOF, 2), dtype=torch.float64)
    assert engine.coeff_second_order("pendulums", [1.0, 2.0, 3.0, 4.0], ppoly, breaks, grid, taulim, None, True,
                                     records, R, 0) == 4 * DOF
    args = lib.last("tb_coeff_second_order")
    assert args[0] == engine.DEVICE_MODELS["pendulums"] and args[2] == 4 and args[13] == 1 and args[14] is None
    engine.xbound_constant(ppoly, breaks, grid, vlim, records, R, 1)
    engine.xbound_varying(ppoly, breaks, grid, torch.ones((G, DOF, 2), dtype=torch.float64), records, R, 1)
    assert lib.last("tb_xbound_varying")[10] == 1
    out = engine.solve_velacc_host(np.linspace(0, 1, 5), np.zeros((B, 5, DOF)), np.linspace(0, 1, G), np.ones((DOF, 2)),
                                   np.ones((B, DOF, 2)), sd_start=0.0)
    args = lib.last("tb_solve_velacc_host")
    assert args[10] == 0 and args[13] is None and out["u"].shape == (B, G - 1)     # mixed limits -> per path; sd_end NULL
    n0 = len(lib.calls)
    for call in (lambda: engine.rows_canlinear(a, a[:, :-1].contiguous(), a, F0, g0, 0, grid, True, records, R, 0),
                 lambda: engine.rows_canlinear(a, a, a, F0, g1, 0, grid, True, records, R, 0),
                 lambda: engine.rows_canlinear(a, a, a, F1[:1].contiguous(), g1, 1, grid, True, records, R, 0),
                 lambda: engine.rows_canlinear(a, a, a, None, g0, 2, grid, True, records, R, 0),
                 lambda: engine.rows_canlinear(a, a, a, F0, g0, 0, grid, True, records[:1], R, 0),
                 lambda: engine.coeff_second_order("pendulums", [1.0], ppoly, breaks, grid, torch.ones((B + 1, DOF, 2),
                                                   dtype=torch.float64), None, True, records, R, 0),
                 lambda: engine.xbound_varying(ppoly, breaks, grid, torch.ones((G + 1, DOF, 2), dtype=torch.float64),
                                               records, R, 1)):
        with pytest.raises(ValueError):
            call()
    assert len(lib.calls) == n0


def test_lp_batches_marshal(lib):
    r, val, var, act = engine.lp2d_batch(np.zeros((2, 3)), np.zeros((2, 5)), np.zeros((2, 5)), np.zeros((2, 5)),
                                         np.zeros((2, 2)), np.ones((2, 2)), np.zeros((2, 2), dtype=np.int64))
    assert r.shape == (2,) and var.shape == (2, 2) and act.dtype == np.int32
    r, val, var, act = engine.lp1d_batch(np.zeros((2, 2)), np.zeros((2, 0)), np.zeros((2, 0)), np.zeros(2), np.ones(2))
    assert lib.last("tb_lp1d_batch")[1] is None and lib.last("tb_lp1d_batch")[6] == 0      # no rows: NULL row pointers


def test_shape_and_dtype_errors_are_raised_before_the_library_is_called(lib):
    ppoly, breaks, grid = _path()
    vlim, alim = _lims()
    R = 2 * DOF * 2
    records, _ = engine.alloc_records(B, G, R, torch.device("cpu"))
    vec = torch.zeros(B, dtype=torch.float64)
    bad_grid = torch.linspace(0, 1, G + 1, dtype=torch.float64)
    bad_vec = torch.zeros(B + 1, dtype=torch.float64)
    x = torch.zeros((B, G), dtype=torch.float64)
    u = torch.zeros((B, G - 1), dtype=torch.float64)
    n0 = len(lib.calls)
    cases = [
        lambda: engine.scan(records, R, bad_grid, vec, vec),
        lambda: engine.scan(records, R, grid, bad_vec, vec),
        lambda: engine.scan(records, R, grid, vec, vec, glen=torch.full((B,), G, dtype=torch.int32)),   # shared grid
        lambda: engine.scan(records, R, grid.expand(B, G).contiguous(), vec, vec, glen=torch.full((B,), G)),  # int64
        lambda: engine.feasible_sets(records, R, bad_grid),
        lambda: engine.reachable_sets(records, R, bad_grid, vec, vec),
        lambda: engine.reachable_sets(records, R, grid, bad_vec, vec),
        lambda: engine.sd_bisect(x, u, x, u, bad_grid, vec),
        lambda: engine.sd_bisect(x, u, x[:, :-1].contiguous(), u, grid, vec),
        lambda: engine.sd_bisect(x, u, x, u, grid, bad_vec),
        lambda: engine.sd_bisect(x, u, x, u, grid, vec, status_in=torch.zeros(B, dtype=torch.int64)),
        lambda: engine.spline_time_stamps(x, bad_grid),
        lambda: engine.coeff_velacc(ppoly, breaks, grid, torch.ones((B + 1, DOF, 2), dtype=torch.float64), alim, True,
                                    records, R),
        lambda: engine.scan(records.to(torch.float32), R, grid, vec, vec),
        lambda: engine.feasible_sets(records.transpose(0, 1), R, grid),
    ]
    for k, call in enumerate(cases):
        with pytest.raises(ValueError):
            call()
        assert len(lib.calls) == n0, "case %d reached the library" % k


def test_ptr_accepts_only_what_the_cabi_takes():
    assert _lib.ptr(None) is None
    assert isinstance(_lib.ptr(torch.zeros(3, dtype=torch.float64)), ctypes.c_void_p)
    assert isinstance(_lib.ptr(torch.zeros(3, dtype=torch.int32)), ctypes.c_void_p)
    for bad in (torch.zeros(3, dtype=torch.float32), torch.zeros(3, dtype=torch.int64), torch.zeros(3, dtype=torch.bool),
                torch.zeros((3, 2), dtype=torch.float64).t()):
        with pytest.raises(ValueError):
            _lib.ptr(bad)
