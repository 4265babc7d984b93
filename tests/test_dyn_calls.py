"""What the host code hands to libtoppra_b200_dyn.so and tb_rows_canlinear, checked without a GPU.

The libraries are replaced by recorders and the tensors are CPU tensors that the package takes for CUDA tensors.  For
each of the 12 RigidBodyModel / RigidBodyFrame methods, and for the device route of each of the six rigid-body
constraints, every C-ABI call is recorded: its entry, its scalars, the contents of every host array (model, frame, S,
object, base) and which tensor sits in each pointer slot, with its shape."""
import contextlib
import ctypes
import os
import types

import numpy as np
import pytest

torch = pytest.importorskip("torch")

ROBOTS = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "robots")

# host-array slots other than the model (slot 0): (entry, slot) -> number of doubles
_HOST = {("tbd_velocity_norm_terms", 3): 36, ("tbd_contact_wrench", 3): 10, ("tbd_contact_wrench_terms", 3): 10,
         ("tbd_support_wrench", 3): 4, ("tbd_support_wrench_terms", 3): 4}
_OUTPUTS = {"tbd_rnea": 1, "tbd_torque_terms": 3, "tbd_frame_velocity": 1, "tbd_velocity_norm_terms": 1,
            "tbd_frame_acceleration": 1, "tbd_acceleration_terms": 2, "tbd_contact_wrench": 1,
            "tbd_contact_wrench_terms": 3, "tbd_frame_inverse_inertia": 1, "tbd_collision_energy_terms": 1,
            "tbd_support_wrench": 1, "tbd_support_wrench_terms": 3}


class _Dev(torch.Tensor):
    """A CPU tensor the package takes for a CUDA tensor."""

    @property
    def is_cuda(self):
        return True


def _dev(x):
    return torch.as_tensor(np.asarray(x, dtype=np.float64)).as_subclass(_Dev)


def _host_doubles(name, slot, args):
    if not name.startswith("tbd_"):
        return None
    if slot == 0:
        return 3 + 27 * args[1]
    if slot == 2 and name not in ("tbd_rnea", "tbd_torque_terms"):
        return 14
    return _HOST.get((name, slot))


class _Recorder(object):
    """Stands in for a library: each call appends [entry, arg...] to the log, with host arrays copied and tensors
    (looked up by address among those passed through _lib.ptr) kept as they are."""

    def __init__(self, protos, log, tensors):
        self.protos, self.log, self.tensors = protos, log, tensors

    def __getattr__(self, name):
        if name not in self.protos:
            raise AttributeError(name)
        argtypes = self.protos[name][0]

        def entry(*args):
            assert len(args) == len(argtypes), name
            rec = [name]
            for slot, x in enumerate(args):
                if isinstance(x, ctypes.c_void_p):
                    x = x.value
                    n = _host_doubles(name, slot, args)
                    if x is None:
                        rec.append(None)
                    elif n is not None:
                        rec.append(np.ctypeslib.as_array((ctypes.c_double * n).from_address(x)).copy())
                    else:
                        rec.append(self.tensors[x])
                else:
                    rec.append(x)
            self.log.append(rec)
            return 0

        return entry


@pytest.fixture
def calls(monkeypatch):
    from toppra_b200 import _lib, _lib_dyn, engine
    log, tensors = [], {}
    real_ptr = _lib.ptr

    def ptr(t):
        p = real_ptr(t)
        if t is not None:
            tensors[p.value] = t
        return p

    main, dyn = _Recorder(_lib._PROTOS, log, tensors), _Recorder(_lib_dyn._PROTOS, log, tensors)
    monkeypatch.setattr(_lib, "ptr", ptr)
    monkeypatch.setattr(_lib, "require_cuda", lambda: torch)
    monkeypatch.setattr(_lib, "load", lambda: main)
    monkeypatch.setattr(_lib_dyn, "load", lambda: dyn)
    monkeypatch.setattr(_lib, "stream_ptr", lambda: ctypes.c_void_p(0))
    monkeypatch.setattr(torch.cuda, "device", lambda dev: contextlib.nullcontext())
    return log


def _canon(log, named):
    """The log with every tensor replaced by (label, shape): the label is the name in `named` it shares its storage
    with, else "<entry>.<slot>" of the dyn output slot it was first seen in, else its contents."""
    labels = {t.data_ptr(): k for k, t in named.items()}
    out = []
    for rec in log:
        name, args = rec[0], rec[1:]
        n_out = _OUTPUTS.get(name, 0)
        row = [name]
        for slot, x in enumerate(args):
            if isinstance(x, torch.Tensor):
                key = x.data_ptr()
                if key not in labels and name.startswith("tbd_") and len(args) - 1 - n_out <= slot < len(args) - 1:
                    labels[key] = "%s.%d" % (name, slot)
                label = labels.get(key, tuple(x.reshape(-1).tolist()))
                row.append((label, tuple(x.shape)))
            elif isinstance(x, np.ndarray):
                row.append(("host", tuple(x.tolist())))
            else:
                row.append(x)
        out.append(row)
    return out


def H(x):
    return ("host", tuple(np.asarray(x, dtype=np.float64).reshape(-1).tolist()))


def T(label, shape):
    return (label, tuple(shape))


@pytest.fixture(scope="module")
def arm():
    import toppra_b200 as ta
    return ta.RigidBodyModel.from_urdf(os.path.join(ROBOTS, "arm6.urdf"))


M = 5


def _inputs(nv, n):
    rng = np.random.default_rng(7)
    return {k: _dev(rng.uniform(-1, 1, (M, nv))) for k in ("q", "qd", "qdd")[:n]}


def test_model_methods(calls, arm):
    nv = arm.nv
    x = _inputs(nv, 3)
    tau = arm(x["q"], x["qd"], x["qdd"])
    assert _canon(calls, dict(x, out=tau)) == [
        ["tbd_rnea", H(arm.packed), nv, M, T("q", (M, nv)), T("qd", (M, nv)), T("qdd", (M, nv)), T("out", (M, nv)),
         None]]
    for fric, fric_slot in ((None, None), (np.zeros(nv), None), (0.5, T(tuple([0.5] * nv), (nv,))),
                            (np.arange(nv) * 0.1, T(tuple((np.arange(nv) * 0.1).tolist()), (nv,)))):
        del calls[:]
        a, b, c = arm.torque_terms(x["q"], x["qd"], x["qdd"], fric)
        assert _canon(calls, dict(x, a=a, b=b, c=c)) == [
            ["tbd_torque_terms", H(arm.packed), nv, M, T("q", (M, nv)), T("qd", (M, nv)), T("qdd", (M, nv)), fric_slot,
             T("a", (M, nv)), T("b", (M, nv)), T("c", (M, nv)), None]]


def test_frame_methods(calls, arm):
    nv = arm.nv
    x = _inputs(nv, 3)
    q, qd, qdd = x["q"], x["qd"], x["qdd"]
    f = arm.frame("tool0" if "tool0" in arm.frames else sorted(arm.frames)[-1], xyz=(0.03, -0.02, 0.1),
                  rpy=(0.3, -0.2, 0.5), reference_frame="local")
    base = arm.frame([k for k, v in arm.frames.items() if v[0] == -1][0], xyz=(0.01, 0.02, 0.0))
    S = np.arange(36.0).reshape(6, 6) / 10
    obj = np.array([0.8, 0.006, -0.004, 0.06, 0.0021, 0.0001, -0.0002, 0.0026, 0.0001, 0.0017])
    pb = np.array([12.0, 0.01, -0.02, 0.1])
    Q, QD, QDD = T("q", (M, nv)), T("qd", (M, nv)), T("qdd", (M, nv))
    cases = [
        (lambda: f(q, qd), "tbd_frame_velocity", [M, Q, QD], [(M, 6)]),
        (lambda: f.velocity_norm_terms(q, qd, S), "tbd_velocity_norm_terms", [H(S), M, Q, QD], [(M,)]),
        (lambda: f.acceleration(q, qd, qdd), "tbd_frame_acceleration", [M, Q, QD, QDD], [(M, 6)]),
        (lambda: f.acceleration_terms(q, qd, qdd, (4, 0, 2)), "tbd_acceleration_terms", [21, M, Q, QD, QDD],
         [(M, 3), (M, 3)]),
        (lambda: f.contact_wrench(obj, q, qd, qdd), "tbd_contact_wrench", [H(obj), M, Q, QD, QDD], [(M, 6)]),
        (lambda: f.contact_wrench_terms(obj, q, qd, qdd), "tbd_contact_wrench_terms", [H(obj), M, Q, QD, QDD],
         [(M, 6)] * 3),
        (lambda: f.inverse_inertia(q), "tbd_frame_inverse_inertia", [M, Q], [(M, 3, 3)]),
        (lambda: f.collision_energy_terms(q, qd, 0.6), "tbd_collision_energy_terms", [0.6, M, Q, QD], [(M,)]),
    ]
    for fr, b_ in ((base, pb), (base, None)):
        packed = pb if b_ is not None else arm.packed_base()
        cases += [
            (lambda fr=fr, b_=b_: fr.support_wrench(b_, q, qd, qdd), "tbd_support_wrench",
             [H(packed), M, Q, QD, QDD], [(M, 6)], fr),
            (lambda fr=fr, b_=b_: fr.support_wrench_terms(b_, q, qd, qdd), "tbd_support_wrench_terms",
             [H(packed), M, Q, QD, QDD], [(M, 6)] * 3, fr)]
    for case in cases:
        run, name, middle, out_shapes = case[:4]
        fr = case[4] if len(case) > 4 else f
        del calls[:]
        out = run()
        outs = out if isinstance(out, tuple) else (out,)
        assert [tuple(o.shape) for o in outs] == out_shapes, name
        named = dict(x, **{"out%d" % i: o for i, o in enumerate(outs)})
        expect = [name, H(arm.packed), nv, H(fr.packed)] + middle + [T("out%d" % i, s) for i, s in enumerate(out_shapes)] + [None]
        assert _canon(calls, named) == [expect], name


class _FakeBatchPath(object):
    """q, q', q'' of a batch: deterministic values that differ by order, path and gridpoint."""

    def __init__(self, B, dof):
        self.B, self.dof, self.device = B, dof, torch.device("cpu")
        self.evals = []

    def eval_device(self, grid, order):
        G = grid.shape[-1]
        v = (np.arange(self.B * G * self.dof).reshape(self.B, G, self.dof) % 17) * 0.01 - 0.05 + 0.3 * order
        t = _dev(v)
        self.evals.append(t)
        return t


def _context(dof, B, G, lo, hi, total):
    from toppra_b200.constraint.linear_constraint import RecordContext
    bp = _FakeBatchPath(hi - lo, dof)
    return RecordContext(bp, torch.linspace(0, 1, G, dtype=torch.float64), None, lo=lo, hi=hi, total=total), bp


W, R_TOTAL, ROW0 = 40, 30, 4


def _run(calls, cons, ctx):
    """num_rows, then append_records on a fresh record buffer; returns (rows, canonical log, the q, qd, qdd tensors)."""
    rows = cons.num_rows(ctx)
    del calls[:]
    records = torch.zeros((ctx.B, ctx.G, W), dtype=torch.float64)
    cons.append_records(ctx, records, R_TOTAL, ROW0)
    named = {"records": records, "grid": ctx.d_grid}
    named.update(("q%d" % i, t) for i, t in enumerate(ctx.bpath.evals))
    return rows, _canon(calls, named)


def _rows_call(a, b, c, F, g, mode, B, G, m, k, interp):
    return ["tb_rows_canlinear", a, b, c, F, g, mode, B, G, m, k, T("grid", (G,)), 1, 1 if interp else 0,
            T("records", (B, G, W)), W, R_TOTAL, ROW0, None]


CHUNKS = [(0, 4, 4), (1, 3, 4)]   # (lo, hi, total): a whole batch, and paths 1..2 of a batch of 4


def _flat(x):
    return tuple(np.asarray(x, dtype=np.float64).reshape(-1).tolist())


@pytest.mark.parametrize("lo,hi,total", CHUNKS)
@pytest.mark.parametrize("interp", [False, True])
def test_joint_torque_route(calls, arm, lo, hi, total, interp):
    from toppra_b200.constraint import JointTorqueConstraint, SecondOrderConstraint
    nv, G = arm.nv, 6
    fric = np.arange(nv) * 0.1
    taulim = np.stack([-np.arange(1.0, nv + 1), np.arange(2.0, nv + 2)], axis=1)
    per_path = np.stack([taulim * (1 + 0.5 * i) for i in range(total)])
    for cons, lim in ((JointTorqueConstraint(arm, taulim, fric, discretization_scheme=int(interp)), taulim),
                      (SecondOrderConstraint.joint_torque_constraint(arm, per_path, fric,
                                                                     discretization_scheme=int(interp)), per_path)):
        ctx, bp = _context(nv, total, G, lo, hi, total)
        B, n = hi - lo, (hi - lo) * G
        rows, log = _run(calls, cons, ctx)
        assert rows == (2 if interp else 1) * 2 * nv
        g = np.concatenate((lim[..., 1], -lim[..., 0]), axis=-1)
        g = g if g.ndim == 1 else g[lo:hi]
        ab = [T("tbd_torque_terms.%d" % s, (B, G, nv)) for s in (7, 8, 9)]
        assert log == [
            ["tbd_torque_terms", H(arm.packed), nv, n, T("q0", (n, nv)), T("q1", (n, nv)), T("q2", (n, nv)),
             T(_flat(fric), (nv,)), T("tbd_torque_terms.7", (n, nv)), T("tbd_torque_terms.8", (n, nv)),
             T("tbd_torque_terms.9", (n, nv)), None],
            _rows_call(ab[0], ab[1], ab[2], None, T(_flat(g), g.shape), 2 if g.ndim == 1 else 3, B, G, nv, 2 * nv,
                       interp)]


@pytest.mark.parametrize("lo,hi,total", CHUNKS)
@pytest.mark.parametrize("interp", [False, True])
def test_cartesian_acceleration_route(calls, arm, lo, hi, total, interp):
    from toppra_b200.constraint import CartesianAccelerationConstraint
    nv, G = arm.nv, 6
    f = arm.frame(sorted(arm.frames)[-1], xyz=(0.0, 0.0, 0.1))
    alim = np.array([[-3.0, 4.0], [-5.0, 6.0]])                 # components (5, 1): row 0 limits wz, row 1 ay
    for lim in (alim, np.stack([alim * (1 + i) for i in range(total)])):
        cons = CartesianAccelerationConstraint(f, lim, components=(5, 1), discretization_scheme=int(interp))
        ctx, bp = _context(nv, total, G, lo, hi, total)
        B, n = hi - lo, (hi - lo) * G
        rows, log = _run(calls, cons, ctx)
        assert rows == (2 if interp else 1) * 4
        srt = lim[..., ::-1, :]                                  # the kernel's columns: ay, wz
        g = np.concatenate((srt[..., 1], -srt[..., 0]), axis=-1)
        g = g if g.ndim == 1 else g[lo:hi]
        assert log == [
            ["tbd_acceleration_terms", H(arm.packed), nv, H(f.packed), 2 + 32, n, T("q0", (n, nv)), T("q1", (n, nv)),
             T("q2", (n, nv)), T("tbd_acceleration_terms.8", (n, 2)), T("tbd_acceleration_terms.9", (n, 2)), None],
            _rows_call(T("tbd_acceleration_terms.8", (B, G, 2)), T("tbd_acceleration_terms.9", (B, G, 2)),
                       T((0.0,) * (B * G * 2), (B, G, 2)), None, T(_flat(g), g.shape), 2 if g.ndim == 1 else 3,
                       B, G, 2, 4, interp)]


@pytest.mark.parametrize("lo,hi,total", CHUNKS)
@pytest.mark.parametrize("interp", [False, True])
@pytest.mark.parametrize("kind", ["contact", "support"])
def test_wrench_routes(calls, arm, lo, hi, total, interp, kind):
    from toppra_b200.constraint import ContactStabilityConstraint, SupportStabilityConstraint
    nv, G = arm.nv, 6
    if kind == "contact":
        f = arm.frame(sorted(arm.frames)[-1], xyz=(0.0, 0.0, 0.1))
        cons = ContactStabilityConstraint(f, 0.8, (0.006, -0.004, 0.06), (0.0021, 0.0001, -0.0002, 0.0026, 0.0001,
                                                                           0.0017), (0.05, 0.04), 0.5,
                                          discretization_scheme=int(interp))
        name, extra = "tbd_contact_wrench_terms", [0.8, 0.006, -0.004, 0.06, 0.0021, 0.0001, -0.0002, 0.0026, 0.0001,
                                                   0.0017]
    else:
        f = arm.frame([k for k, v in arm.frames.items() if v[0] == -1][0], xyz=(0.01, 0.0, 0.0))
        cons = SupportStabilityConstraint(f, polygon=[[-0.1, -0.1], [0.12, -0.1], [0.1, 0.1], [-0.1, 0.08]],
                                          friction=0.6, base_mass=9.0, base_com=(0.0, 0.01, 0.05),
                                          discretization_scheme=int(interp))
        name, extra = "tbd_support_wrench_terms", [9.0, 0.0, 0.01, 0.05]
    k = cons.F.shape[0]
    ctx, bp = _context(nv, total, G, lo, hi, total)
    B, n = hi - lo, (hi - lo) * G
    rows, log = _run(calls, cons, ctx)
    assert rows == (2 if interp else 1) * k
    assert log == [
        [name, H(arm.packed), nv, H(f.packed), H(extra), n, T("q0", (n, nv)), T("q1", (n, nv)), T("q2", (n, nv)),
         T(name + ".8", (n, 6)), T(name + ".9", (n, 6)), T(name + ".10", (n, 6)), None],
        _rows_call(T(name + ".8", (B, G, 6)), T(name + ".9", (B, G, 6)), T(name + ".10", (B, G, 6)),
                   T(_flat(cons.F), (k, 6)), T((0.0,) * k, (k,)), 0, B, G, 6, k, interp)]


@pytest.mark.parametrize("lo,hi,total", CHUNKS)
@pytest.mark.parametrize("interp", [False, True])
@pytest.mark.parametrize("kind", ["velocity", "energy"])
def test_sd2_routes(calls, arm, lo, hi, total, interp, kind):
    from toppra_b200.constraint import CartesianVelocityNorm, CollisionEnergyConstraint
    nv, G = arm.nv, 6
    f = arm.frame(sorted(arm.frames)[-1], xyz=(0.0, 0.0, 0.1))
    S = np.diag([1.0, 1.0, 1.0, 0.1, 0.1, 0.1])
    for limit in (2.5, 0.0, np.arange(total) * 0.5 + 1.0):
        if kind == "velocity":
            cons = CartesianVelocityNorm(f, S, limit, discretization_scheme=int(interp))
            name, extra = "tbd_velocity_norm_terms", [H(S)]
        else:
            cons = CollisionEnergyConstraint(f, limit, 0.6, discretization_scheme=int(interp))
            name, extra = "tbd_collision_energy_terms", [0.6]
        ctx, bp = _context(nv, total, G, lo, hi, total)
        B, n = hi - lo, (hi - lo) * G
        rows, log = _run(calls, cons, ctx)
        assert rows == (2 if interp else 1)
        lim = np.broadcast_to(np.asarray(limit, dtype=np.float64).reshape(-1)[lo:hi] if np.ndim(limit) else limit, B)
        c = np.repeat(0.0 - lim, G)
        assert log == [
            [name, H(arm.packed), nv, H(f.packed)] + extra + [n, T("q0", (n, nv)), T("q1", (n, nv)),
                                                              T(name + ".%d" % (len(extra) + 6), (n,)), None],
            _rows_call(T((0.0,) * (B * G), (B, G, 1)), T(name + ".%d" % (len(extra) + 6), (B, G, 1)),
                       T(_flat(c), (B, G, 1)), T((1.0,), (1, 1)), T((0.0,), (1,)), 0, B, G, 1, 1, interp)]
