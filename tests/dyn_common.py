"""Helpers shared by the tests of the rigid-body layer (libtoppra_b200_dyn.so, toppra_b200.dynamics and the rigid-body
constraints): the robot fixtures, the C-ABI's error codes, comparisons, and the oracle rows of the limits they share."""
import os
import re

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ROBOTS = os.path.join(ROOT, "tests", "golden", "robots")
DYN_LIB = os.path.join(ROOT, "toppra_b200", "libtoppra_b200_dyn.so")
LOCKED = {"finger_left_joint": 0.013, "finger_right_joint": 0.021}
TB_ERR_ARG, TB_ERR_UNSUPPORTED = -1, -2
CASES = [("arm6.urdf", None), ("arm7_gripper.urdf", LOCKED), ("arm7_gripper.urdf", None)]
OFFSET = dict(xyz=(0.03, -0.02, 0.1), rpy=(0.3, -0.2, 0.5))


def urdf(name):
    return open(os.path.join(ROBOTS, name)).read()


def model_of(name, locked=None):
    from toppra_b200 import RigidBodyModel
    return RigidBodyModel.from_urdf(urdf(name), locked_joints=locked)


def close(got, ref, tol):
    """|got - ref| <= tol * max(1, max|ref|) (the scale of the state)."""
    ref = np.asarray(ref, dtype=np.float64)
    scale = max(1.0, float(np.max(np.abs(ref))))
    err = float(np.max(np.abs(np.asarray(got) - ref)))
    assert err <= tol * scale, (err, scale)
    return err / scale


def _offset_spec(off):
    from toppra_b200.dynamics import rpy_matrix
    return (rpy_matrix(off["rpy"]) if off else np.eye(3)), (np.asarray(off["xyz"]) if off else np.zeros(3))


def _dyn_header():
    text = open(os.path.join(ROOT, "include", "toppra_b200_dyn.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    out = {}
    for name, args in re.findall(r"\bint\s+(tbd_[a-z0-9_]+)\s*\(([^)]*)\)\s*;", text):
        out[name] = ["ptr" if "*" in a else ("double" if "double" in a else "int")
                     for a in (x.strip() for x in args.split(",")) if a not in ("", "void")]
    return out


def _gpu_present():
    import torch
    return torch.cuda.is_available()


def _dev(x):
    import torch
    return torch.as_tensor(np.asarray(x, dtype=np.float64), device="cuda")


def _eq(x, y):
    return np.array_equal(np.asarray(x), np.asarray(y), equal_nan=True)


def _model_from_packed(ta, packed):
    nv = (len(packed) - 3) // 27
    b = packed[3:].reshape(nv, 27)
    return ta.RigidBodyModel(b[:, 0], b[:, 1], b[:, 2:5], b[:, 5:14], b[:, 14:17], b[:, 17], b[:, 18:21], b[:, 21:27],
                             gravity=packed[:3])


def _assert_solution(got, ref_K, ref_sd, st, ref_st):
    assert st == ref_st
    if ref_st == 0:
        np.testing.assert_allclose(got[0], ref_K, rtol=1e-8, atol=1e-9)
        np.testing.assert_allclose(got[1], ref_sd, rtol=1e-8, atol=1e-9)


def _problems(B, nv, seed, velocity):
    rng = np.random.RandomState(seed)
    way = np.cumsum(rng.uniform(-0.7, 0.7, (B, 5, nv)), axis=1)
    vel = np.where(np.isfinite(velocity), velocity, 3.0)
    vlim = np.tile(np.stack([-vel, vel], axis=1), (B, 1, 1))
    al = rng.uniform(6, 10, (B, nv))
    return np.linspace(0, 1, 5), way, vlim, np.stack([-al, al], axis=-1)


def _oracle_rows(F, a, b, c, grid, interp):
    """(G, 3, R) rows a F^T, b F^T, c F^T - 0 of the constraint for the oracle."""
    from toppra_b200.constraint.linear_constraint import canlinear_colloc_to_interpolate
    g = np.zeros(F.shape[0])
    if interp:
        a, b, c, F, g = canlinear_colloc_to_interpolate(a, b, c, F, g, None, None, grid, identical=True)[:5]
    return np.stack((a.dot(F.T), b.dot(F.T), c.dot(F.T) - g), axis=1)


def _oracle_joint_rows(qs, qss, vlim, alim):
    """(G, 3, 2 nv) rows of JointAccelerationConstraint under collocation for the oracle: a = q', b = q'', c = 0,
    F = [I; -I], g = [upper; -lower]."""
    nv = qs.shape[1]
    Fj = np.vstack((np.eye(nv), -np.eye(nv)))
    g = np.concatenate((alim[:, 1], -alim[:, 0]))
    G = qs.shape[0]
    return np.stack((qs.dot(Fj.T), qss.dot(Fj.T), np.zeros((G, nv)).dot(Fj.T) - g), axis=1)


class FakePath(object):
    """The batch size, dof and device of a path: enough for RecordContext where no row is written."""

    def __init__(self, B, dof):
        self.B, self.dof, self.device = B, dof, "cpu"


class _CountingLib(object):
    """Forwards to libtoppra_b200_dyn.so and counts the calls of each entry."""

    def __init__(self, lib):
        self._lib, self.calls = lib, {}

    def __getattr__(self, name):
        fn = getattr(self._lib, name)

        def call(*args):
            self.calls[name] = self.calls.get(name, 0) + 1
            return fn(*args)
        return call


def _assert_one_terms_launch(ta, monkeypatch, cons, path, grid, entry):
    """BatchTOPPRA with the constraints `cons()` on a batch of 10 paths makes ONE `entry` launch, and one per record
    chunk in chunks of 4, 4 and 2."""
    from toppra_b200 import _lib_dyn
    assert path.B == 10
    counting = _CountingLib(_lib_dyn.load())
    monkeypatch.setattr(_lib_dyn, "_dlib", counting)
    whole = ta.BatchTOPPRA(cons(), path, grid)
    whole.compute_parameterization(0, 0)
    assert counting.calls == {entry: 1}, counting.calls
    per_path = 8 * ta.engine.record_doubles(whole.R) * whole.G
    counting.calls.clear()
    parts = ta.BatchTOPPRA(cons(), path, grid, max_record_bytes=4 * per_path)
    assert parts.chunk_size() == 4
    parts.compute_parameterization(0, 0)
    assert counting.calls == {entry: 3}, counting.calls
