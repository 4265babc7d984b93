"""Second-order (inverse-dynamics) constraint — same surface as the reference
`toppra/constraint/linear_second_order.py:9-173`.

    A(q) qdd + qd^T B(q) qd + C(q) + custom = w,   F(q) w <= g(q)
    c = w(q,0,0);  a = w(q,0,q') - c;  b = w(q,q',q'') - c;  c += custom_term       (:142-165)

The three inverse-dynamics evaluations per gridpoint are USER code.  Two ways to supply it:
  * reference style (default): `inv_dyn(q, qd, qdd)` on 1-D numpy arrays, called 3 x (N+1) times on the host
    (what the reference does); the coefficient rows F.a, F.b, F.c - g and the interpolation lift are then
    assembled on the GPU (csrc/tb_coeff.cu: tb_rows_canlinear);
  * `batched=True`: `inv_dyn(q, qd, qdd)` on CUDA tensors of shape (M, dof) -> (M, m); three calls in total for
    the whole batch x grid, everything stays on the device (general fallback for arbitrary models);
  * `device_terms(q, qs, qss) -> (a, b, c)` on CUDA tensors (M, dof) -> (M, m), set by the constructors of the
    rigid-body limits: the batched route with the three terms of every gridpoint of the batch from ONE fused launch of
    libtoppra_b200_dyn.so.  A `toppra_b200.RigidBodyModel` as `inv_dyn` of joint_torque_constraint (and
    JointTorqueConstraint) sets `model.torque_terms` with the friction, bit-identical to three `model(...)` calls plus
    the operations above; CartesianAccelerationConstraint, ContactStabilityConstraint and SupportStabilityConstraint
    set theirs;
  * `device_model=(name, params)` (joint_torque_constraint only): the inverse dynamics is one of the models compiled
    into the library (`engine.DEVICE_MODELS`, include/toppra_b200.h TB_INVDYN_*): ONE kernel evaluates q, q', q'' and
    the three inverse-dynamics terms per gridpoint and writes the torque rows straight into the stage records
    (tb_coeff_second_order) — the path BatchTOPPRA uses for BASELINE cfg 3."""
import numpy as np

from .constraint import DiscretizationType
from .linear_constraint import LinearConstraint, canlinear_colloc_to_interpolate, check_dof
from .. import engine
from ..dynamics import RigidBodyModel


class SecondOrderConstraint(LinearConstraint):
    """See module docstring.  `constraint_F(q) -> (k, m)`, `constraint_g(q) -> (k,)`;
    `custom_term(path, s) -> (m,)` (reference style) or `custom_term(q, qd) -> (M, m)` tensors (batched).

    Row forms on the device: the eye form (F = [I; -I], g per path or shared), the constant form (one F (k, m) for
    every gridpoint, g = 0) and, reference style, the host F(q), g(q) of every gridpoint."""

    def __init__(self, inv_dyn, constraint_F, constraint_g, dof, custom_term=None, discretization_scheme=1,
                 batched=False):
        super(SecondOrderConstraint, self).__init__()
        self.set_discretization_type(discretization_scheme)
        self.inv_dyn = inv_dyn
        self.constraint_F = constraint_F
        self.constraint_g = constraint_g
        self.dof = dof
        self.custom_term = custom_term
        self.batched = batched
        self.device_model = None  # (name, params): inverse dynamics evaluated by tb_coeff_second_order
        self.device_terms = None  # (q, qs, qss) -> (a, b, c): the fused terms launch of the batched route
        self._eye_form = None  # (g [k] or [B,k], friction [m] or None): F = [I;-I] fast form
        self._const_F = None  # F (k, m) shared by every gridpoint, g = 0
        self._format_string = "    Kind: Generalized Second-order constraint\n"
        self._format_string = "    Dimension:\n"
        if not batched:
            self._format_string += "        F in R^({:d}, {:d})\n".format(*constraint_F(np.zeros(dof)).shape)

    @classmethod
    def joint_torque_constraint(cls, inv_dyn, taulim, joint_friction, **kwargs):
        """Joint torque limits taulim (dof, 2) [or batched (B, dof, 2)] with dry friction `joint_friction` (dof,)
        (reference :114-140): F = [I; -I], g = [tau_max; -tau_min], custom = sign(q') * friction."""
        taulim = np.asarray(taulim, dtype=np.float64)
        dof = np.shape(taulim)[-2]
        joint_friction = np.asarray(joint_friction, dtype=np.float64)
        stacked_eyes = np.vstack((np.eye(dof), -np.eye(dof)))
        g_aug = np.concatenate((taulim[..., 1], -taulim[..., 0]), axis=-1)
        device_model = kwargs.pop("device_model", None)
        batched = kwargs.get("batched", False) or device_model is not None or isinstance(inv_dyn, RigidBodyModel)
        kwargs["batched"] = batched
        if taulim.ndim == 3 and not batched:
            raise ValueError("batched torque limits need batched=True or a device_model")
        if device_model is not None and device_model[0] not in engine.DEVICE_MODELS:
            raise ValueError("unknown device model %r (known: %s)" % (device_model[0], sorted(engine.DEVICE_MODELS)))
        g_single = g_aug if g_aug.ndim == 1 else g_aug[0]
        constraint_F = lambda _: stacked_eyes  # noqa: E731
        constraint_g = lambda _: g_single  # noqa: E731
        if batched:
            custom_term = None
        else:
            custom_term = lambda path, s: np.sign(path(s, 1)) * joint_friction  # noqa: E731
        obj = cls(inv_dyn, constraint_F, constraint_g, dof, custom_term, **kwargs)
        obj._eye_form = (g_aug, joint_friction)
        if isinstance(inv_dyn, RigidBodyModel):
            obj.device_terms = lambda q, qs, qss: inv_dyn.torque_terms(q, qs, qss, joint_friction)
        obj._taulim = taulim
        obj.device_model = device_model
        return obj

    @property
    def interpolation(self):
        return self.discretization_type == DiscretizationType.Interpolation

    # ---- reference-style host evaluation (user callbacks) ------------------------------------------------
    def _colloc_host(self, path, gridpoints):
        """Host evaluation with the user's numpy callbacks, gridpoint by gridpoint: w(q, 0, 0), w(q, 0, q'), w(q, q', q'')
        and F(q), g(q) — what the reference does 3 (N + 1) times per path (linear_second_order.py:142-165)."""
        q, qs, qss = (np.atleast_2d(path(gridpoints, order)) for order in (0, 1, 2))
        still = np.zeros(path.dof)
        n = len(gridpoints)
        rest = [np.asarray(self.inv_dyn(q[i], still, still), dtype=np.float64) for i in range(n)]
        a = np.stack([np.asarray(self.inv_dyn(q[i], still, qs[i]), dtype=np.float64) - rest[i] for i in range(n)])
        b = np.stack([np.asarray(self.inv_dyn(q[i], qs[i], qss[i]), dtype=np.float64) - rest[i] for i in range(n)])
        c = np.stack(rest)
        if self.custom_term is not None:
            c = c + np.stack([np.asarray(self.custom_term(path, s), dtype=np.float64) for s in gridpoints])
        F = np.stack([np.asarray(self.constraint_F(qi)) for qi in q])
        g = np.stack([np.asarray(self.constraint_g(qi)) for qi in q])
        return a, b, c, F, g

    def compute_constraint_params(self, path, gridpoints):
        check_dof(self.dof, path.dof)
        if self.batched:
            raise NotImplementedError("batched SecondOrderConstraint: use BatchTOPPRA / TOPPRA, not the host 7-tuple")
        a_vec, b_vec, c_vec, F_vec, g_vec = self._colloc_host(path, np.asarray(gridpoints))
        if self.discretization_type == DiscretizationType.Collocation:
            return a_vec, b_vec, c_vec, F_vec, g_vec, None, None
        if self.discretization_type == DiscretizationType.Interpolation:
            return canlinear_colloc_to_interpolate(a_vec, b_vec, c_vec, F_vec, g_vec, None, None, gridpoints)
        raise NotImplementedError("Other form of discretization not supported!")

    # ---- device protocol ----------------------------------------------------------------------------------
    def _k(self):
        if self._eye_form is not None:
            return self._eye_form[0].shape[-1]   # F = [I; -I]: 2 dof rows for torques, 2 k for frame accelerations
        if self._const_F is not None:
            return self._const_F.shape[0]
        if self.batched:
            raise NotImplementedError("batched SecondOrderConstraint with a general F: use joint_torque_constraint")
        return self.constraint_F(np.zeros(self.dof)).shape[0]

    def _check_batch(self, ctx):
        """The checks of the device route, before its rows are counted and before they are written."""
        check_dof(self.dof, ctx.bpath.dof)

    def num_rows(self, ctx):
        self._check_batch(ctx)
        return (2 if self.interpolation else 1) * self._k()

    def _colloc_device(self, ctx):
        """(a, b, c) as CUDA tensors [B, G, m]."""
        torch = engine.torch_mod()
        bp = ctx.bpath
        B, G, dof = ctx.B, ctx.G, bp.dof
        if self.batched:
            q = bp.eval_device(ctx.d_grid, 0).reshape(B * G, dof)
            qd = bp.eval_device(ctx.d_grid, 1).reshape(B * G, dof)
            qdd = bp.eval_device(ctx.d_grid, 2).reshape(B * G, dof)
            if self.device_terms is not None:
                a, b, c = self.device_terms(q, qd, qdd)
                m = c.shape[-1]
                return a.reshape(B, G, m), b.reshape(B, G, m), c.reshape(B, G, m)
            zero = torch.zeros_like(q)
            c = self.inv_dyn(q, zero, zero)
            a = self.inv_dyn(q, zero, qd) - c
            b = self.inv_dyn(q, qd, qdd) - c
            if self._eye_form is not None and np.any(self._eye_form[1] != 0):
                c = c + torch.sign(qd) * engine.as_device(self._eye_form[1], ctx.device)
            elif self.custom_term is not None:
                c = c + self.custom_term(q, qd)
            m = c.shape[-1]
            return (a.reshape(B, G, m).contiguous(), b.reshape(B, G, m).contiguous(), c.reshape(B, G, m).contiguous())
        if ctx.path is None or ctx.grid_host is None:
            raise NotImplementedError("reference-style (numpy callback) SecondOrderConstraint needs a single path; "
                                      "pass batched=True for BatchTOPPRA")
        a, b, c, F, g = self._colloc_host(ctx.path, ctx.grid_host)
        self._host_Fg = (F, g)
        d = lambda x: engine.as_device(np.asarray(x, dtype=np.float64)[None], ctx.device)  # noqa: E731
        return d(a), d(b), d(c)

    def append_records(self, ctx, records, R_total, row0):
        self._check_batch(ctx)
        if self.device_model is not None:
            cache = self.__dict__.setdefault("_d_taulim", {})   # limits stay resident across solves and chunks
            if str(ctx.device) not in cache:
                cache[str(ctx.device)] = engine.as_device(self._taulim, ctx.device)
            tl = cache[str(ctx.device)]
            if tl.dim() == 3:
                tl = tl[ctx.lo:ctx.hi].contiguous()
            fric = self._eye_form[1]
            fric_d = engine.as_device(fric, ctx.device) if np.any(fric != 0) else None
            engine.coeff_second_order(self.device_model[0], self.device_model[1], ctx.bpath.d_ppoly, ctx.bpath.d_ss,
                                      ctx.d_grid, tl, fric_d, self.interpolation, records, R_total, row0)
            return
        a, b, c = self._colloc_device(ctx)
        if self._eye_form is not None:
            g = self._eye_form[0]
            gd = engine.as_device(g, ctx.device)
            if g.ndim == 2:
                gd = gd[ctx.lo:ctx.hi].contiguous()
            mode = 2 if g.ndim == 1 else 3
            engine.rows_canlinear(a, b, c, None, gd, mode, ctx.d_grid, self.interpolation, records, R_total, row0)
        elif self._const_F is not None:
            Fd = engine.as_device(self._const_F, ctx.device)
            gd = engine.as_device(np.zeros(self._const_F.shape[0]), ctx.device)
            engine.rows_canlinear(a, b, c, Fd, gd, 0, ctx.d_grid, self.interpolation, records, R_total, row0)
        else:
            F, g = self._host_Fg
            Fd = engine.as_device(np.asarray(F, dtype=np.float64)[None], ctx.device)
            gd = engine.as_device(np.asarray(g, dtype=np.float64)[None], ctx.device)
            engine.rows_canlinear(a, b, c, Fd, gd, 1, ctx.d_grid, self.interpolation, records, R_total, row0)
