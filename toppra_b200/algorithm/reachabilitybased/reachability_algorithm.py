"""Reachability-analysis based parameterisation — same surface as the reference
`toppra/algorithm/reachabilitybased/reachability_algorithm.py:14-431`, executed by the GPU kernels
(csrc/tb_scan.cu) through `toppra_b200.solverwrapper.B200SolverWrapper`."""
import logging

import numpy as np

from ..algorithm import ParameterizationAlgorithm, ParameterizationReturnCode, STATUS_CODES
from ...constraint import ConstraintType
from ... import exceptions
from ...solverwrapper import B200SolverWrapper, available_solvers

logger = logging.getLogger(__name__)


class ReachabilityAlgorithm(ParameterizationAlgorithm):
    """Base class for Reachability Analysis-based path parameterization algorithms.

    Parameters are those of the reference class; `solver_wrapper` may be None, "seidel" (the reference
    solver whose semantics the kernels reproduce bit-for-bit) or "b200" (same thing).  The other reference
    wrappers (qpoases, hotqpoases, ecos, cvxpy) are third-party back-ends that are out of scope here."""

    def __init__(self, constraint_list, path, gridpoints=None, solver_wrapper=None, parametrizer=None, **kwargs):
        super(ReachabilityAlgorithm, self).__init__(constraint_list, path, gridpoints=gridpoints,
                                                    parametrizer=parametrizer, **kwargs)
        has_conic = any(c.get_constraint_type() == ConstraintType.CanonicalConic for c in constraint_list)
        solver_wrapper_given = solver_wrapper
        if solver_wrapper is None:
            logger.info("Solver wrapper not supplied. Choose solver wrapper automatically!")
            solver_wrapper = "seidel"
        name = solver_wrapper.lower()
        valid = [s for s, avail in available_solvers(output_msg=False) if avail]
        if has_conic:
            # reference :78-84: conic problems need a conic solver ("ecos"/"cvxpy").  Those names (and "b200") map
            # to the GPU conic scan (csrc/tb_robust.cu); "seidel" keeps the reference's assertion.
            if solver_wrapper_given is None:
                name = "b200"
            assert name in ["cvxpy", "ecos", "b200"], \
                "Problem has conic constraints, solver {:} is not suitable".format(solver_wrapper)
        else:
            assert name in ["cvxpy", "qpoases", "ecos", "hotqpoases", "seidel", "b200"], \
                "Solver {:} not found".format(solver_wrapper)
            if name not in valid:
                raise NotImplementedError("Solver wrapper {:} not found!".format(solver_wrapper))
        self.solver_wrapper = B200SolverWrapper(self.constraints, self.path, self.gridpoints)

    def compute_feasible_sets(self):
        """Sets of feasible squared velocities X (N+1, 2) (reference :131-164)."""
        X = self.solver_wrapper.feasible_sets()
        self._problem_data.X = X
        return X

    def compute_controllable_sets(self, sdmin, sdmax):
        """Sets of controllable squared path velocities K (N+1, 2) (reference :166-202)."""
        assert sdmin <= sdmax and 0 <= sdmin
        K, status = self.solver_wrapper.controllable_sets(sdmin, sdmax)
        if status != 0:
            logger.warning("A numerical error occurs: The controllable set can't be computed.")
        return K

    def compute_reachable_sets(self, sdmin, sdmax):
        """Sets of reachable squared velocities L (N+1, 2) (reference :378-431): the feasible-set pass and the forward
        recursion run as ONE launch of tb_reachable_sets (csrc/tb_scan.cu) — the B = 1 case of
        `BatchTOPPRA.compute_reachable_sets`; robust problems run a feasible-set launch and one launch of
        tbr_reachable_sets_robust (csrc/tb_reach.cu).  Rows after a failed stage stay 0 like the reference's."""
        assert sdmin <= sdmax and 0 <= sdmin
        X, L, fail_stage = self.solver_wrapper.reachable_sets(sdmin, sdmax)
        self._problem_data.X = X
        if fail_stage >= 0:
            logger.warning("L[{:d}]={:}. Path not parametrizable.".format(fail_stage, L[fail_stage]))
        return L

    def compute_parameterization(self, sd_start, sd_end, return_data=False):
        """Compute a path parameterization (reference :240-376).

        Returns (sdd_vec (N,), sd_vec (N+1,), v_vec (N, 0)[, K (N+1, 2)]); (None, None, None[, K]) when the
        instance is not controllable; arrays contain NaN if the forward pass failed."""
        if sd_end < 0 or sd_start < 0:
            raise exceptions.BadInputVelocities(
                "Negative path velocities: path velocities must be positive: (%s, %s)" % (sd_start, sd_end))
        res = self.solver_wrapper.parameterize(sd_start, sd_end)
        K, status = res["K"], res["status"]
        code = STATUS_CODES[status]
        if code == ParameterizationReturnCode.FailUncontrollable:
            if np.isnan(K).any():
                logger.warning("An error occurred when computing controllable velocities. "
                               "The path is not controllable, or is badly conditioned.")
            else:
                self._problem_data.K = K
                logger.warning("The initial velocity is not controllable. {:f} not in ({:f}, {:f})".format(
                    sd_start ** 2, K[0, 0], K[0, 1]))
            self._problem_data.return_code = ParameterizationReturnCode.FailUncontrollable
            if return_data:
                return None, None, None, K
            return None, None, None
        self._problem_data.K = K
        sd_vec, sdd_vec = res["sd"], res["u"]
        v_vec = np.zeros((self._N, self.solver_wrapper.get_no_vars() - 2))
        self._problem_data.sd_vec = sd_vec
        self._problem_data.sdd_vec = sdd_vec
        if np.isnan(sd_vec).any():
            self._problem_data.return_code = ParameterizationReturnCode.ErrUnknown
        else:
            self._problem_data.return_code = ParameterizationReturnCode.Ok
        if return_data:
            return sdd_vec, sd_vec, v_vec, K
        return sdd_vec, sd_vec, v_vec
