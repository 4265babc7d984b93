"""toppra_b200 — batched TOPP-RA (time-optimal path parameterisation by reachability analysis) on NVIDIA H100.

Keeps the public names of hungpham2511/toppra (`SplineInterpolator`, `constraint.*`, `algorithm.TOPPRA`,
`ParametrizeSpline`, ...) and adds the batched entry points `BatchSplineInterpolator` / `BatchTOPPRA`.
All numbers come from hand-written sm_90a CUDA kernels behind the C-ABI in include/toppra_b200.h; there is no
CPU fallback (importing works anywhere, computing needs the GPU and the built libtoppra_b200.so)."""
import logging

from . import constants, exceptions
from .interpolator import (AbstractGeometricPath, BatchPiecewisePolyPath, BatchSplineInterpolator, PiecewisePolyPath,
                           PolynomialPath, PPolyPath, SplineInterpolator, UnivariateSplineInterpolator,
                           propose_gridpoints)
from .simplepath import SimplePath
from .parametrizer import (BatchParametrizeConstAccel, BatchParametrizeSpline, ParametrizeConstAccel,
                           ParametrizeSpline)
from . import constraint
from . import solverwrapper
from . import algorithm
from .batch import BatchResult, BatchTOPPRA, BatchTOPPRAsd, solve_batch
from .dynamics import Drives, RigidBodyFrame, RigidBodyModel
from .constraint import MotorSpeedConstraint, MotorTorqueConstraint
from .utils import setup_logging

__version__ = "0.1.0"

logging.getLogger("toppra_b200").addHandler(logging.NullHandler())

__all__ = ["AbstractGeometricPath", "BatchSplineInterpolator", "BatchPiecewisePolyPath", "PiecewisePolyPath", "PPolyPath", "PolynomialPath", "SimplePath", "SplineInterpolator", "UnivariateSplineInterpolator", "propose_gridpoints",
           "ParametrizeConstAccel", "ParametrizeSpline", "BatchParametrizeConstAccel", "BatchParametrizeSpline", "constraint", "solverwrapper", "algorithm", "BatchResult",
           "BatchTOPPRA", "BatchTOPPRAsd", "solve_batch", "RigidBodyFrame", "RigidBodyModel", "Drives",
           "MotorTorqueConstraint", "MotorSpeedConstraint", "constants", "exceptions", "setup_logging"]
