"""Constraints — same names as the reference `toppra/constraint/__init__.py`."""
from .constraint import ConstraintType, DiscretizationType, Constraint
from .linear_constraint import LinearConstraint, canlinear_colloc_to_interpolate, RecordContext
from .linear_joint_acceleration import JointAccelerationConstraint
from .linear_joint_velocity import JointVelocityConstraint, JointVelocityConstraintVarying
from .linear_second_order import SecondOrderConstraint
from .joint_torque import JointTorqueConstraint
from .cartesian_velocity_norm import CartesianVelocityNorm
from .cartesian_acceleration import CartesianAccelerationConstraint
from .contact_stability import ContactStabilityConstraint, contact_wrench_cone
from .collision_energy import CollisionEnergyConstraint
from .support_stability import SupportStabilityConstraint, support_polygon_rows
from .separation_monitoring import SeparationMonitoringConstraint
from .motor_limits import MotorSpeedConstraint, MotorTorqueConstraint
from .joint_wrench import JointWrenchConstraint
from .kinetic_energy import KineticEnergyConstraint, MomentumConstraint
from ..dynamics import Drives
from .conic_constraint import ConicConstraint, RobustLinearConstraint

__all__ = ["ConstraintType", "DiscretizationType", "Constraint", "LinearConstraint",
           "canlinear_colloc_to_interpolate", "JointAccelerationConstraint", "JointVelocityConstraint", "JointVelocityConstraintVarying",
           "SecondOrderConstraint", "JointTorqueConstraint", "CartesianVelocityNorm", "CartesianAccelerationConstraint",
           "ContactStabilityConstraint", "contact_wrench_cone", "CollisionEnergyConstraint",
           "SupportStabilityConstraint", "support_polygon_rows", "SeparationMonitoringConstraint", "RecordContext",
           "Drives", "MotorTorqueConstraint", "MotorSpeedConstraint", "JointWrenchConstraint",
           "KineticEnergyConstraint", "MomentumConstraint",
           "ConicConstraint", "RobustLinearConstraint"]
