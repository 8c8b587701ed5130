"""Path planners on the batched hot path — same names as ``abr_control.controllers.path_planners``."""
from . import position_profiles, velocity_profiles
from .inverse_kinematics import InverseKinematics
from .path_planner import PathPlanner

__all__ = ["InverseKinematics", "PathPlanner", "position_profiles", "velocity_profiles"]
