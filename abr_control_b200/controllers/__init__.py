"""Batched controllers of the hot path.

The public names are those of ``abr_control.controllers`` so that a user switches packages by changing one import line
(INTEGRATION.md S1).  Which kernel of ``libabrb.so`` stands behind each name:

=================  ==========================================================================================
name               native entry point (include/abrb.h) / kernel (abr_control_b200/csrc/kernels.cu)
=================  ==========================================================================================
OSC                abrb_osc_generate_* / osc_kernel (+ osc_finish_kernel in the two-launch mode), rollout_kernel
OSC.rollout_path   abrb_osc_rollout_path_* / rollout_kernel with per-step targets (RolloutPathArgs)
Damping            secondary-controller kind 1: fused into osc_kernel, or abrb_null_generate_* / null_kernel
RestingConfig      secondary-controller kind 2 (same two routes)
AvoidObstacles     secondary-controller kind 3 (same two routes)
AvoidJointLimits   secondary-controller kind 4 (same two routes)
Joint, Floating    abrb_joint_generate_* / abrb_floating_generate_* / ctrl_kernel
Sliding            abrb_sliding_generate_* / sliding_kernel
=================  ==========================================================================================

``path_planners.InverseKinematics`` (abrb_ik_path_* / ik_kernel) lives in the sub-package of that name, as in the
reference.  Every class takes one joint state (reference contract: float64 result of shape ``(n,)``) or a batch
``(B, n)`` as NumPy host buffers or CUDA tensors.
"""
from .controller import Controller
from .osc import OSC
from ._null import NullController
from .damping import Damping
from .resting_config import RestingConfig
from .avoid_obstacles import AvoidObstacles
from .avoid_joint_limits import AvoidJointLimits
from .joint import Joint
from .floating import Floating
from .sliding import Sliding

__all__ = ["Controller", "NullController", "OSC", "Damping", "RestingConfig", "AvoidObstacles", "AvoidJointLimits",
           "Joint", "Floating", "Sliding"]
