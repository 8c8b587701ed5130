"""Loader for libabrb.so (the sm_90a CUDA library behind include/abrb.h).

There is deliberately no fallback: if the shared library is missing, or no CUDA device is visible when a
compute entry point is called, the call raises.
"""
import ctypes as C
import os
import threading

from . import _abi

_HERE = os.path.dirname(os.path.abspath(__file__))
# ABRB_LIBRARY: another build of the same library (e.g. of another commit, for an A/B run of bench.py); default is the
# in-tree build
LIB_PATH = os.environ.get("ABRB_LIBRARY") or os.path.join(_HERE, "libabrb.so")

_lock = threading.Lock()
_lib = None


class AbrbError(RuntimeError):
    def __init__(self, code, message):
        super().__init__(f"libabrb error {code}: {message}")
        self.code = code


# every symbol include/abrb.h declares: name -> (restype, argtypes)
_VP, _I, _I64, _D, _CP = C.c_void_p, C.c_int, C.c_int64, C.c_double, C.c_char_p
_gen = [_VP, _I, _VP, _VP, _VP, _VP, _I, _VP, _I, _VP, _VP, _VP, _I64]  # ... u, training_signal, integrated_error, B
_roll = [_VP, _I, _VP, _VP, _VP, _VP, _I, _I, _D, _VP, _VP, _VP, _VP, _I64, _VP]
# c, frame_id, x_off, q, dq, path, path_stride, path_velocity, pv_stride, steps, dt, effort_weight,
# q_traj, dq_traj, u_traj, x_traj, cost, integrated_error, B, stream
_roll_path = [_VP, _I, _VP, _VP, _VP, _VP, _I, _VP, _I, _I, _D, _D, _VP, _VP, _VP, _VP, _VP, _VP, _I64, _VP]
_dyn = [_VP, _VP, _VP, _VP, _VP, _I64, _VP]  # m, q, dq, u | ddq, ddq | u (| Yt), B, stream
# m, frame_id, x_off, q, dq, u, u_stride, compensate_gravity, path, path_stride, steps, dt, effort_weight,
# q_traj, dq_traj, u_traj, x_traj, cost, B, stream
_plant = [_VP, _I, _VP, _VP, _VP, _VP, _I, _I, _VP, _I, _I, _D, _D, _VP, _VP, _VP, _VP, _VP, _I64, _VP]
# m, q, dq, u | ddq, d_q, d_dq, d_u | d_ddq, B, stream
_djac = [_VP, _VP, _VP, _VP, _VP, _VP, _VP, _I64, _VP]
# m, frame_id, x_off, q0, dq0, u, u_stride, compensate_gravity, path, path_stride, steps, dt, effort_weight,
# q_traj, dq_traj, g_cost, g_q, g_dq, g_q_traj, g_dq_traj, g_u_traj, g_x_traj, gu, gq0, gdq0, B, stream
_vjp = [_VP, _I, _VP, _VP, _VP, _VP, _I, _I, _VP, _I, _I, _D, _D] + [_VP] * 12 + [_I64, _VP]
# m, kp, kv, account_for_gravity, frame_id, x_off, q, dq, path, path_stride, path_velocity, pv_stride, steps, dt,
# effort_weight, q_traj, dq_traj, u_traj, x_traj, cost, B, stream
_joint_roll = [_VP, _D, _D, _I, _I, _VP, _VP, _VP, _VP, _I, _VP, _I, _I, _D, _D, _VP, _VP, _VP, _VP, _VP, _I64, _VP]
# m, kd, lamb, cartesian, frame_id, x_off, q, dq, path, path_stride, path_velocity, pv_stride, path_acc, pa_stride,
# steps, dt, effort_weight, q_traj, dq_traj, u_traj, x_traj, cost, B, stream
_sliding_roll = _joint_roll[:12] + [_VP, _I] + _joint_roll[12:]
# m, kp, kv, account_for_gravity, frame_id, x_off, q0, dq0, path, path_stride, path_velocity, pv_stride, steps, dt,
# effort_weight, q_traj, dq_traj, g_cost, g_q, g_dq, g_q_traj, g_dq_traj, g_u_traj, g_x_traj, g_path,
# g_path_velocity, g_gains, gq0, gdq0, B, stream
_joint_vjp = _joint_roll[:15] + [_VP] * 14 + [_I64, _VP]
# m, q0, dq0, u, u_stride, compensate_gravity, steps, effort_weight, q_traj, dq_traj, gu, g_cost, g_u_traj, g_theta,
# B, stream
_theta_vjp = [_VP, _VP, _VP, _VP, _I, _I, _I, _D] + [_VP] * 6 + [_I64, _VP]
SIGNATURES = {
    "abrb_version": (_I, []),
    "abrb_last_error": (_CP, []),
    "abrb_device_count": (_I, []),
    "abrb_model_create": (_I, [C.POINTER(_abi.ChainDesc), C.POINTER(_VP)]),
    "abrb_model_destroy": (_I, [_VP]),
    "abrb_model_n_joints": (_I, [_VP]),
    "abrb_model_is_orthonormal": (_I, [_VP]),
    "abrb_frame_id": (_I, [_VP, _CP]),
    "abrb_rbd_eval_f64": (_I, [_VP, _I, _VP, _VP, _VP, _I64, C.POINTER(_abi.RbdOut), _VP]),
    "abrb_rbd_eval_f32": (_I, [_VP, _I, _VP, _VP, _VP, _I64, C.POINTER(_abi.RbdOut), _VP]),
    "abrb_rbd_eval_host_f64": (_I, [_VP, _I, _VP, _VP, _VP, _I64, C.POINTER(_abi.RbdOut)]),
    "abrb_rbd_eval_host_f32": (_I, [_VP, _I, _VP, _VP, _VP, _I64, C.POINTER(_abi.RbdOut)]),
    "abrb_osc_create": (_I, [_VP, C.POINTER(_abi.OscParams), C.POINTER(_VP)]),
    "abrb_osc_destroy": (_I, [_VP]),
    "abrb_osc_set_option": (_I, [_VP, C.c_char_p, C.c_double]),
    "abrb_osc_generate_f64": (_I, _gen + [_VP]),
    "abrb_osc_generate_f32": (_I, _gen + [_VP]),
    "abrb_osc_generate_host_f64": (_I, _gen),
    "abrb_osc_generate_host_f32": (_I, _gen),
    "abrb_osc_generate_host_async_f64": (_I, _gen + [_I]),
    "abrb_osc_generate_host_async_f32": (_I, _gen + [_I]),
    "abrb_osc_host_wait": (_I, [_VP, _I]),
    "abrb_gather_create": (_I, [_I, _I, _I64, _I, C.POINTER(_VP)]),
    "abrb_gather_destroy": (_I, [_VP]),
    "abrb_gather_export": (_I, [_VP, C.c_char_p]),
    "abrb_gather_import": (_I, [_VP, _I, C.c_char_p]),
    "abrb_gather_buffer": (_VP, [_VP, _I]),
    "abrb_gather_wait": (_I, [_VP, _VP]),
    "abrb_gather_status": (_I, [_VP]),
    "abrb_osc_generate_gather_f64": (_I, _gen + [_VP, _I, _I64, _VP]),
    "abrb_osc_generate_gather_f32": (_I, _gen + [_VP, _I, _I64, _VP]),
    "abrb_null_generate_f64": (_I, [_VP, C.POINTER(_abi.NullParams), _VP, _VP, _VP, _I64, _VP]),
    "abrb_null_generate_f32": (_I, [_VP, C.POINTER(_abi.NullParams), _VP, _VP, _VP, _I64, _VP]),
    "abrb_joint_generate_f64": (_I, [_VP, _D, _D, _I, _VP, _VP, _VP, _I, _VP, _I, _VP, _I64, _VP]),
    "abrb_joint_generate_f32": (_I, [_VP, _D, _D, _I, _VP, _VP, _VP, _I, _VP, _I, _VP, _I64, _VP]),
    "abrb_floating_generate_f64": (_I, [_VP, _I, _I, _VP, _VP, _VP, _I64, _VP]),
    "abrb_floating_generate_f32": (_I, [_VP, _I, _I, _VP, _VP, _VP, _I64, _VP]),
    "abrb_sliding_generate_f64": (_I, [_VP, _D, _D, _I, _I, _VP, _VP, _VP, _VP, _I, _VP, _I, _VP, _I, _VP, _VP, _I64, _VP]),
    "abrb_sliding_generate_f32": (_I, [_VP, _D, _D, _I, _I, _VP, _VP, _VP, _VP, _I, _VP, _I, _VP, _I, _VP, _VP, _I64, _VP]),
    "abrb_ik_path_f64": (_I, [_VP, _D, _D, _D, _I, _D, _I, _VP, _VP, _I, _VP, _VP, _I64, _VP]),
    "abrb_ik_path_f32": (_I, [_VP, _D, _D, _D, _I, _D, _I, _VP, _VP, _I, _VP, _VP, _I64, _VP]),
    "abrb_osc_rollout_f64": (_I, _roll),
    "abrb_osc_rollout_f32": (_I, _roll),
    "abrb_osc_rollout_path_f64": (_I, _roll_path),
    "abrb_osc_rollout_path_f32": (_I, _roll_path),
    "abrb_forward_dynamics_f64": (_I, _dyn),
    "abrb_forward_dynamics_f32": (_I, _dyn),
    "abrb_inverse_dynamics_f64": (_I, _dyn),
    "abrb_inverse_dynamics_f32": (_I, _dyn),
    "abrb_inverse_dynamics_regressor_f64": (_I, _dyn),
    "abrb_inverse_dynamics_regressor_f32": (_I, _dyn),
    "abrb_plant_rollout_f64": (_I, _plant),
    "abrb_plant_rollout_f32": (_I, _plant),
    "abrb_forward_dynamics_derivatives_f64": (_I, _djac),
    "abrb_forward_dynamics_derivatives_f32": (_I, _djac),
    "abrb_inverse_dynamics_derivatives_f64": (_I, _djac),
    "abrb_inverse_dynamics_derivatives_f32": (_I, _djac),
    "abrb_plant_rollout_vjp_f64": (_I, _vjp),
    "abrb_plant_rollout_vjp_f32": (_I, _vjp),
    "abrb_plant_rollout_theta_vjp_f64": (_I, _theta_vjp),
    "abrb_plant_rollout_theta_vjp_f32": (_I, _theta_vjp),
    "abrb_joint_rollout_path_f64": (_I, _joint_roll),
    "abrb_joint_rollout_path_f32": (_I, _joint_roll),
    "abrb_joint_rollout_path_vjp_f64": (_I, _joint_vjp),
    "abrb_joint_rollout_path_vjp_f32": (_I, _joint_vjp),
    "abrb_sliding_rollout_path_f64": (_I, _sliding_roll),
    "abrb_sliding_rollout_path_f32": (_I, _sliding_roll),
    "abrb_path_plan": (_I, [C.POINTER(_abi.PathParams)] + [_VP] * 8 + [_I64, _VP]),
    "abrb_path_fill_f64": (_I, [C.POINTER(_abi.PathParams)] + [_VP] * 9 + [_I64, _VP, _I64, _VP]),
    "abrb_path_fill_f32": (_I, [C.POINTER(_abi.PathParams)] + [_VP] * 9 + [_I64, _VP, _I64, _VP]),
    "abrb_launch_count": (_I64, []),
}


def lib():
    """The loaded library (loads on first use; raises if it has not been built)."""
    global _lib
    with _lock:
        if _lib is None:
            if not os.path.exists(LIB_PATH):
                raise ImportError(
                    f"{LIB_PATH} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                    "or `make -C abr_control_b200/csrc -j8` (there is no CPU fallback)"
                )
            handle = C.CDLL(LIB_PATH)
            for name, (res, args) in SIGNATURES.items():
                fn = getattr(handle, name)  # AttributeError if the symbol is missing
                fn.restype, fn.argtypes = res, args
            _lib = handle
    return _lib


def check(rc):
    if rc < 0:
        raise AbrbError(rc, lib().abrb_last_error().decode())
    return rc
