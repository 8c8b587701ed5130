"""``torch.autograd`` for the Joint closed loop: ``Joint.rollout_path``.

Used only when grad mode is on and ``q``, ``dq``, the path, the path velocity or a 0-d gain tensor requires grad;
every other call takes the value-only path.  The forward pass is ``abrb_joint_rollout_path_*`` as it is (it also
records ``q`` and ``dq``, which the backward pass reads); the backward pass is ``abrb_joint_rollout_path_vjp_*``, the
adjoint recursion of the closed loop over the recorded states (DESIGN.md S3.6).  The Function is once-differentiable:
a gradient of a gradient raises.
"""
import ctypes as C

import numpy as np
import torch
from torch.autograd.function import once_differentiable

from .. import _lib
from ..arms._autograd import _like, _ptr, _stream
from . import _batch


def _check_grad_inputs(named):
    for what, x in named:
        if _batch.is_torch(x) and x.requires_grad:
            if not x.is_cuda or x.dtype not in (torch.float32, torch.float64):
                raise ValueError(f"differentiable inputs must be float32 or float64 CUDA tensors ({what})")


def _gain(x, ref, what):
    """a gain as a 0-d tensor on ``ref``'s device (its own dtype for a tensor: its gradient keeps it)"""
    if _batch.is_torch(x):
        if x.dim() != 0:
            raise ValueError(f"{what} must be a scalar (a 0-d CUDA tensor to differentiate with respect to it)")
        if not x.is_cuda:
            raise ValueError(f"{what}: torch inputs must be CUDA tensors (use NumPy for host data)")
        return x
    return torch.tensor(float(x), dtype=torch.float64, device=ref.device)


def _offset(xyz_offset):
    if xyz_offset is not None and not np.allclose(np.asarray(xyz_offset, dtype=float), 0):
        return (C.c_double * 3)(*[float(v) for v in np.asarray(xyz_offset, dtype=float).reshape(3)])
    return None


class _JointRollout(torch.autograd.Function):
    @staticmethod
    def forward(ctx, ctrl, opts, q0, dq0, path, pv, kp, kv):
        ctx.set_materialize_grads(False)
        rc = ctrl.robot_config
        rec = opts["record"]
        inner = tuple(k for k in ("q", "dq", "u", "x") if k in rec or k in ("q", "dq"))
        gains = (float(kp), float(kv), int(bool(ctrl.account_for_gravity)))
        qf, dqf, traj, cost = _batch.ctrl_rollout(
            rc, ("abrb_joint_rollout_path_f64", "abrb_joint_rollout_path_f32"), gains, q0, dq0,
            [(path, "path"), (pv, "path_velocity")], rc.N_JOINTS, opts["dt"], opts["ref_frame"], opts["xyz_offset"],
            inner, opts["effort_weight"], "rollout_path")
        ctx.rc, ctx.opts, ctx.gains = rc, opts, gains
        ctx.save_for_backward(q0, dq0, path, pv, kp, kv, traj["q"], traj["dq"])
        return (qf, dqf, cost) + tuple(traj[k] for k in rec)

    @staticmethod
    @once_differentiable
    def backward(ctx, g_qf, g_dqf, g_cost, *g_rec):
        q0, dq0, path, pv, kp, kv, q_traj, dq_traj = ctx.saved_tensors
        rc, opts = ctx.rc, ctx.opts
        B, n = q0.shape
        S = path.shape[0]
        need = ctx.needs_input_grad
        g = dict(zip(opts["record"], g_rec))
        cot = [None if t is None else t.contiguous() for t in (g_cost, g_qf, g_dqf, g.get("q"), g.get("dq"),
                                                                 g.get("u"), g.get("x"))]
        rows = lambda: torch.empty((S, B, n), dtype=q0.dtype, device=q0.device)  # noqa: E731
        g_path = rows() if need[4] else None
        g_pv = rows() if need[5] else None
        g_gains = torch.empty((B, 2), dtype=q0.dtype, device=q0.device) if need[6] or need[7] else None
        gq0, gdq0 = torch.empty_like(q0), torch.empty_like(dq0)
        L = _lib.lib()
        fn = L.abrb_joint_rollout_path_vjp_f32 if q0.dtype == torch.float32 else L.abrb_joint_rollout_path_vjp_f64
        kpf, kvf, grav = ctx.gains
        with torch.cuda.device(q0.device):
            _lib.check(fn(rc.handle, kpf, kvf, grav, rc.frame_id(opts["ref_frame"]), _offset(opts["xyz_offset"]),
                          q0.data_ptr(), dq0.data_ptr(), path.data_ptr(), 0 if path.dim() == 2 else n, _ptr(pv),
                          0 if pv is None or pv.dim() == 2 else n, int(S), float(opts["dt"]),
                          float(opts["effort_weight"]), _ptr(q_traj), _ptr(dq_traj), *[_ptr(t) for t in cot],
                          _ptr(g_path), _ptr(g_pv), _ptr(g_gains), gq0.data_ptr(), gdq0.data_ptr(), B, _stream(q0)))
        if g_path is not None and path.dim() == 2:
            g_path = g_path.sum(1)
        if g_pv is not None and pv.dim() == 2:
            g_pv = g_pv.sum(1)
        g_kp = g_kv = None
        if g_gains is not None:
            tot = g_gains.sum(0)
            g_kp = tot[0].to(kp.dtype) if need[6] else None
            g_kv = tot[1].to(kv.dtype) if need[7] else None
        return None, None, gq0, gdq0, g_path, g_pv, g_kp, g_kv


def joint_rollout_path(ctrl, q, dq, path, dt, path_velocity, ref_frame, xyz_offset, record, effort_weight):
    rc = ctrl.robot_config
    n = rc.N_JOINTS
    _check_grad_inputs((("q", q), ("dq", dq), ("path", path), ("path_velocity", path_velocity), ("kp", ctrl.kp),
                        ("kv", ctrl.kv)))
    cuda = [x for x in (q, dq, path, path_velocity, ctrl.kp, ctrl.kv) if _batch.is_torch(x) and x.requires_grad]
    dtype = q.dtype if _batch.is_torch(q) else (dq.dtype if _batch.is_torch(dq) else cuda[0].dtype)
    if dtype not in (torch.float32, torch.float64):
        raise ValueError("differentiable inputs must be float32 or float64 CUDA tensors (q)")
    ref = torch.empty((), dtype=dtype, device=cuda[0].device)
    qa, dqa = _like(q, ref, "q"), _like(dq, ref, "dq")
    if tuple(qa.shape) != tuple(dqa.shape) or qa.dim() not in (1, 2) or qa.shape[-1] != n:
        raise ValueError("q and dq must have the same type, dtype and shape")
    single = qa.dim() == 1
    qa, dqa = qa.reshape(-1, n).contiguous(), dqa.reshape(-1, n).contiguous()
    pa = _like(path, ref, "path").contiguous()
    va = None if path_velocity is None else _like(path_velocity, ref, "path_velocity").contiguous()
    kp, kv = _gain(ctrl.kp, ref, "kp"), _gain(ctrl.kv, ref, "kv")
    for k in record:
        if k not in ("q", "dq", "u", "x"):
            raise ValueError(f"rollout_path can record 'q', 'dq', 'u' and 'x', not {k!r}")
    opts = dict(dt=dt, effort_weight=effort_weight, ref_frame=ref_frame, xyz_offset=xyz_offset, record=tuple(record))
    out = _JointRollout.apply(ctrl, opts, qa, dqa, pa, va, kp, kv)
    qf, dqf, cost = out[:3]
    traj = dict(zip(opts["record"], out[3:]))
    if single:
        return qf[0], dqf[0], {k: v[:, 0] for k, v in traj.items()}, cost[0]
    return qf, dqf, traj, cost
