"""``torch.autograd`` for the plant: ``forward_dynamics``, ``inverse_dynamics`` and ``simulate`` of ``BaseConfig``.

Used only when grad mode is on and a CUDA tensor input requires grad; every other call takes the value-only path.
The backward passes are the library's derivative entry points (include/abrb.h):

* dynamics: ``J^T g`` with the ``(B, n, n)`` derivatives of ``abrb_{forward,inverse}_dynamics_derivatives_*``; the
  link inertias ``theta`` through the regressor ``Y`` (``inverse_dynamics_regressor``): ``sum_b Y_b^T g_b`` for the
  inverse dynamics, ``-sum_b Y_b^T M_b^-1 g_b`` (``Y`` at the computed ``ddq``) for the forward dynamics;
* ``simulate``: ``abrb_plant_rollout_vjp_*``, the adjoint recursion over the recorded states (DESIGN.md S3.6), then
  ``abrb_plant_rollout_theta_vjp_*`` for ``theta`` (DESIGN.md S3.8).

The Functions are once-differentiable: a gradient of a gradient raises.
"""
import ctypes as C

import numpy as np
import torch
from torch.autograd.function import once_differentiable

from .. import _lib


def _like(x, ref, what):
    """``x`` as a tensor on ``ref``'s device and dtype (differentiable for tensors)."""
    if isinstance(x, torch.Tensor):
        if not x.is_cuda:
            raise ValueError(f"{what}: torch inputs must be CUDA tensors (use NumPy for host data)")
        return x.to(device=ref.device, dtype=ref.dtype)
    return torch.as_tensor(np.asarray(x, dtype=np.float64), device=ref.device).to(ref.dtype)


def _ref_tensor(*xs):
    for x in xs:
        if isinstance(x, torch.Tensor) and x.requires_grad:
            if not x.is_cuda or x.dtype not in (torch.float32, torch.float64):
                raise ValueError("differentiable inputs must be float32 or float64 CUDA tensors")
            return x
    raise AssertionError("no input requires grad")


def _stream(t):
    return torch.cuda.current_stream(t.device).cuda_stream


def _ptr(t):
    return None if t is None else t.data_ptr()


class _Dynamics(torch.autograd.Function):
    @staticmethod
    def forward(ctx, rc, kind, q, dq, x, theta):
        ctx.rc, ctx.kind = rc, kind
        out = (rc.forward_dynamics if kind == 0 else rc.inverse_dynamics)(q, dq, x)
        ctx.save_for_backward(q, dq, x, out if theta is not None else None, theta)
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        q, dq, x, out, theta = ctx.saved_tensors
        g = g.contiguous()
        gq = gdq = gx = gth = None
        if any(ctx.needs_input_grad[2:5]):
            d_q, d_dq, d_x = ctx.rc._derivatives(q, dq, x, ctx.kind, want_in=ctx.needs_input_grad[4])

            def vjp(d, need):
                return torch.bmm(g[:, None, :], d)[:, 0] if need else None

            gq, gdq, gx = (vjp(d, ctx.needs_input_grad[i]) for d, i in ((d_q, 2), (d_dq, 3), (d_x, 4)))
        if ctx.needs_input_grad[5]:
            if ctx.kind == 1:  # u = Y(q, dq, ddq) theta
                w, Y = g, ctx.rc.inverse_dynamics_regressor(q, dq, x)
            else:  # at fixed u, d ddq / d theta = -M^-1 Y(q, dq, ddq)
                L = torch.linalg.cholesky(ctx.rc.eval(q, want=("M",))["M"])
                w, Y = -torch.cholesky_solve(g[:, :, None], L)[:, :, 0], ctx.rc.inverse_dynamics_regressor(q, dq, out)
            gth = torch.sum(torch.bmm(w[:, None, :], Y)[:, 0], 0).to(theta.dtype)
        return None, None, gq, gdq, gx, gth


def dynamics(rc, kind, q, dq, x, theta=None):
    n = rc.N_JOINTS
    ref = _ref_tensor(q, dq, x, theta)
    dtype = q.dtype if isinstance(q, torch.Tensor) else ref.dtype
    ref = torch.empty((), dtype=dtype, device=ref.device)
    qa, dqa, xa = (_like(a, ref, w) for a, w in ((q, "q"), (dq, "dq"), (x, "u" if kind == 0 else "ddq")))
    single = qa.dim() == 1
    for a, w in ((qa, "q"), (dqa, "dq"), (xa, "u" if kind == 0 else "ddq")):
        if tuple(a.shape) != tuple(qa.shape) or a.shape[-1] != n or a.dim() not in (1, 2):
            raise ValueError(f"{w} must have the shape of q, ({n},) or (B, {n}), got {tuple(a.shape)}")
    qa, dqa, xa = (a.reshape(-1, n).contiguous() for a in (qa, dqa, xa))
    out = _Dynamics.apply(rc, kind, qa, dqa, xa, _grad_theta(theta, ref))
    return out[0] if single else out


def _grad_theta(theta, ref):
    """``theta`` when it takes part in the graph (a tensor that requires grad, on the inputs' device), else None"""
    if not (isinstance(theta, torch.Tensor) and theta.requires_grad):
        return None
    if theta.device != ref.device:
        raise ValueError(f"theta is on {theta.device}, the other inputs on {ref.device}")
    return theta


class _Simulate(torch.autograd.Function):
    @staticmethod
    def forward(ctx, rc, opts, q0, dq0, u, path, theta):
        ctx.set_materialize_grads(False)
        rec = opts["record"]
        inner = tuple(k for k in ("q", "dq", "u", "x") if k in rec or k in ("q", "dq"))
        qf, dqf, traj, cost = rc.simulate(q0, dq0, u, dt=opts["dt"], path=path, effort_weight=opts["effort_weight"],
                                          compensate_gravity=opts["compensate_gravity"], ref_frame=opts["ref_frame"],
                                          xyz_offset=opts["xyz_offset"], record=inner)
        ctx.rc, ctx.opts = rc, opts
        ctx.save_for_backward(q0, dq0, u, path, traj["q"], traj["dq"], theta)
        return (qf, dqf, cost) + tuple(traj[k] for k in rec)

    @staticmethod
    @once_differentiable
    def backward(ctx, g_qf, g_dqf, g_cost, *g_rec):
        q0, dq0, u, path, q_traj, dq_traj, theta = ctx.saved_tensors
        rc, opts = ctx.rc, ctx.opts
        B, n = q0.shape
        S = u.shape[0]
        g = dict(zip(opts["record"], g_rec))
        cot = [None if t is None else t.contiguous() for t in (g_cost, g_qf, g_dqf, g.get("q"), g.get("dq"),
                                                                 g.get("u"), g.get("x"))]
        gu = torch.empty((S, B, n), dtype=q0.dtype, device=q0.device)
        gq0, gdq0 = torch.empty_like(q0), torch.empty_like(dq0)
        xo = opts["xyz_offset"]
        if xo is not None and not np.allclose(np.asarray(xo, dtype=float), 0):
            xo = (C.c_double * 3)(*[float(v) for v in np.asarray(xo, dtype=float).reshape(3)])
        else:
            xo = None
        L = _lib.lib()
        fn = L.abrb_plant_rollout_vjp_f32 if q0.dtype == torch.float32 else L.abrb_plant_rollout_vjp_f64
        with torch.cuda.device(q0.device):
            _lib.check(fn(rc.handle, rc.frame_id(opts["ref_frame"]), xo, q0.data_ptr(), dq0.data_ptr(), _ptr(u),
                          0 if u.dim() == 2 else n, 1 if opts["compensate_gravity"] else 0, _ptr(path),
                          0 if path is None or path.dim() == 2 else 6, int(S), float(opts["dt"]),
                          float(opts["effort_weight"]), _ptr(q_traj), _ptr(dq_traj), *[_ptr(t) for t in cot],
                          gu.data_ptr(), gq0.data_ptr(), gdq0.data_ptr(), B, _stream(q0)))
        gth = None
        if ctx.needs_input_grad[6]:
            gth = torch.empty((B, 6 * n), dtype=q0.dtype, device=q0.device)
            fn = L.abrb_plant_rollout_theta_vjp_f32 if q0.dtype == torch.float32 else L.abrb_plant_rollout_theta_vjp_f64
            with torch.cuda.device(q0.device):
                _lib.check(fn(rc.handle, q0.data_ptr(), dq0.data_ptr(), _ptr(u), 0 if u.dim() == 2 else n,
                              1 if opts["compensate_gravity"] else 0, int(S), float(opts["effort_weight"]),
                              _ptr(q_traj), _ptr(dq_traj), gu.data_ptr(), _ptr(cot[0]), _ptr(cot[5]), gth.data_ptr(),
                              B, _stream(q0)))
            gth = torch.sum(gth, 0).to(theta.dtype)
        if u.dim() == 2:
            gu = gu.sum(1)
        return None, None, gq0, gdq0, gu, None, gth


def simulate(rc, q, dq, u, dt, path, effort_weight, compensate_gravity, ref_frame, xyz_offset, record, theta=None):
    n = rc.N_JOINTS
    ref = _ref_tensor(q, dq, u, theta)
    dtype = q.dtype if isinstance(q, torch.Tensor) else ref.dtype
    ref = torch.empty((), dtype=dtype, device=ref.device)
    qa, dqa = _like(q, ref, "q"), _like(dq, ref, "dq")
    if tuple(qa.shape) != tuple(dqa.shape) or qa.dim() not in (1, 2) or qa.shape[-1] != n:
        raise ValueError("q and dq must have the same type, dtype and shape")
    single = qa.dim() == 1
    qa, dqa = qa.reshape(-1, n).contiguous(), dqa.reshape(-1, n).contiguous()
    ua = _like(u, ref, "u").contiguous()
    pa = None if path is None else _like(path, ref, "path").contiguous()
    for k in record:
        if k not in ("q", "dq", "u", "x"):
            raise ValueError(f"simulate can record 'q', 'dq', 'u' and 'x', not {k!r}")
    opts = dict(dt=dt, effort_weight=effort_weight, compensate_gravity=compensate_gravity, ref_frame=ref_frame,
                xyz_offset=xyz_offset, record=tuple(record))
    out = _Simulate.apply(rc, opts, qa, dqa, ua, pa, _grad_theta(theta, ref))
    qf, dqf, cost = out[:3]
    traj = dict(zip(opts["record"], out[3:]))
    if single:
        return qf[0], dqf[0], {k: v[:, 0] for k, v in traj.items()}, cost[0]
    return qf, dqf, traj, cost
