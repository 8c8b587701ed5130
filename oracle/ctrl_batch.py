"""TEST INFRASTRUCTURE — batched CPU references (NumPy, fp64) for ``Joint``, ``Floating``, ``Sliding`` and
``InverseKinematics``.

``osc_oracle`` (``Joint``, ``Floating``, ``Sliding``) and ``ik_oracle`` evaluate one state per call, too slow for
references of tens of thousands of states.  This module restates them on stacked ``(B, ...)`` arrays, on top of
``ChainOracle``'s batched ``J``, ``dJ``, ``Tx``, ``M``, ``g`` and ``osc_batch.coriolis``, with the same stacked NumPy
calls (``pinv``, ``inv``, ``det``, ``solve``).  ``tests/test_ctrl_batch.py`` pins each function to the per-state oracle.

Every function returns a namespace of ``(B, ...)`` arrays: the controller's output and, per state, how close the state
is to a point where the output is discontinuous or ill-conditioned, so that a comparison can leave those states out:

  smin   the smallest singular value, relative to the largest, that a truncating pseudo-inverse (``numpy.linalg.pinv``,
         rcond = 1e-15, or rcond = 1e-4 for ``Floating``) keeps, over every pseudo-inverse the state takes (and, for
         IK, every step); 1 where none is taken.  For IK method 2 (no pseudo-inverse) it is 1 / cond(J J^T + 0.001 I),
         the damped solve's amplification of rounding.  Singular values the reference drops are exact zeros up to fp64
         rounding.  A small kept one is amplified by 1 / smin and lies where a kernel of lower precision drops it, so
         the output legitimately differs there (DESIGN.md, "fp32 pseudo-inverse cut").
  wrap   ``Joint``: distance of ``target - q + pi`` to a multiple of 2 pi, where q_tilde jumps from pi to -pi.
  pinv   ``Floating`` (task space): ``det(J M^-1 J^T) <= 1e-3``, the ``pinv(rcond=1e-4)`` route (floating.py's strict
         ``>``); ``det_gap``: ``|det / 1e-3 - 1|``, how close rounding is to switching routes; ``amb``: a singular
         value of that pinv within 0.1 % of its cut-off; ``cond``: cond(J M^-1 J^T) (1 without task_space).

Only ``tests/`` may import this.
"""
import types

import numpy as np

from . import rbd_oracle as ro
from .osc_batch import Walk, coriolis, quaternion_from_matrix, unit_vector

_RCOND = 1e-15  # numpy.linalg.pinv's default


def _mv(A, x):
    return np.einsum("bij,bj->bi", A, x)


def _chain(arm):
    return arm if isinstance(arm, ro.ChainOracle) else ro.ChainOracle(arm)


def _rows(x, B, w):
    """None / scalar / (w,) / (B, w) -> (B, w)"""
    if x is None:
        return np.zeros((B, w))
    return np.broadcast_to(np.asarray(x, dtype=np.float64), (B, w))


def _pinv(A, rcond=_RCOND):
    """numpy.linalg.pinv of a (B, r, c) stack, the smallest kept relative singular value of each, and whether one of
    its singular values lies within 0.1 % of the cut-off (rounding decides whether it is dropped)"""
    s = np.linalg.svd(A, compute_uv=False)
    rel = s / np.where(s[:, :1] > 0, s[:, :1], 1.0)
    kept = np.where(rel > rcond, rel, np.inf).min(axis=1)
    amb = np.any(np.abs(rel / rcond - 1) <= 1e-3, axis=1)
    return np.linalg.pinv(A, rcond=rcond), np.where(np.isinf(kept), 1.0, kept), amb


def _pinv_norm(A):
    """|pinv(A)|_2 (numpy's rcond): 1 / the smallest kept singular value, 0 for a zero matrix"""
    s = np.linalg.svd(A, compute_uv=False)
    kept = np.where(s > _RCOND * s[:, :1], s, np.inf).min(axis=1)
    return np.where(np.isfinite(kept) & (kept > 0), 1.0 / kept, 0.0)


def _ns(parts):
    return types.SimpleNamespace(**{k: np.concatenate([p[k] for p in parts]) for k in parts[0]})


# ---------------------------------------------------------------------------------------------- Joint
def joint(arm, q, dq, target, target_velocity=None, kp=1, kv=None, account_for_gravity=True, chunk=8192):
    """``Joint(kp, kv, account_for_gravity).generate`` (controllers/joint.py:104-131) -> namespace(u, wrap, scale);
    scale: the larger of max|M (kp q_tilde + kv (tv - dq))| and max|g|, the terms whose rounding u inherits (u itself
    can be much smaller where they cancel)"""
    ch = _chain(arm)
    q, dq = np.asarray(q, np.float64), np.asarray(dq, np.float64)
    B, n = q.shape
    kv = np.sqrt(kp) if kv is None else kv
    tg, tv = _rows(target, B, n), _rows(target_velocity, B, n)
    parts = []
    for b0 in range(0, B, chunk):
        sl = slice(b0, b0 + chunk)
        M, g = Walk(ch, q[sl]).M_g()
        m = (tg[sl] - q[sl] + np.pi) % (np.pi * 2)
        u = _mv(M, kp * (m - np.pi) + kv * (tv[sl] - dq[sl]))
        scale = np.maximum(np.abs(u).max(axis=1), np.abs(g).max(axis=1) if account_for_gravity else 0.0)
        parts.append(dict(u=u - g if account_for_gravity else u, wrap=np.minimum(m, 2 * np.pi - m).min(axis=1),
                          scale=scale))
    return _ns(parts)


# ---------------------------------------------------------------------------------------------- Floating
def floating(arm, q, dq, dynamic=False, task_space=False, chunk=8192):
    """``Floating(dynamic, task_space).generate`` (controllers/floating.py:27-71) -> namespace(u, pinv, det_gap, amb, cond, smin)"""
    ch = _chain(arm)
    q, dq = np.asarray(q, np.float64), np.asarray(dq, np.float64)
    B = len(q)
    parts = []
    for b0 in range(0, B, chunk):
        qc, dqc = q[b0:b0 + chunk], dq[b0:b0 + chunk]
        Bc = len(qc)
        W = Walk(ch, qc)
        M, g = W.M_g()
        info = dict(pinv=np.zeros(Bc, bool), det_gap=np.full(Bc, np.inf), smin=np.ones(Bc), amb=np.zeros(Bc, bool),
                    cond=np.ones(Bc))
        if task_space:
            J = W.J("EE")[:, :3]
            Minv = np.linalg.inv(M)
            S = J @ Minv @ np.swapaxes(J, 1, 2)
            det = np.linalg.det(S)
            well = np.abs(det) > 1e-3
            Mx = np.empty_like(S)
            if well.any():
                Mx[well] = np.linalg.inv(S[well])
            if (~well).any():
                Mx[~well], info["smin"][~well], info["amb"][~well] = _pinv(S[~well], 1e-4)
            Jbar = Minv @ np.swapaxes(J, 1, 2) @ Mx
            u = _mv(np.swapaxes(J, 1, 2), -1 * _mv(np.swapaxes(Jbar, 1, 2), g))
            info.update(pinv=~well, det_gap=np.abs(np.abs(det) / 1e-3 - 1), cond=np.linalg.cond(S))
        else:
            u = -g
        if dynamic:
            u = u - _mv(M, dqc)
        parts.append(dict(u=u, **info))
    return _ns(parts)


# ---------------------------------------------------------------------------------------------- Sliding
def sliding(arm, q, dq, target, target_velocity=None, target_acc=None, kd=160.0, lamb=30.0, cartesian=True,
            ref_frame="EE", offset=None, chunk=1024):
    """``Sliding(kd, lamb, cartesian).generate`` (controllers/sliding.py:27-99) -> namespace(u, s, smin).  Rows of
    ``target`` / ``target_velocity`` / ``target_acc`` (None: zero) are 3 wide in Cartesian mode, n in joint mode, per
    state or one broadcast row.  ``chunk`` bounds the memory of the second-order walks behind dJ and C."""
    ch = _chain(arm)
    q, dq = np.asarray(q, np.float64), np.asarray(dq, np.float64)
    B, n = q.shape
    w = 3 if cartesian else n
    tg, tv, ta = _rows(target, B, w), _rows(target_velocity, B, w), _rows(target_acc, B, w)
    x = None if offset is None else np.asarray(offset, dtype=np.float64)
    parts = []
    for b0 in range(0, B, chunk):
        sl = slice(b0, b0 + chunk)
        qc, dqc = q[sl], dq[sl]
        W = Walk(ch, qc)
        smin = np.ones(len(qc))
        if cartesian:
            J = W.J(ref_frame, x)[:, :3]
            J_inv, smin, _ = _pinv(J)
            dJ = ch.dJ(ref_frame, qc, dqc, x)[:, :3]
            dq_ref = _mv(J_inv, tv[sl] + lamb * (tg[sl] - W.Tx(ref_frame, x)))
            ddq_ref = _mv(J_inv, ta[sl] + lamb * (tv[sl] - _mv(J, dqc)) - _mv(dJ, dq_ref))
        else:
            dq_ref = tv[sl] - lamb * (qc - tg[sl])
            ddq_ref = ta[sl] - lamb * (dqc - tv[sl])
        M, g = W.M_g()
        s = dqc - dq_ref
        u = _mv(M, ddq_ref) + _mv(coriolis(ch, qc, dqc), dq_ref) + g - kd * s
        parts.append(dict(u=u, s=s, smin=smin))
    return _ns(parts)


# ---------------------------------------------------------------------------------------------- InverseKinematics
def quaternion_from_euler_sxyz(a):
    """ik_oracle.quaternion_from_euler_sxyz on (B, 3) angles"""
    ai, aj, ak = a[:, 0] / 2.0, a[:, 1] / 2.0, a[:, 2] / 2.0
    ci, si, cj, sj, ck, sk = np.cos(ai), np.sin(ai), np.cos(aj), np.sin(aj), np.cos(ak), np.sin(ak)
    cc, cs, sc, ss = ci * ck, ci * sk, si * ck, si * sk
    return np.stack([cj * cc + sj * ss, cj * sc - sj * cs, cj * ss + sj * cc, cj * cs - sj * sc], axis=1)


def ik_step(arm, q, target, dt=0.001, method=3, max_dx=0.2, max_dr=2 * np.pi, max_dq=np.pi, chunk=8192):
    """One iteration of ``InverseKinematics.generate_path`` (inverse_kinematics.py:83-137): the joint step dq from
    each (B, n) state towards its (B, 6) or (6,) target -> namespace(dq, smin, scale).  scale: the size of the terms
    dq is summed from (|pinv(J)| |b|, |J| |y|, ...), which can be far larger than dq itself where b lies mostly outside
    the range of J; rounding is relative to it."""
    ch = _chain(arm)
    q = np.asarray(q, dtype=np.float64)
    B, n = q.shape
    tg = _rows(target, B, 6)
    max_dq, max_dx, max_dr = max_dq * dt, max_dx * dt, max_dr * dt
    parts = []
    for b0 in range(0, B, chunk):
        sl = slice(b0, b0 + chunk)
        Qd = unit_vector(quaternion_from_euler_sxyz(tg[sl, 3:]))
        W = Walk(ch, q[sl])
        J = W.J("EE")
        dx = tg[sl, :3] - W.Tx("EE")
        Qe = unit_vector(quaternion_from_matrix(W.R("EE")))
        dr = Qe[:, :1] * Qd[:, 1:] - Qd[:, :1] * Qe[:, 1:] - np.cross(Qd[:, 1:], Qe[:, 1:])  # :93
        ndx, ndr = np.linalg.norm(dx, axis=1, keepdims=True), np.linalg.norm(dr, axis=1, keepdims=True)
        dx = np.where(ndx > max_dx, dx / np.where(ndx > 0, ndx, 1.0) * max_dx, dx)
        dr = np.where(ndr > max_dr, dr / np.where(ndr > 0, ndr, 1.0) * max_dr, dr)
        smin = np.ones(len(J))
        nrm = lambda v: np.linalg.norm(v, axis=1)  # noqa: E731
        if method == 1:
            Jp, smin, _ = _pinv(J)
            b = np.hstack([dx, dr])
            dq = _mv(Jp, b)
            scale = _pinv_norm(J) * nrm(b)
        elif method == 2:
            S = J @ np.swapaxes(J, 1, 2) + np.eye(6) * 0.001
            y = np.linalg.solve(S, np.hstack([dx, dr * 0.3])[..., None])[..., 0]
            dq = _mv(np.swapaxes(J, 1, 2), y)
            smin = 1.0 / np.linalg.cond(S)  # no pseudo-inverse: the solve's amplification of rounding
            scale = np.linalg.norm(J, 2, axis=(1, 2)) * nrm(y)
        else:
            Jx = J[:, :3]
            pinv_Jx, kx, _ = _pinv(Jx)
            pinv_Jr, kr, _ = _pinv(J[:, 3:])
            dq = _mv(pinv_Jx, dx) + _mv(np.eye(n) - pinv_Jx @ Jx, _mv(pinv_Jr, dr))
            smin = np.minimum(kx, kr)
            scale = _pinv_norm(Jx) * nrm(dx) + 2 * _pinv_norm(J[:, 3:]) * nrm(dr)
        big = np.abs(dq).max(axis=1, keepdims=True)
        dq = np.where(big > max_dq, dq / np.where(big > 0, big, 1.0) * max_dq, dq)
        scale = np.where(big[:, 0] > max_dq, scale / np.where(big[:, 0] > 0, big[:, 0], 1.0) * max_dq, scale)
        parts.append(dict(dq=dq, smin=smin, scale=scale))
    return _ns(parts)


def ik_path(arm, position, target, n_timesteps=200, dt=0.001, method=3, **init):
    """``InverseKinematics(**init).generate_path`` for (B, n) starts and (B, 6) or (6,) targets ->
    namespace(pos, vel, smin, smin_t); pos and vel are (B, n_timesteps, n), smin_t (B, n_timesteps) is each step's
    smin and smin their minimum over the path."""
    ch = _chain(arm)
    q = np.array(position, dtype=np.float64)
    B, n = q.shape
    pos, vel, smin_t = np.zeros((B, n_timesteps, n)), np.zeros((B, n_timesteps, n)), np.ones((B, n_timesteps))
    for t in range(n_timesteps):
        st = ik_step(ch, q, target, dt, method, **init)
        pos[:, t], vel[:, t], smin_t[:, t] = q, st.dq, st.smin
        q = q + st.dq
    return types.SimpleNamespace(pos=pos, vel=vel, smin=smin_t.min(axis=1), smin_t=smin_t)
