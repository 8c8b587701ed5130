"""TEST INFRASTRUCTURE — batched CPU oracle for ``OSC.generate`` and the secondary controllers (NumPy, fp64).

``osc_oracle`` evaluates one state per call, which is too slow for references of a few hundred thousand states.  This
module restates it step for step on stacked ``(B, ...)`` arrays; ``tests/test_gpu_general_fullsize.py`` pins the two
together on every entry of ``tests/cases.py``.

* rigid-body quantities: one ``ChainOracle.walk(q, 1)`` per chunk of states (every frame's T and D), plus
  ``ChainOracle.C`` where ``use_C`` asks for it.  A Jacobian at a per-state point is ``D_k [x, 1]`` state by state
  (J is linear in ``[x, 1]``), which is what ``AvoidObstacles`` needs;
* ``OSC._Mx``: ``inv`` / ``det`` / ``pinv(rcond=1e-4)`` on ``(B, k, k)`` stacks;
* orientation error, algorithms 0 and 1: ``quaternion_from_matrix`` as ``eigh`` of a ``(B, 4, 4)`` stack;
* ``vmax``; the per-state ``np.all(target_velocity == 0)`` branch (osc.py:275); ``use_C`` / ``use_g``; the training
  signal; ``ki`` with one integrator row per state;
* ``Damping``, ``RestingConfig``, ``AvoidJointLimits`` and ``AvoidObstacles``, each projected as in osc.py:310-318.

Besides u it returns, per state, how far the state is from a point where u is discontinuous, so that a comparison can
leave out the states where rounding legitimately picks the side of a jump (see ``generate``).

Only ``tests/`` may import this.
"""
import types

import numpy as np

from . import rbd_oracle as ro

ETA = 0.02  # avoid_obstacles.py:92
_NULL = ("Damping", "RestingConfig", "AvoidObstacles", "AvoidJointLimits")


# ---------------------------------------------------------------------------------------------- rigid-body quantities
class Walk:
    """The frames of one ``ChainOracle.walk(q, 1)`` over a batch."""

    def __init__(self, ch, q):
        self.ch, self.s, self.B = ch, ch.walk(q, 1), len(q)

    def _xh(self, x):
        xh = np.zeros((self.B, 4))
        xh[:, 3] = 1.0
        if x is not None:
            xh[:, :3] = x
        return xh

    def Tx(self, name, x=None):
        return np.einsum("bij,bj->bi", self.s[name].T, self._xh(x))[:, :3]

    def R(self, name):
        return self.s[name].T[:, :3, :3]

    def T_inv_apply(self, name, p):
        """T_inv(name) [p, 1] (transpose form, base_config.py:791-837)"""
        T = self.s[name].T
        Rt = np.swapaxes(T[:, :3, :3], 1, 2)
        return np.einsum("bij,bj->bi", Rt, p - T[:, :3, 3])

    def J(self, name, x=None):
        """(B, 6, n); x None, (3,) or one point per state (B, 3)"""
        xh = self._xh(x)
        ch = self.ch
        J = np.zeros((self.B, 6, ch.n))
        ep = ch.end_point(name)
        for k in range(ch.n):
            J[:, :3, k] = np.einsum("bij,bj->bi", self.s[name].D[k], xh)[:, :3]
            if k < ep:
                J[:, 3:, k] = self.s[f"joint{k}"].T[:, :3, 2]
        return J

    def M_g(self):
        ch = self.ch
        M, g = 0.0, 0.0
        for l in range(ch.n_links):
            Jl = ch._J_from(self.s, f"link{l}")
            M = M + np.einsum("bik,i,bij->bkj", Jl, ch.W[l], Jl)
            g = g + np.einsum("bik,i->bk", Jl, ch.W[l] * ch.gravity)
        return M, g


def coriolis(ch, q, dq, chunk=2048):
    """ChainOracle.C in chunks (its second-order walk holds n^2 matrices per frame)"""
    return np.concatenate([ch.C(q[b:b + chunk], dq[b:b + chunk]) for b in range(0, len(q), chunk)])


def _mv(A, x):
    return np.einsum("bij,bj->bi", A, x)


# ---------------------------------------------------------------------------------------------- quaternions
def quaternion_from_matrix(R):
    """rbd_oracle.quaternion_from_matrix on a (B, 3, 3) stack"""
    m = R
    K = np.zeros((len(R), 4, 4))
    K[:, 0, 0] = m[:, 0, 0] - m[:, 1, 1] - m[:, 2, 2]
    K[:, 1, 0] = m[:, 0, 1] + m[:, 1, 0]
    K[:, 1, 1] = m[:, 1, 1] - m[:, 0, 0] - m[:, 2, 2]
    K[:, 2, 0] = m[:, 0, 2] + m[:, 2, 0]
    K[:, 2, 1] = m[:, 1, 2] + m[:, 2, 1]
    K[:, 2, 2] = m[:, 2, 2] - m[:, 0, 0] - m[:, 1, 1]
    K[:, 3, 0] = m[:, 2, 1] - m[:, 1, 2]
    K[:, 3, 1] = m[:, 0, 2] - m[:, 2, 0]
    K[:, 3, 2] = m[:, 1, 0] - m[:, 0, 1]
    K[:, 3, 3] = m[:, 0, 0] + m[:, 1, 1] + m[:, 2, 2]
    K /= 3.0
    w, V = np.linalg.eigh(K)  # lower triangle, as the per-state call
    top = V[np.arange(len(R)), :, np.argmax(w, axis=1)]
    qv = top[:, [3, 0, 1, 2]]
    return np.where(qv[:, :1] < 0.0, -qv, qv)


def unit_vector(v):
    return v / np.sqrt(np.sum(v * v, axis=1, keepdims=True))


def quaternion_from_euler_rxyz(a):
    """rbd_oracle.quaternion_from_euler_rxyz on (B, 3) angles"""
    ai, aj, ak = a[:, 2] / 2.0, -a[:, 1] / 2.0, a[:, 0] / 2.0  # frame: ai <-> ak; parity: aj = -aj
    ci, si, cj, sj, ck, sk = np.cos(ai), np.sin(ai), np.cos(aj), np.sin(aj), np.cos(ak), np.sin(ak)
    cc, cs, sc, ss = ci * ck, ci * sk, si * ck, si * sk
    qv = np.empty((len(a), 4))
    qv[:, 0] = cj * cc + sj * ss
    qv[:, 3] = cj * sc - sj * cs  # i = 3
    qv[:, 2] = -(cj * ss + sj * cc)  # j = 2, negated by parity
    qv[:, 1] = cj * cs - sj * sc  # k = 1
    return qv


def euler_matrix_rxyz(a):
    """rbd_oracle.euler_matrix_rxyz on (B, 3) angles: i, j, k = 2, 1, 0"""
    ai, aj, ak = -a[:, 2], -a[:, 1], -a[:, 0]
    si, sj, sk = np.sin(ai), np.sin(aj), np.sin(ak)
    ci, cj, ck = np.cos(ai), np.cos(aj), np.cos(ak)
    cc, cs, sc, ss = ci * ck, ci * sk, si * ck, si * sk
    M = np.zeros((len(a), 3, 3))
    M[:, 2, 2] = cj * ck
    M[:, 2, 1] = sj * sc - cs
    M[:, 2, 0] = sj * cc + ss
    M[:, 1, 2] = cj * sk
    M[:, 1, 1] = sj * ss + cc
    M[:, 1, 0] = sj * cs - sc
    M[:, 0, 2] = -sj
    M[:, 0, 1] = cj * si
    M[:, 0, 0] = cj * ci
    return M


def quaternion_multiply(q1, q0):
    w0, x0, y0, z0 = q0.T
    w1, x1, y1, z1 = q1.T
    return np.stack([-x1 * x0 - y1 * y0 - z1 * z0 + w1 * w0, x1 * w0 + y1 * z0 - z1 * y0 + w1 * x0,
                     -x1 * z0 + y1 * w0 + z1 * x0 + w1 * y0, x1 * y0 - y1 * x0 + z1 * w0 + w1 * z0], axis=1)


def orientation_error(alg, W, frame, abg):
    """osc.py:149-196 -> ((B, 3) error, (B,) w of the quaternion whose sign decides it)"""
    if alg == 0:
        want = unit_vector(quaternion_from_euler_rxyz(abg))
        have = unit_vector(quaternion_from_matrix(W.R(frame)))
        rel = quaternion_multiply(want, have * np.array([1.0, -1, -1, -1]))
        return -rel[:, 1:] * np.sign(rel[:, :1]), rel[:, 0]
    if alg == 1:
        R_e = W.R(frame)
        rel = unit_vector(quaternion_from_matrix(np.swapaxes(R_e, 1, 2) @ euler_matrix_rxyz(abg)))
        return -1 * _mv(R_e, rel[:, 1:]), rel[:, 0]
    raise Exception(f"Invalid algorithm number {alg}")


# ---------------------------------------------------------------------------------------------- secondary controllers
# Each returns (tau (B, n), info): info holds the per-state distances to the controller's discontinuities (inf where
# it has none) and `active`, whether its term is non-zero.
def _inf(B):
    return np.full(B, np.inf)


def damping(W, q, dq, M, Minv, kv):
    return _mv(M, -kv * dq), dict(active=np.any(dq != 0, axis=1))


def resting_config(W, q, dq, M, Minv, rest_angles, kp=1, kv=None):
    kv = np.sqrt(kp) if kv is None else kv
    idx = np.array([v is not None for v in rest_angles])
    rest = np.array([0.0 if v is None else v for v in rest_angles])
    q_tilde = np.zeros_like(q)
    m = (rest[idx] - q[:, idx] + np.pi) % (np.pi * 2)
    q_tilde[:, idx] = m - np.pi
    wrap = np.minimum(m, 2 * np.pi - m).min(axis=1) if idx.any() else _inf(len(q))  # the wrap at +-pi
    return _mv(M, kp * q_tilde + kv * (0.0 - dq)), dict(active=np.ones(len(q), bool), wrap=wrap)


def avoid_joint_limits(W, q, dq, M, Minv, min_joint_angles, max_joint_angles, max_torque=None, cross_zero=None,
                       gradient=None):
    """osc_oracle.AvoidJointLimits on (B, n)"""
    n = q.shape[1]
    lo = np.array([np.nan if v is None else v - np.pi for v in min_joint_angles], dtype=float)
    hi = np.array([np.nan if v is None else v - np.pi for v in max_joint_angles], dtype=float)
    cz = np.array([False] * n if cross_zero is None else cross_zero)
    gr = np.array([False] * n if gradient is None else gradient)
    lo, hi = np.where(cz, hi, lo), np.where(cz, lo, hi)
    tmax = np.ones(n) if max_torque is None else np.asarray(max_torque, dtype=float)
    q = q - np.pi
    with np.errstate(all="ignore"):
        nearer_hi = np.abs(q - lo) >= np.abs(q - hi)
        nearer_lo = np.abs(q - lo) <= np.abs(q - hi)
        a_lo, a_hi = np.zeros_like(q), np.zeros_like(q)
        a_lo[:, gr] = np.minimum(np.exp(1.0 / (q[:, gr] - lo[gr])), tmax[gr])
        a_hi[:, gr] = -np.minimum(np.exp(-1.0 / (q[:, gr] - hi[gr])), tmax[gr])
        below = (q - lo) < 0
        above = (q - hi) > 0
        below[:, cz] = below[:, cz] & ((q[:, cz] - hi[cz]) > 0) & nearer_lo[:, cz]
        above[:, cz] = above[:, cz] & ((q[:, cz] - lo[cz]) < 0) & nearer_hi[:, cz]
        a_lo = np.where(below, tmax, a_lo)
        a_lo[:, np.isnan(lo)] = 0.0
        a_hi = np.where(above, -tmax, a_hi)
        a_hi[:, np.isnan(hi)] = 0.0
        # steps: q at a limit, and on cross_zero joints the nearer_lo / nearer_hi tie
        step = np.fmin(np.abs(q - lo), np.abs(q - hi))
        step = np.where(np.isnan(step), np.inf, step).min(axis=1)
        tie = np.abs(np.abs(q - lo) - np.abs(q - hi))
        tie = np.where(cz & ~np.isnan(tie), tie, np.inf).min(axis=1)
        # conditioning of the exp(1/(q - lim)) gradient: |d a / d q| / max|a| over the gradient joints on the
        # smooth side of the clip
        slope = np.zeros(len(q))
        for j in np.where(gr)[0]:
            for a, lim in ((a_lo[:, j], lo[j]), (a_hi[:, j], hi[j])):
                if np.isnan(lim):
                    continue
                smooth = (np.abs(a) < tmax[j]) & (a != 0)
                slope = np.maximum(slope, np.where(smooth, np.abs(a) / (q[:, j] - lim) ** 2, 0.0))
    tau = a_lo + a_hi
    return tau, dict(active=np.any(tau != 0, axis=1), step=step, tie=tie, slope=slope)


def avoid_obstacles(W, q, dq, M, Minv, obstacles=None, threshold=0.2, gain=1, maximum=500):
    """osc_oracle.AvoidObstacles on (B, n): one term per (obstacle, segment) pair, the pair's Jacobian at its closest
    point, and the rcond = 0.01 pinv of its Jp M^-1 Jp^T (avoid_obstacles.py:38-120)"""
    B, n = q.shape
    thr = threshold
    total = np.zeros((B, n))
    trunc = np.zeros(B, bool)  # a singular value of a pair's Jp M^-1 Jp^T within 0.1 % of the cut-off
    pairs = np.zeros(B, int)
    for ob in np.array([] if obstacles is None else obstacles, dtype=float).reshape(-1, 4):
        centre, radius = ob[:3], ob[3]
        for seg in range(n):
            p_a = W.Tx(f"joint{seg}")
            p_b = W.Tx("EE") if seg == n - 1 else W.Tx(f"joint{seg + 1}")
            sv = p_b - p_a
            with np.errstate(all="ignore"):
                s = np.sum((centre - p_a) * sv, axis=1) / np.sum(sv ** 2, axis=1)
                near = np.where((s < 0)[:, None], p_a, np.where((s > 1)[:, None], p_b, p_a + s[:, None] * sv))
                rho = np.sqrt(np.sum((centre - near) ** 2, axis=1)) - radius
            rho = np.where(rho < thr / 50, thr / 50, rho)  # Python's max(rho, thr / 50): a NaN rho stays NaN, inactive
            on = rho < thr
            if not on.any():
                continue
            r = rho[on][:, None]
            force = ETA * (1.0 / r - 1.0 / thr) * 1.0 / r ** 1.5 * ((centre - near[on]) / r)
            local = W.T_inv_apply(f"link{seg + 1}", near)
            Jp = W.J(f"link{seg + 1}", local)[on, :3]
            S = Jp @ Minv[on] @ np.swapaxes(Jp, 1, 2)
            Mx_pt = np.linalg.pinv(S, rcond=0.01)
            total[on] += -1 * _mv(np.swapaxes(Jp, 1, 2), _mv(Mx_pt, force))
            sig = np.linalg.svd(S, compute_uv=False)
            trunc[on] |= np.any(np.abs(sig / (0.01 * sig[:, :1]) - 1) <= 1e-3, axis=1)
            pairs[on] += 1
    tau = np.clip(total * gain, -maximum, maximum)
    return tau, dict(active=pairs > 0, trunc=trunc, pairs=pairs)


NULL = dict(Damping=damping, RestingConfig=resting_config, AvoidJointLimits=avoid_joint_limits,
            AvoidObstacles=avoid_obstacles)


def _merge(info, B, part):
    for k, v in part.items():
        if k in ("active", "trunc"):
            info[k] = info.get(k, np.zeros(B, bool)) | v
        elif k == "pairs":
            info[k] = info.get(k, 0) + v
        elif k == "slope":
            info[k] = np.maximum(info.get(k, np.zeros(B)), v)
        else:
            info[k] = np.minimum(info.get(k, _inf(B)), v)


def null_generate(arm, kind, kw, q, dq, chunk=8192):
    """one secondary controller alone (osc_oracle.run_null_case) -> namespace(u, active, and the distances)"""
    ch = ro.ChainOracle(arm) if isinstance(arm, str) else arm
    us, infos = [], []
    for b0 in range(0, len(q), chunk):
        qc, dqc = q[b0:b0 + chunk], dq[b0:b0 + chunk]
        W = Walk(ch, qc)
        M, _ = W.M_g()
        u, info = NULL[kind](W, qc, dqc, M, np.linalg.inv(M), **kw)
        full = {}
        _merge(full, len(qc), info)
        us.append(u)
        infos.append(full)
    return _namespace(dict(u=np.concatenate(us)), infos)


def _namespace(out, infos):
    for k in infos[0]:
        out[k] = np.concatenate([np.broadcast_to(i[k], (len(i["active"]),)) for i in infos])
    return types.SimpleNamespace(**out)


# ---------------------------------------------------------------------------------------------- OSC.generate
def _osc_chunk(ch, case, q, dq, tg, tv, es, Cm):
    kw = case["osc"]
    n = ch.n
    kp = kw.get("kp", 1)
    ko = kp if kw.get("ko") is None else kw["ko"]
    kv = np.sqrt(kp + ko) if kw.get("kv") is None else kw["kv"]
    ki, vmax = kw.get("ki", 0), kw.get("vmax")
    sel = np.array(kw.get("ctrlr_dof") or [1, 1, 1, 0, 0, 0], dtype=bool)
    gains = np.array([kp] * 3 + [ko] * 3, dtype=float)
    frame = case.get("ref_frame") or "EE"
    x = None if case.get("xyz_offset") is None else np.asarray(case["xyz_offset"], dtype=float)
    B = len(q)
    W = Walk(ch, q)
    J = W.J(frame, x)[:, sel]  # osc.py:242-244
    M, g = W.M_g()
    Minv = np.linalg.inv(M)  # _Mx, osc.py:120-147
    S = J @ Minv @ np.swapaxes(J, 1, 2)
    well = np.abs(np.linalg.det(S)) >= 1e-3
    Mx = np.empty_like(S)
    if well.any():
        Mx[well] = np.linalg.inv(S[well])
    if (~well).any():
        Mx[~well] = np.linalg.pinv(S[~well], rcond=1e-4)
    err = np.zeros((B, 6))
    w = np.full(B, np.inf)
    if sel[:3].any():  # osc.py:253-255
        err[:, :3] = W.Tx(frame, x) - tg[:, :3]
    if sel[3:].any():  # osc.py:258-259
        err[:, 3:], w = orientation_error(kw.get("orientation_algorithm", 0), W, frame, tg[:, 3:])
    if ki != 0:  # osc.py:262-264
        es = es + err
        err = err + ki * es
    if vmax is not None:  # osc.py:198-215
        lim_xyz, lim_abg = vmax[0] / kp * kv, vmax[1] / ko * kv
        s = np.ones((B, 6))
        nx, na = np.linalg.norm(err[:, :3], axis=1), np.linalg.norm(err[:, 3:], axis=1)
        with np.errstate(all="ignore"):
            s[:, :3] *= np.where(nx > lim_xyz, lim_xyz / nx, 1.0)[:, None]
            s[:, 3:] *= np.where(na > lim_abg, lim_abg / na, 1.0)[:, None]
        err = kv * s * (gains / kv) * err
    else:
        err = err * gains
    rest = np.all(tv == 0, axis=1)  # osc.py:275-282, per state
    u = np.where(rest[:, None], -1 * kv * _mv(M, dq), 0.0)
    xdot = np.zeros((B, 6))
    xdot[:, sel] = _mv(J, dq)
    err = np.where(rest[:, None], err, err + kv * (xdot - tv))
    u = u - _mv(np.swapaxes(J, 1, 2), _mv(Mx, err[:, sel]))  # osc.py:285-288
    if kw.get("use_C", False):
        u = u - _mv(Cm, dq)
    tr = u.copy()  # osc.py:297
    if kw.get("use_g", True):
        u = u - g
    info = {"active": np.zeros(B, bool)}
    tau_sum = np.zeros((B, n))
    if case.get("null"):
        P = np.eye(n) - np.swapaxes(J, 1, 2) @ np.swapaxes(Minv @ np.swapaxes(J, 1, 2) @ Mx, 1, 2)
        for kind, nkw in case["null"]:
            tau, part = NULL[kind](W, q, dq, M, Minv, **nkw)
            u = u + _mv(P, tau)  # osc.py:310-318
            tau_sum = tau_sum + tau
            _merge(info, B, part)
        info.update(tau=np.abs(tau_sum).max(axis=1))
    evs = np.linalg.eigvalsh(S)
    info.update(pinv=~well, amb=np.any(np.abs(evs / (1e-4 * evs[:, -1:]) - 1) <= 1e-3, axis=1),
                cond=np.linalg.cond(S), w=np.abs(w), rest=rest)
    return dict(u=u, tr=tr, err_sum=es), info


def generate(case, q, dq, target, target_velocity=None, err_sum=None, C=None, chunk=8192):
    """``OSC(**case["osc"], null_controllers=case["null"]).generate`` over a batch, as osc_oracle.run_case evaluates
    one state at a time (tests/cases.py case format).  target_velocity: None, (6,) or (B, 6).  err_sum: the (B, 6)
    integrator rows before the call (ki != 0).  C: precomputed (B, n, n) Coriolis matrices (use_C), else computed.

    Returns a namespace of (B, ...) arrays: u, tr (training signal), err_sum (after the call), and per state
      pinv    |det S| < 1e-3, S = J M^-1 J^T: the truncating pseudo-inverse route;
      amb     an eigenvalue of S within 0.1 % of the cut-off 1e-4 lambda_max (rounding decides the truncation);
      cond    cond(S);
      w       |w| of the orientation quaternion whose sign u follows (inf when no orientation row is controlled);
      rest    the target velocity row is all zero (the osc.py:275 branch);
      active  some secondary controller's term is non-zero;
    and, from the secondary controllers present: wrap (RestingConfig: distance to the +-pi wrap), step (joint
    limits: distance of q - pi to a limit), tie (cross_zero joints: | |q - lo| - |q - hi| |), slope (joint limits:
    |da/dq| / |a| of the exp(1/(q - lim)) gradient), trunc (an obstacle pair's singular value within 0.1 % of its
    cut-off), pairs (active obstacle pairs), and tau (max|sum of the secondary torques| before the projection).
    case["arm"] may also be an arm description (dict), e.g. one with perturbed constants."""
    ch = ro.ChainOracle(case["arm"])
    q, dq, target = (np.asarray(a, dtype=np.float64) for a in (q, dq, target))
    B = len(q)
    tv = np.zeros((B, 6)) if target_velocity is None else np.broadcast_to(np.asarray(target_velocity, float), (B, 6))
    es = np.zeros((B, 6)) if err_sum is None else np.asarray(err_sum, dtype=np.float64)
    if case["osc"].get("use_C", False) and C is None:
        C = coriolis(ch, q, dq)
    outs, infos = [], []
    for b0 in range(0, B, chunk):
        sl = slice(b0, b0 + chunk)
        o, info = _osc_chunk(ch, case, q[sl], dq[sl], target[sl], tv[sl], es[sl], None if C is None else C[sl])
        outs.append(o)
        infos.append(info)
    return _namespace({k: np.concatenate([o[k] for o in outs]) for k in outs[0]}, infos)
