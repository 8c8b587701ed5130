"""TEST INFRASTRUCTURE: an independent NumPy statement of the path planner (include/abrb.h, abrb_path_*).

Same definition as the reference's PathPlanner.generate_path (path_planner.py:144-397, orientation.py:157-198,
transformations.py), restated with array operations over the steps of a path, for many rows per call.  The velocity
search is scalar per row.  Rows the reference cannot plan get a negative length (the ABRB_PATH_* reasons).

``near_integer``: rows where the constant segment's int() argument, (curve length - ramp distances) / max_v / dt, lies
within 1e-9 of an integer, or where the search compared two distances within 1e-9 of each other.  Both depend on sums
(the curve length, the ramp distances), so there a different summation order (the device's) can legitimately change
the length by one.  The ramps' own counts depend on the speeds alone and are computed identically everywhere.
"""
import numpy as np

EPS = np.finfo(float).eps * 4.0
NEAR = 1e-9
AXES = {
    "sxyz": (0, 0, 0, 0), "sxyx": (0, 0, 1, 0), "sxzy": (0, 1, 0, 0), "sxzx": (0, 1, 1, 0),
    "syzx": (1, 0, 0, 0), "syzy": (1, 0, 1, 0), "syxz": (1, 1, 0, 0), "syxy": (1, 1, 1, 0),
    "szxy": (2, 0, 0, 0), "szxz": (2, 0, 1, 0), "szyx": (2, 1, 0, 0), "szyz": (2, 1, 1, 0),
    "rzyx": (0, 0, 0, 1), "rxyx": (0, 0, 1, 1), "ryzx": (0, 1, 0, 1), "rxzx": (0, 1, 1, 1),
    "rxzy": (1, 0, 0, 1), "ryzy": (1, 0, 1, 1), "rzxy": (1, 1, 0, 1), "ryxy": (1, 1, 1, 1),
    "ryxz": (2, 0, 0, 1), "rzxz": (2, 0, 1, 1), "rxyz": (2, 1, 0, 1), "rzyz": (2, 1, 1, 1),
}
NEXT = [1, 2, 0, 1]


def ramp(kind, dt, acc, n_sigma, va, vb):
    """-> (samples, the int() argument); kind "gaussian" or "linear"."""
    x = (vb - va) / acc / dt
    if not x < 2 ** 28:
        return None, x
    n = int(x)
    if n < 2:
        return None, x
    if kind == "linear":
        return np.linspace(va, vb, n), x
    dv = vb - va
    s = 1 / (dv * np.sqrt(np.pi * 2))
    u = n_sigma * s
    g = 1 / (s * np.sqrt(2 * np.pi)) * np.exp(-0.5 * ((np.linspace(0, u, n) - u) / s) ** 2)
    g = g - g[0]
    return g * (dv / g[-1]) + va, x


def _near(x):
    return abs(x - round(x)) < NEAR


def align(d):
    """align_vectors((1,1,1)/sqrt3, d) for rows d (B, 3) -> (R (B,3,3), ok (B,))"""
    a = np.full(3, 1 / np.sqrt(3))
    a = a / np.linalg.norm(a)
    b = d / np.linalg.norm(d, axis=1, keepdims=True)
    v = np.cross(a[None], b)
    c = b @ a
    ok = 1 + c > 0
    h = 1 / np.where(ok, 1 + c, 1.0)
    V = np.zeros((len(d), 3, 3))
    V[:, 0, 1], V[:, 0, 2], V[:, 1, 0] = -v[:, 2], v[:, 1], v[:, 2]
    V[:, 1, 2], V[:, 2, 0], V[:, 2, 1] = -v[:, 0], -v[:, 1], v[:, 0]
    return np.eye(3)[None] + V + (V @ V) * h[:, None, None], ok


def search(curve, kind, dt, acc, n_sigma, vmax, v0, v1):
    """The max_v search of one row -> (stacked velocity profile or a negative reason, near_integer)."""
    near = False
    s_spec, e_spec = v0 == vmax, v1 == vmax
    sp, ep = ([v0 * dt] if s_spec else None), ([v1 * dt] if e_spec else None)
    sd, ed = (0.0 if s_spec else None), (0.0 if e_spec else None)
    max_v = vmax
    while True:
        if max_v <= 0:
            return -3, near
        if sd is None or sd != 0:
            sp, x = ramp(kind, dt, acc, n_sigma, v0, max_v)
            if sp is None:
                return (-5 if not x < 2 ** 28 else -4), near
            sd = np.sum(sp * dt)
        if ed is None or ed != 0:
            r, x = ramp(kind, dt, acc, n_sigma, v1, max_v)
            if r is None:
                return (-5 if not x < 2 ** 28 else -4), near
            ep = r[::-1]
            ed = np.sum(ep * dt)
        near |= abs(curve - (sd + ed)) < NEAR
        if curve > sd + ed:
            x = (curve - (ed + sd)) / max_v / dt
            near |= _near(x)
            if not x < 2 ** 28:
                return -5, near
            return np.hstack((sp, np.ones(int(x)) * max_v, ep)), near
        if curve == sd + ed:
            return np.hstack((sp, ep)), near
        max_v -= 0.1


def quat_from_euler(e, axes):
    fa, par, rep, frm = AXES[axes]
    i = fa + 1
    j = NEXT[i + par - 1] + 1
    k = NEXT[i - par] + 1
    ai, aj, ak = e
    if frm:
        ai, ak = ak, ai
    if par:
        aj = -aj
    ci, si, cj, sj, ck, sk = np.cos(ai / 2), np.sin(ai / 2), np.cos(aj / 2), np.sin(aj / 2), np.cos(ak / 2), np.sin(ak / 2)
    cc, cs, sc, ss = ci * ck, ci * sk, si * ck, si * sk
    q = np.empty(4)
    if rep:
        q[0], q[i], q[j], q[k] = cj * (cc - ss), cj * (cs + sc), sj * (cc + ss), sj * (cs - sc)
    else:
        q[0], q[i], q[j], q[k] = cj * cc + sj * ss, cj * sc - sj * cs, cj * ss + sj * cc, cj * cs - sj * sc
    if par:
        q[j] *= -1.0
    return q


def slerp(q0, q1, f):
    """quaternion_slerp for fractions f (S,) -> (S, 4)"""
    q0, q1 = q0 / np.sqrt(q0 @ q0), q1 / np.sqrt(q1 @ q1)
    q1u = q1
    out = np.empty((len(f), 4))
    d = q0 @ q1
    if abs(abs(d) - 1.0) < EPS:
        out[:] = q0
    else:
        if d < 0:
            d, q1 = -d, -q1
        ang = np.arccos(d)
        if abs(ang) < EPS:
            out[:] = q0
        else:
            isin = 1.0 / np.sin(ang)
            out[:] = q0[None] * (np.sin((1.0 - f) * ang) * isin)[:, None] + q1[None] * (np.sin(f * ang) * isin)[:, None]
    out[f == 0.0] = q0
    out[f == 1.0] = q1u
    return out


def euler_from_quat(q, axes):
    """euler_from_matrix(quaternion_matrix(q)) for q (S, 4) -> (S, 3)"""
    n = np.sum(q * q, axis=1)
    qs = q * np.sqrt(2.0 / np.where(n < EPS, 1.0, n))[:, None]
    o = qs[:, :, None] * qs[:, None, :]
    M = np.empty((len(q), 3, 3))
    M[:, 0] = np.stack([1 - o[:, 2, 2] - o[:, 3, 3], o[:, 1, 2] - o[:, 3, 0], o[:, 1, 3] + o[:, 2, 0]], 1)
    M[:, 1] = np.stack([o[:, 1, 2] + o[:, 3, 0], 1 - o[:, 1, 1] - o[:, 3, 3], o[:, 2, 3] - o[:, 1, 0]], 1)
    M[:, 2] = np.stack([o[:, 1, 3] - o[:, 2, 0], o[:, 2, 3] + o[:, 1, 0], 1 - o[:, 1, 1] - o[:, 2, 2]], 1)
    M[n < EPS] = np.eye(3)
    fa, par, rep, frm = AXES[axes]
    i, j, k = fa, NEXT[fa + par], NEXT[fa - par + 1]
    if rep:
        sy = np.sqrt(M[:, i, j] ** 2 + M[:, i, k] ** 2)
        big = sy > EPS
        ax = np.where(big, np.arctan2(M[:, i, j], M[:, i, k]), np.arctan2(-M[:, j, k], M[:, j, j]))
        ay = np.arctan2(sy, M[:, i, i])
        az = np.where(big, np.arctan2(M[:, j, i], -M[:, k, i]), 0.0)
    else:
        cy = np.sqrt(M[:, i, i] ** 2 + M[:, j, i] ** 2)
        big = cy > EPS
        ax = np.where(big, np.arctan2(M[:, k, j], M[:, k, k]), np.arctan2(-M[:, j, k], M[:, j, j]))
        ay = np.arctan2(-M[:, k, i], cy)
        az = np.where(big, np.arctan2(M[:, j, i], M[:, i, i]), 0.0)
    if par:
        ax, ay, az = -ax, -ay, -az
    if frm:
        ax, az = az, ax
    return np.stack([ax, ay, az], axis=1)


def plan(table, start, target, max_velocity, start_velocity, target_velocity, kind, dt, acceleration, n_sigma=3,
         axes="rxyz", start_orientation=None, target_orientation=None):
    """Rows (B, 3) -> dict(lengths (B,) int64 (negative: reason), paths: list of (S_b, w) arrays (None where
    rejected), near_integer (B,) bool).  Speeds are scalars or (B,); orientations (3,) or (B, 3) or None."""
    table = np.asarray(table, dtype=np.float64)
    start, target = np.atleast_2d(np.asarray(start, float)), np.atleast_2d(np.asarray(target, float))
    B = len(start)
    vm, v0, v1 = (np.broadcast_to(np.asarray(v, float), (B,)) for v in (max_velocity, start_velocity, target_velocity))
    d = target - start
    dist = np.linalg.norm(d, axis=1)
    good = (dist > 0) & np.isfinite(dist)
    R, ok = align(np.where(good[:, None], d, 1.0))
    warped = np.einsum("bij,bpj->bpi", R, (1 / np.sqrt(3)) * table[None] * dist[:, None, None]) + start[:, None]
    seg = np.linalg.norm(np.diff(warped, axis=1), axis=2)
    arc = np.concatenate([np.zeros((B, 1)), np.cumsum(seg, axis=1)], axis=1)
    curve = np.sum(np.concatenate([np.zeros((B, 1)), seg], axis=1), axis=1)
    orient = start_orientation is not None
    if orient:
        so = np.broadcast_to(np.asarray(start_orientation, float), (B, 3))
        to = np.broadcast_to(np.asarray(target_orientation, float), (B, 3))
    lengths = np.zeros(B, dtype=np.int64)
    near = np.zeros(B, dtype=bool)
    paths = []
    for b in range(B):
        if not good[b] or not ok[b]:
            lengths[b] = -1 if not good[b] else -2
            paths.append(None)
            continue
        stacked, near[b] = search(curve[b], kind, dt, acceleration, n_sigma, vm[b], v0[b], v1[b])
        if isinstance(stacked, int):
            lengths[b] = stacked
            paths.append(None)
            continue
        s = np.cumsum(stacked * dt)
        x = arc[b]
        idx = np.clip(np.searchsorted(x, s, side="left"), 1, len(x) - 1)
        xl, xh = x[idx - 1], x[idx]
        y = ((s - xl) / (xh - xl))[:, None] * warped[b][idx] + ((xh - s) / (xh - xl))[:, None] * warped[b][idx - 1]
        cols = [y, np.gradient(y, dt, axis=0)]
        if orient:
            err = np.sqrt(np.sum((y[-1] - y) ** 2, axis=1)) / np.sqrt(np.sum((y[-1] - y[0]) ** 2))
            e = euler_from_quat(slerp(quat_from_euler(so[b], axes), quat_from_euler(to[b], axes), 1 - err), axes)
            cols += [e, np.gradient(e, dt, axis=0)]
        paths.append(np.hstack(cols))
        lengths[b] = len(stacked)
    return dict(lengths=lengths, paths=paths, near_integer=near)


def padded(paths, lengths):
    """(B, S_max, w) with each path's last row repeated past its length (rows of rejected paths: NaN)."""
    s_max = int(max(lengths.max(), 0))
    w = next(p.shape[1] for p in paths if p is not None)
    out = np.full((len(paths), s_max, w), np.nan)
    for b, p in enumerate(paths):
        if p is not None:
            out[b, : len(p)] = p
            out[b, len(p):] = p[-1]
    return out
