"""Closed-loop Joint and Sliding rollouts along a path (``Joint.rollout_path``, ``Sliding.rollout_path``;
``abrb_joint_rollout_path_*``, ``abrb_sliding_rollout_path_*``).

Semantics (include/abrb.h), for t = 0 .. S-1 from the state (q_t, dq_t) before the step:
    u_t = Joint.generate(q_t, dq_t, path[t], path_velocity[t])   or   Sliding.generate(q_t, dq_t, path[t], pv[t], pa[t])
    x_t = control point at q_t;  ddq = M^-1 (u_t + g - C dq_t);  dq_{t+1} = dq_t + ddq dt;  q_{t+1} = q_t + dq_{t+1} dt
    cost += e_t + w |u_t|^2,  e_t = |wrap(path[t] - q_t)|^2 (Joint), |x_t - path[t]|^2 (cartesian Sliding),
                              |q_t - path[t]|^2 (joint-mode Sliding)

CPU part: the NumPy definition (``oracle_ctrl_rollout``, on ``osc_oracle.Joint`` / ``osc_oracle.Sliding`` and
``rbd_oracle.ChainOracle``) against the kernel's per-step code run on the host through tests/hostsim/ctrlsim.cpp (TEST
INFRASTRUCTURE, never loaded by the package); the recorded torques against the single-state controllers and through
the plant rollout, bit for bit; convergence on gravity-free arms; argument checking of the C entry points.
GPU part: the kernels against the oracle and against ``generate``, the replay through ``simulate``, layout and size
properties, the input forms, the inverse-kinematics pipeline and random chains.
"""
import ctypes as C
import os

import numpy as np
import pytest

import cases
import test_plant as tp
from abr_control_b200 import _abi
from oracle import osc_oracle, rbd_oracle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ARMS = ("ur5", "jaco2", "threejoint", "twojoint")
STEPS, DT, EFFORT = 28, 1e-3, 1e-4
TOL = tp.TOL
JOINT, SLIDING = 0, 1


def wrap(d):
    return ((d + np.pi) % (np.pi * 2)) - np.pi


# ---------------------------------------------------------------------------------------------- the definition
def oracle_ctrl_rollout(arm, kind, kw, q, dq, path, dt, path_velocity=None, path_acc=None, effort_weight=0.0,
                        ref_frame="EE", offset=None):
    """NumPy stepping of the closed loop, float64.  ``kind``: "joint" or "sliding" with the controller's keyword
    arguments ``kw``; ``path``, ``path_velocity``, ``path_acc``: (S, w) shared or (S, B, w).
    -> dict(q, dq, u, x: (S, B, .); e: (S, B) the tracking terms; cost: (B,); q_final, dq_final)"""
    q, dq = np.array(q, dtype=np.float64), np.array(dq, dtype=np.float64)
    B, n = q.shape
    S = path.shape[0]

    def rows(a):
        return None if a is None else (np.broadcast_to(a[:, None], (S, B, a.shape[-1])) if a.ndim == 2 else a)

    P, PV, PA = rows(path), rows(path_velocity), rows(path_acc)
    ro = osc_oracle.RobotOracle(arm)
    ch = ro.chain
    ctrl = osc_oracle.Joint(ro, **kw) if kind == "joint" else osc_oracle.Sliding(ro, **kw)
    task = kind == "sliding" and ctrl.cartesian
    xo = None if offset is None else np.asarray(offset, dtype=np.float64)
    out = {k: np.zeros((S, B, 3 if k == "x" else n)) for k in ("q", "dq", "u", "x")}
    out["e"] = np.zeros((S, B))
    cost = np.zeros(B)
    for t in range(S):
        u = np.zeros((B, n))
        for b in range(B):
            if kind == "joint":
                u[b] = ctrl.generate(q[b], dq[b], P[t, b], None if PV is None else PV[t, b])
            else:
                extra = dict(ref_frame=ref_frame, offset=xo) if task else {}
                u[b] = ctrl.generate(q[b], dq[b], P[t, b], 0 if PV is None else PV[t, b], 0 if PA is None else PA[t, b],
                                     **extra)
        x = ch.Tx(ref_frame, q, xo)
        d = wrap(P[t] - q) if kind == "joint" else (x - P[t] if task else q - P[t])
        e = np.sum(d ** 2, axis=1)
        rhs = u + ch.g(q) - np.einsum("bij,bj->bi", ch.C(q, dq), dq)
        ddq = np.linalg.solve(ch.M(q), rhs[..., None])[..., 0]
        dq = dq + ddq * dt
        q = q + dq * dt
        cost += e + effort_weight * np.sum(u ** 2, axis=1)
        out["q"][t], out["dq"][t], out["u"][t], out["x"][t], out["e"][t] = q, dq, u, x, e
    out.update(cost=cost, q_final=q, dq_final=dq)
    return out


# the host and device cases: (controller, kwargs, row layout, path velocity?, path acceleration?, frame, offset)
VARIANTS = {
    "joint_grav_shared": ("joint", dict(kp=300, kv=20), "shared", False, False, "EE", None),
    "joint_grav_per_vel": ("joint", dict(kp=300, kv=20), "per", True, False, "EE", None),
    "joint_nograv_per": ("joint", dict(kp=300, kv=20, account_for_gravity=False), "per", False, False, "mid",
                         [0.02, -0.03, 0.05]),
    "joint_nograv_shared_vel": ("joint", dict(kp=100, kv=15, account_for_gravity=False), "shared", True, False, "EE",
                                None),
    "sliding_xyz_ee_per": ("sliding", dict(kd=8.0, lamb=20.0), "per", True, True, "EE", None),
    "sliding_xyz_mid_offset_shared": ("sliding", dict(kd=3.0, lamb=10.0), "shared", True, True, "mid",
                                      [0.01, 0.02, -0.04]),
    "sliding_joint_per": ("sliding", dict(kd=8.0, lamb=10.0, cartesian=False), "per", True, True, "mid",
                          [0.03, 0.0, 0.02]),
    "sliding_joint_shared": ("sliding", dict(kd=8.0, lamb=10.0, cartesian=False), "shared", False, False, "EE", None),
}


# a frame other than the end effector: on the 6-joint arms one that every joint but the last moves (a Sliding loop on a
# frame that fewer joints move left the oracle unstable at a 1 ms step); on twojoint the end effector with an offset
MID = {"ur5": "link5", "jaco2": "link5", "threejoint": "link3", "twojoint": "EE"}


def _task(kind, kw):
    return kind == "sliding" and kw.get("cartesian", True)


def _effective_cond(J):
    """condition number of each J over its non-negligible singular values (planar arms have an exactly zero z row)"""
    s = np.linalg.svd(J, compute_uv=False)
    keep = s > 1e-9 * s[:, :1]
    return s[:, 0] / np.where(keep, s, np.inf).min(axis=1)


def well_conditioned_starts(arm, B, frame="EE", offset=None, cond_max=12.0):
    """The first B seeded states whose J[:3] at the control point is well conditioned: across a truncated
    pseudo-inverse a Sliding trajectory turns chaotic, so neither the oracle nor the kernels could be compared."""
    q, dq, _, _ = cases.states(arm, 8 * B)
    ch = rbd_oracle.ChainOracle(arm)
    keep = _effective_cond(ch.J(frame, q, offset)[:, :3]) < cond_max
    assert keep.sum() >= B, (arm, frame, keep.sum())
    return np.ascontiguousarray(q[keep][:B]), np.ascontiguousarray(0.2 * dq[keep][:B])


def variant_inputs(arm, variant, B, S=STEPS, seed=0):
    """Well-conditioned starts and a short path from each: a ramp in joint space (with whole turns added for Joint,
    which wraps the error) or a 5 cm line in task space from the control point."""
    kind, kw, lay, vel, acc, frame, off = VARIANTS[variant]
    frame = MID[arm] if frame == "mid" else frame
    q, dq = well_conditioned_starts(arm, B, frame, off)
    n = q.shape[1]
    rng = np.random.default_rng(seed + cases.hash_name(arm + variant))
    if lay == "shared":  # one path for all: start every trajectory near the first one, which the path starts from
        q = np.ascontiguousarray(q[:1] + rng.uniform(-0.02, 0.02, q.shape))
    s = (np.arange(S) / S)[:, None, None]
    if _task(kind, kw):
        x0 = rbd_oracle.ChainOracle(arm).Tx(frame, q, off)
        d = rng.normal(size=x0.shape)
        d *= 0.05 / np.linalg.norm(d, axis=1, keepdims=True)
        path = x0[None] + s * d[None]
        w = 3
    else:
        d = rng.normal(size=q.shape) * 0.3
        path = q[None] + s * d[None]
        if kind == "joint":
            path = path + 2 * np.pi * rng.integers(-1, 2, size=q.shape)[None]
        w = n
    pv = rng.normal(size=(S, B, w)) * 0.2 if vel else None
    pa = rng.normal(size=(S, B, w)) * 0.5 if acc else None
    if lay == "shared":
        path, pv, pa = path[:, 0], None if pv is None else pv[:, 0], None if pa is None else pa[:, 0]
    c = lambda a: None if a is None else np.ascontiguousarray(a)  # noqa: E731
    return q, dq, c(path), c(pv), c(pa), kind, kw, frame, off


_ORACLE = {}


def oracle_for(arm, variant, B):
    key = (arm, variant, B)
    if key not in _ORACLE:
        q, dq, path, pv, pa, kind, kw, frame, off = variant_inputs(arm, variant, B)
        _ORACLE[key] = oracle_ctrl_rollout(arm, kind, kw, q, dq, path, DT, pv, pa, EFFORT, frame, off)
    return _ORACLE[key]


def _pre_states(q0, rec):
    """(S, B, n) states before each step from the start and the after-step records"""
    return np.concatenate([np.asarray(q0)[None], np.asarray(rec)[:-1]], axis=0)


def _bcast(a, S, B):
    return None if a is None else (np.broadcast_to(a[:, None], (S, B, a.shape[-1])) if a.ndim == 2 else a)


def test_oracle_cost_is_the_sum_over_its_own_records():
    """The oracle's cost equals its tracking terms recomputed from the records (pre-step q and x) plus the effort."""
    for arm, variant in (("ur5", "joint_grav_per_vel"), ("jaco2", "sliding_xyz_mid_offset_shared"),
                         ("threejoint", "sliding_joint_per")):
        B = 6
        q, dq, path, pv, pa, kind, kw, frame, off = variant_inputs(arm, variant, B, S=8)
        o = oracle_ctrl_rollout(arm, kind, kw, q, dq, path, DT, pv, pa, 0.3, frame, off)
        P = _bcast(path, 8, B)
        qpre = _pre_states(q, o["q"])
        d = wrap(P - qpre) if kind == "joint" else (o["x"] - P if _task(kind, kw) else qpre - P)
        cost = np.sum(d ** 2, axis=(0, 2)) + 0.3 * np.sum(o["u"] ** 2, axis=(0, 2))
        assert np.allclose(o["cost"], cost, rtol=1e-13, atol=0), variant
        ch = rbd_oracle.ChainOracle(arm)
        assert np.array_equal(o["x"][0], ch.Tx(frame, q, None if off is None else np.asarray(off)))


# ---------------------------------------------------------------------------------------------- host shims
@pytest.fixture(scope="module")
def ctrlsim(tmp_path_factory):
    return tp._build(tmp_path_factory, "ctrlsim")


@pytest.fixture(scope="module")
def plantsim(tmp_path_factory):
    return tp._build(tmp_path_factory, "plantsim")


@pytest.fixture(scope="module")
def hostsim(tmp_path_factory):
    return tp._build(tmp_path_factory, "hostsim")


_p = tp._p


def _desc(arm):
    return arm if isinstance(arm, _abi.ChainDesc) else _abi.chain_desc_from_dict(
        arm if isinstance(arm, dict) else _abi.load_arm_json(arm))


def _gains(kind, kw):
    if kind == "joint":
        kp = kw.get("kp", 1)
        return JOINT, float(kp), float(kw.get("kv", np.sqrt(kp))), int(kw.get("account_for_gravity", True))
    return SLIDING, float(kw.get("kd", 160.0)), float(kw.get("lamb", 30.0)), int(kw.get("cartesian", True))


def shim_rollout(cs, arm, kind, kw, q, dq, path, pv=None, pa=None, frame="EE", xoff=None, f32=0, dt=DT, effort=EFFORT):
    cd = _desc(arm)
    n, B = cd.n_joints, len(q)
    S = path.shape[0]
    w = 3 if _task(kind, kw) else n
    q, dq = np.array(q, dtype=np.float64), np.array(dq, dtype=np.float64)
    out = {k: np.zeros((S, B, 3 if k == "x" else n)) for k in ("q", "dq", "u", "x")}
    cost = np.zeros(B)
    xo = None if xoff is None else (C.c_double * 3)(*xoff)
    k, k1, k2, flag = _gains(kind, kw)
    arr = lambda a: None if a is None else np.ascontiguousarray(a, dtype=np.float64)  # noqa: E731
    stride = lambda a: 0 if a is None or a.ndim == 2 else w  # noqa: E731
    path, pv, pa = arr(path), arr(pv), arr(pa)
    rc = cs.cs_rollout(C.byref(cd), f32, k, C.c_double(k1), C.c_double(k2), flag, cs.hs_frame_id(n, frame.encode()), xo,
                       _p(q), _p(dq), _p(path), stride(path), _p(pv), stride(pv), _p(pa), stride(pa), S, C.c_double(dt),
                       C.c_double(effort), _p(out["q"]), _p(out["dq"]), _p(out["u"]), _p(out["x"]), _p(cost),
                       C.c_int64(B))
    assert rc == 0
    out.update(cost=cost, q_final=q, dq_final=dq)
    return out


@pytest.mark.parametrize("f32", [0, 1])
@pytest.mark.parametrize("variant", list(VARIANTS))
@pytest.mark.parametrize("arm", ARMS)
def test_host_rollout_vs_oracle(ctrlsim, arm, variant, f32):
    B = 24
    q, dq, path, pv, pa, kind, kw, frame, off = variant_inputs(arm, variant, B)
    ref = oracle_for(arm, variant, B)
    got = shim_rollout(ctrlsim, arm, kind, kw, q, dq, path, pv, pa, frame, off, f32=f32)
    tp.assert_matches_oracle(got, ref, f32, f"{arm} {variant}")
    assert np.abs(got["q_final"] - ref["q_final"]).max() < TOL[f32]["q"]


# the bookkeeping cases: every variant on UR5, the cartesian ones also on threejoint, joint mode on twojoint.  (The
# single-state Sliding code reads a 3-value target through an N-long array, so cartesian rows on a 2-joint arm are not
# compared against it.)
BOOK = [("ur5", v) for v in VARIANTS] + [("threejoint", "sliding_xyz_ee_per"), ("twojoint", "sliding_joint_per"),
                                         ("jaco2", "joint_nograv_per")]


@pytest.mark.parametrize("f32", [0, 1])
@pytest.mark.parametrize("arm,variant", BOOK)
def test_host_recorded_torques_are_the_controllers_and_replay_through_the_plant(ctrlsim, plantsim, hostsim, arm,
                                                                                 variant, f32):
    """Each recorded u_t is what joint_state / sliding_state give (hs_ctrl / hs_sliding) at the recorded pre-step
    state and row t, and u_traj replayed through the plant rollout (pl_rollout, no path, same effort weight) gives back
    q, dq and x: all bit for bit, since both sides run the same host code."""
    B, S = 10, 12
    q, dq, path, pv, pa, kind, kw, frame, off = variant_inputs(arm, variant, B, S=S)
    got = shim_rollout(ctrlsim, arm, kind, kw, q, dq, path, pv, pa, frame, off, f32=f32)
    cd = _desc(arm)
    n = cd.n_joints
    qpre, dqpre = _pre_states(q, got["q"]), _pre_states(dq, got["dq"])
    P, PV, PA = (_bcast(a, S, B) for a in (path, pv, pa))
    k, k1, k2, flag = _gains(kind, kw)
    fid = hostsim.hs_frame_id(n, frame.encode())
    xo = None if off is None else (C.c_double * 3)(*off)
    for t in range(S):
        u = np.zeros((B, n))
        c = lambda a: None if a is None else np.ascontiguousarray(a[t])  # noqa: E731
        qt, dqt, pt, pvt, pat = np.ascontiguousarray(qpre[t]), np.ascontiguousarray(dqpre[t]), c(P), c(PV), c(PA)
        if k == JOINT:
            rc = hostsim.hs_ctrl(C.byref(cd), f32, 0, 0, C.c_double(k1), C.c_double(k2), flag, 0, _p(qt), _p(dqt), _p(pt),
                                 _p(pvt), C.c_int64(B), _p(u))
        else:
            rc = hostsim.hs_sliding(C.byref(cd), f32, 0, C.c_double(k1), C.c_double(k2), flag, fid, xo, _p(qt), _p(dqt),
                                    _p(pt), _p(pvt), _p(pat), C.c_int64(B), _p(u), None)
        assert rc == 0
        assert np.array_equal(u, got["u"][t]), t
    rep = tp.shim_simulate(plantsim, arm, q, dq, got["u"], None, False, frame, off, f32=f32)
    for key in ("q", "dq", "u", "x"):
        assert np.array_equal(rep[key], got[key]), key
    assert np.array_equal(rep["q_final"], got["q_final"]) and np.array_equal(rep["dq_final"], got["dq_final"])


def test_threejoint_and_twojoint_are_gravity_free():
    """The convergence checks below run where g(q) is identically zero, so Sliding's +g (the reference's sign) does not
    enter: the planar arms move in the horizontal plane."""
    for arm in ("threejoint", "twojoint"):
        q, _, _, _ = cases.states(arm, 256)
        assert np.abs(rbd_oracle.ChainOracle(arm).g(q)).max() == 0.0, arm
    assert np.abs(rbd_oracle.ChainOracle("ur5").g(cases.states("ur5", 8)[0])).max() > 1.0


# constant-target convergence, calibrated on the oracle: (arm, controller, kwargs, steps, factor the error must fall by)
CONVERGE = {
    "joint_threejoint": ("threejoint", "joint", dict(kp=300, kv=20), 300, 10.0),
    "sliding_xy_twojoint": ("twojoint", "sliding", dict(kd=160.0, lamb=20.0), 300, 10.0),
}


def converge_inputs(arm, kind, B=8):
    """From rest, a constant target 0.4 rad (Joint) or 8 cm in the plane of the arm (Sliding) away"""
    q, _ = well_conditioned_starts(arm, B)
    rng = np.random.default_rng(cases.hash_name(arm + kind))
    if kind == "joint":
        d = rng.normal(size=q.shape)
        target = q + 0.4 * d / np.linalg.norm(d, axis=1, keepdims=True)
    else:
        x0 = rbd_oracle.ChainOracle(arm).Tx("EE", q)
        d = rng.normal(size=x0.shape)
        d[:, 2] = 0.0
        target = x0 + 0.08 * d / np.linalg.norm(d, axis=1, keepdims=True)
    return q, np.zeros_like(q), np.ascontiguousarray(target)


def tracking_error(kind, q, x, target):
    return np.linalg.norm(wrap(target - q) if kind == "joint" else x - target, axis=-1)


@pytest.mark.parametrize("name", list(CONVERGE))
def test_host_constant_target_error_falls(ctrlsim, name):
    """On a gravity-free arm the tracking error of a constant target falls by the stated factor over the horizon (on the
    oracle, over the same 300 steps: Joint by 19 at least, Sliding by 24 at least)."""
    arm, kind, kw, S, factor = CONVERGE[name]
    q, dq, target = converge_inputs(arm, kind)
    path = np.ascontiguousarray(np.broadcast_to(target[None], (S,) + target.shape))
    o = shim_rollout(ctrlsim, arm, kind, kw, q, dq, path, effort=0.0)
    x_end = rbd_oracle.ChainOracle(arm).Tx("EE", o["q_final"])
    e0 = tracking_error(kind, q, o["x"][0], target)
    e1 = tracking_error(kind, o["q_final"], x_end, target)
    print(name, "error start", e0.min(), "end", e1.max(), "min ratio", (e0 / e1).min())
    assert (e1 * factor < e0).all(), e0 / e1


# ---------------------------------------------------------------------------------------------- ABI checks
@pytest.fixture(scope="module")
def native():
    from abr_control_b200 import _lib

    lib = _lib.lib()
    cd = _desc("ur5")
    m = C.c_void_p()
    _lib.check(lib.abrb_model_create(C.byref(cd), C.byref(m)))
    buf = np.zeros(4096)
    yield lib, m, buf
    lib.abrb_model_destroy(m)


_JOINT_KEYS = ("m", "k1", "k2", "flag", "frame", "xoff", "q", "dq", "path", "ps", "pv", "pvs", "steps", "dt", "ew",
               "qt", "dqt", "ut", "xt", "cost", "B", "stream")
_SLIDING_KEYS = _JOINT_KEYS[:12] + ("pa", "pas") + _JOINT_KEYS[12:]


def _args(fn, **over):
    a = dict(m=None, k1=10.0, k2=3.0, flag=1, frame=0, xoff=None, q=None, dq=None, path=None, ps=0, pv=None, pvs=0,
             pa=None, pas=0, steps=4, dt=1e-3, ew=0.0, qt=None, dqt=None, ut=None, xt=None, cost=None, B=8, stream=None)
    a.update(over)
    return [a[k] for k in (_SLIDING_KEYS if "sliding" in fn else _JOINT_KEYS)]


ROLLOUT_FNS = ["abrb_joint_rollout_path_f64", "abrb_joint_rollout_path_f32", "abrb_sliding_rollout_path_f64",
               "abrb_sliding_rollout_path_f32"]


@pytest.mark.parametrize("fn", ROLLOUT_FNS)
def test_abi_rollout_rejects_bad_arguments_before_any_device_work(native, fn):
    lib, m, buf = native
    f = getattr(lib, fn)
    p = buf.ctypes.data
    ok = dict(m=m, q=p, dq=p, path=p)
    sliding = "sliding" in fn
    bad = [
        (dict(m=None), _abi.EINVAL, "model"),
        (dict(q=None), _abi.EINVAL, "NULL q"),
        (dict(dq=None), _abi.EINVAL, "NULL dq"),
        (dict(path=None), _abi.EINVAL, "NULL path"),
        (dict(ps=5), _abi.EINVAL, "path_stride"),
        (dict(ps=6 * 8), _abi.EINVAL, "path_stride"),
        (dict(pv=p, pvs=2), _abi.EINVAL, "pv_stride"),
        (dict(steps=-1), _abi.EINVAL, "steps"),
        (dict(B=-1), _abi.EINVAL, "B < 0"),
        (dict(ew=-1.0), _abi.EINVAL, "effort_weight"),
        (dict(ew=float("nan")), _abi.EINVAL, "effort_weight"),
        (dict(ew=float("inf")), _abi.EINVAL, "effort_weight"),
        (dict(q=p + 1), _abi.EINVAL, "misaligned pointer (q)"),
        (dict(dq=p + 1), _abi.EINVAL, "misaligned pointer (dq)"),
        (dict(path=p + 2), _abi.EINVAL, "misaligned pointer (path)"),
        (dict(pv=p + 2), _abi.EINVAL, "misaligned pointer (path_velocity)"),
        (dict(cost=p + 1), _abi.EINVAL, "misaligned pointer (cost)"),
        (dict(qt=p + 2), _abi.EINVAL, "misaligned pointer (q_traj)"),
        (dict(xt=p + 2), _abi.EINVAL, "misaligned pointer (x_traj)"),
        (dict(ut=p + 1), _abi.EINVAL, "misaligned pointer (u_traj)"),
        (dict(frame=99), _abi.EFRAME, "frame"),
        (dict(frame=-1), _abi.EFRAME, "frame"),
    ]
    if sliding:
        # cartesian (flag 1): rows of 3, so n_joints is a bad stride; joint mode (flag 0): rows of n, so 3 is
        bad += [(dict(ps=6), _abi.EINVAL, "path_stride"), (dict(flag=0, ps=3), _abi.EINVAL, "path_stride"),
                (dict(pa=p, pas=6), _abi.EINVAL, "pa_stride"), (dict(pa=p + 1), _abi.EINVAL, "misaligned pointer (path_acc)")]
    else:
        bad += [(dict(ps=3), _abi.EINVAL, "path_stride")]
    who = fn.rsplit("_", 1)[0]
    for over, code, word in bad:
        rc = f(*_args(fn, **{**ok, **over}))
        assert rc == code, (over, rc)
        msg = lib.abrb_last_error().decode()
        assert msg.startswith(who) and word in msg, (over, msg)
    # B == 0 is a no-op whatever the pointers
    assert f(*_args(fn, **{**ok, "B": 0, "q": None, "dq": None, "path": None})) == 0


def test_abi_valid_rollout_calls_without_a_device_fail_with_ecuda(native):
    lib, m, buf = native
    if lib.abrb_device_count() > 0:
        pytest.skip("a CUDA device is present")
    p = buf.ctypes.data
    for fn in ROLLOUT_FNS:
        stride = 3 if "sliding" in fn else 6
        assert getattr(lib, fn)(*_args(fn, m=m, q=p, dq=p, path=p, ps=stride, steps=3)) == _abi.ECUDA
        assert getattr(lib, fn)(*_args(fn, m=m, q=p, dq=p, steps=0, cost=p)) == _abi.ECUDA
    assert "no CUDA device" in lib.abrb_last_error().decode()


def test_signatures_and_header_cover_the_rollout_entry_points():
    from abr_control_b200 import _lib

    for fn in ROLLOUT_FNS:
        res, args = _lib.SIGNATURES[fn]
        sliding = "sliding" in fn
        assert res is C.c_int and len(args) == (24 if sliding else 22)
        assert args[1] is C.c_double and args[2] is C.c_double and args[3] is C.c_int and args[4] is C.c_int
        i = 14 if sliding else 12
        assert args[i] is C.c_int and args[i + 1] is C.c_double and args[i + 2] is C.c_double
        assert args[-2] is C.c_int64
    with open(os.path.join(ROOT, "include", "abrb.h")) as fh:
        hdr = fh.read()
    for fn in ROLLOUT_FNS:
        assert f"int {fn}(" in hdr


# ============================================================================================== GPU
def _cfg(arm, dtype=np.float64):
    import abr_control_b200.arms as arms
    from abr_control_b200.arms.base_config import BaseConfig

    if isinstance(arm, dict):
        return BaseConfig(arm, dtype=dtype)
    return getattr(arms, arm).Config(dtype=dtype)


def _ctrl(rc, kind, kw):
    from abr_control_b200 import controllers

    return controllers.Joint(rc, **kw) if kind == "joint" else controllers.Sliding(rc, **kw)


def _run(c, kind, q, dq, path, pv, pa, frame, off, **kw):
    if kind == "joint":
        return c.rollout_path(q, dq, path, path_velocity=pv, ref_frame=frame, xyz_offset=off, **kw)
    return c.rollout_path(q, dq, path, path_velocity=pv, path_acc=pa, ref_frame=frame, offset=off, **kw)


def _np(x):
    return x.cpu().numpy() if hasattr(x, "cpu") else np.asarray(x)


@pytest.mark.gpu
@pytest.mark.parametrize("variant", list(VARIANTS))
@pytest.mark.parametrize("arm", ARMS)
def test_device_rollout_vs_oracle(arm, variant):
    B = 24
    q, dq, path, pv, pa, kind, kw, frame, off = variant_inputs(arm, variant, B)
    ref = oracle_for(arm, variant, B)
    qf, dqf, tr, cost = _run(_ctrl(_cfg(arm), kind, kw), kind, q, dq, path, pv, pa, frame, off, dt=DT,
                             effort_weight=EFFORT)
    tp.assert_matches_oracle(dict(tr, cost=cost), ref, 0, f"{arm} {variant}")
    f = np.float32
    c = lambda a: None if a is None else a.astype(f)  # noqa: E731
    qf, dqf, tr, cost = _run(_ctrl(_cfg(arm, f), kind, kw), kind, q.astype(f), dq.astype(f), c(path), c(pv), c(pa),
                             frame, off, dt=DT, effort_weight=EFFORT)
    assert tr["u"].dtype == np.float32 and cost.dtype == np.float32
    tp.assert_matches_oracle(dict(tr, cost=cost), ref, 1, f"{arm} {variant} fp32")


@pytest.mark.gpu
@pytest.mark.parametrize("arm,variant", [("ur5", "joint_grav_per_vel"), ("jaco2", "joint_nograv_per"),
                                         ("ur5", "sliding_xyz_ee_per"), ("jaco2", "sliding_xyz_mid_offset_shared"),
                                         ("ur5", "sliding_joint_per")])
def test_device_recorded_torques_are_generate(arm, variant):
    """Every recorded u_t against the controller's generate at the recorded pre-step state and row t, relative 1e-12 in
    fp64.  Not required to be bit-identical: the two kernels may contract FMAs differently."""
    import torch

    B, S = 256, 16
    q, dq, path, pv, pa, kind, kw, frame, off = variant_inputs(arm, variant, 32, S=S)
    rep = lambda a: None if a is None else torch.as_tensor(  # noqa: E731
        np.tile(a, (1, B // 32, 1)) if a.ndim == 3 else a, device="cuda")
    tq, tdq = torch.as_tensor(np.tile(q, (B // 32, 1)), device="cuda"), torch.as_tensor(np.tile(dq, (B // 32, 1)),
                                                                                         device="cuda")
    tq = tq + 1e-3 * torch.randn_like(tq)
    P, PV, PA = rep(path), rep(pv), rep(pa)
    c = _ctrl(_cfg(arm), kind, kw)
    qf, dqf, tr, cost = _run(c, kind, tq, tdq, P, PV, PA, frame, off, dt=DT, effort_weight=EFFORT)
    qpre = torch.cat([tq[None], tr["q"][:-1]])
    dqpre = torch.cat([tdq[None], tr["dq"][:-1]])
    row = lambda a, t: None if a is None else (a[t] if a.dim() == 3 else a[t])  # noqa: E731
    worst = 0.0
    for t in range(S):
        if kind == "joint":
            u = c.generate(qpre[t], dqpre[t], row(P, t), target_velocity=row(PV, t))
        else:
            kws = dict(ref_frame=frame, offset=off) if _task(kind, kw) else {}
            u = c.generate(qpre[t], dqpre[t], row(P, t), target_velocity=0 if PV is None else row(PV, t),
                           target_acc=0 if PA is None else row(PA, t), **kws)
        rel = ((u - tr["u"][t]).abs().amax(1) / tr["u"][t].abs().amax(1).clamp_min(1.0)).max().item()
        worst = max(worst, rel)
    print(f"{arm} {variant}: recorded u vs generate, max rel {worst:.2e}")
    assert worst < 1e-12


def _straight_inputs(B, S, seed):
    """UR5 starts away from J[:3] singularities, a joint path (a ramp from the start) and a 5 cm task-space line"""
    import torch

    rc = _cfg("ur5")
    rng = np.random.default_rng(seed)
    pool = rng.uniform(0, 2 * np.pi, (2048, 6))
    pool = pool[_effective_cond(rbd_oracle.ChainOracle("ur5").J("EE", pool)[:, :3]) < 12]
    q = np.tile(pool, (B // len(pool) + 1, 1))[:B] + rng.uniform(-1e-2, 1e-2, (B, 6))
    q = torch.as_tensor(q, device="cuda")
    dq = torch.as_tensor(rng.uniform(-0.3, 0.3, (B, 6)), device="cuda")
    ramp = torch.linspace(0, 1, S, device="cuda", dtype=torch.float64)[:, None, None]
    jpath = (q[None] + ramp * torch.as_tensor(rng.normal(size=(B, 6)) * 0.3, device="cuda")[None]).contiguous()
    x0 = rc.Tx("EE", q)
    end = torch.as_tensor(rng.normal(size=(B, 3)), device="cuda")
    end = 0.05 * end / end.norm(dim=1, keepdim=True)
    xpath = (x0[None] + ramp * end[None]).contiguous()
    return rc, q, dq, jpath, xpath


CTRLS = {"joint": ("joint", dict(kp=300, kv=20)), "sliding": ("sliding", dict(kd=3.0, lamb=10.0))}


@pytest.mark.gpu
@pytest.mark.parametrize("which", list(CTRLS))
def test_device_replay_through_simulate(which):
    """traj["u"] through simulate from the same start (no path, same effort weight): u equal, q, dq, x within the bounds
    of test_plant's replay of OSC rollouts, at 4 096 x 128 UR5."""
    import torch

    B, S, ew = 4096, 128, 1e-4
    rc, q, dq, jpath, xpath = _straight_inputs(B, S, 5)
    kind, kw = CTRLS[which]
    c = _ctrl(rc, kind, kw)
    qf, dqf, tr, cost = _run(c, kind, q, dq, jpath if kind == "joint" else xpath, None, None, "EE", None, dt=DT,
                             effort_weight=ew)
    qs, dqs, ts, cs = rc.simulate(q, dq, tr["u"], dt=DT, effort_weight=ew)
    errs = dict(q=(ts["q"] - tr["q"]).abs().max().item(), dq=(ts["dq"] - tr["dq"]).abs().max().item(),
                x=(ts["x"] - tr["x"]).abs().max().item(), u=(ts["u"] - tr["u"]).abs().max().item())
    print(f"replay {which}: " + ", ".join(f"{k} {v:.2e}" for k, v in errs.items()))
    assert errs["u"] == 0.0
    assert errs["q"] < 1e-9 and errs["x"] < 1e-9 and errs["dq"] < 1e-7, errs
    assert torch.isfinite(cost).all()


@pytest.mark.gpu
@pytest.mark.parametrize("variant", ["joint_grav_per_vel", "sliding_xyz_ee_per", "sliding_joint_per"])
def test_layouts_permutation_and_zero_steps_are_bit_identical(variant):
    import torch

    B, S = 96, 16
    q, dq, path, pv, pa, kind, kw, frame, off = variant_inputs("ur5", variant, B, S=S)
    q, dq, path, pv, pa = (None if a is None else torch.as_tensor(a, device="cuda") for a in (q, dq, path, pv, pa))
    c = _ctrl(_cfg("ur5"), kind, kw)
    kwr = dict(dt=DT, effort_weight=1e-3)
    keys = ("q", "dq", "u", "x")
    # a shared (S, w) path (and velocity, acceleration) equals the same tiled to (S, B, w)
    sp = lambda a: None if a is None else a[:, 0].contiguous()  # noqa: E731
    tile = lambda a: None if a is None else a[:, None].expand(S, B, a.shape[-1]).contiguous()  # noqa: E731
    _, _, a, ca = _run(c, kind, q, dq, sp(path), sp(pv), sp(pa), frame, off, **kwr)
    _, _, b, cb = _run(c, kind, q, dq, tile(sp(path)), tile(sp(pv)), tile(sp(pa)), frame, off, **kwr)
    for k in keys:
        assert torch.equal(a[k], b[k]), k
    assert torch.equal(ca, cb)
    # permuting trajectories with their rows permutes every output
    qa, dqa, a, ca = _run(c, kind, q, dq, path, pv, pa, frame, off, **kwr)
    perm = torch.randperm(B, device="cuda")
    pm = lambda a: None if a is None else a[:, perm].contiguous()  # noqa: E731
    qp, dqp, p, cp = _run(c, kind, q[perm].contiguous(), dq[perm].contiguous(), pm(path), pm(pv), pm(pa), frame, off,
                          **kwr)
    for k in keys:
        assert torch.equal(p[k], a[k][:, perm]), k
    assert torch.equal(cp, ca[perm]) and torch.equal(qp, qa[perm]) and torch.equal(dqp, dqa[perm])
    # step indexing: changing row t0 of the path leaves every record before t0, and x_t0, alone
    t0 = 5
    p2 = path.clone()
    p2[t0] += 0.01
    _, _, c2, _ = _run(c, kind, q, dq, p2, pv, pa, frame, off, **kwr)
    for k in keys:
        assert torch.equal(c2[k][:t0], a[k][:t0]), k
    assert torch.equal(c2["x"][t0], a["x"][t0]) and not torch.equal(c2["u"][t0], a["u"][t0])
    # no steps: the start state, zero cost, empty records
    z = lambda a: None if a is None else a[:0]  # noqa: E731
    q0, dq0, tz, cz = _run(c, kind, q, dq, z(path), z(pv), z(pa), frame, off, **kwr)
    assert torch.equal(q0, q) and torch.equal(dq0, dq) and torch.equal(cz, torch.zeros_like(cz))
    assert tz["u"].shape == (0, B, 6) and tz["x"].shape == (0, B, 3)


@pytest.mark.gpu
@pytest.mark.parametrize("B,S", [(4096, 128), (140000, 8)])
@pytest.mark.parametrize("which", list(CTRLS))
def test_full_size_cost_only_equals_full_records(which, B, S):
    import torch

    rc, q, dq, jpath, xpath = _straight_inputs(B, S, B + S)
    kind, kw = CTRLS[which]
    c = _ctrl(rc, kind, kw)
    path = jpath if kind == "joint" else xpath
    qa, dqa, _, cost_only = _run(c, kind, q, dq, path, None, None, "EE", None, dt=DT, effort_weight=1e-4, record=())
    qb, dqb, tr, cost = _run(c, kind, q, dq, path, None, None, "EE", None, dt=DT, effort_weight=1e-4)
    # bit for bit, NaN where NaN: a Sliding loop on UR5 runs against the 2 g bias of the reference's +g, and on an H100
    # one of these 4 096 x 128 trajectories drifted into a singularity of J[:3] and diverged (the same in both calls)
    for x, y in ((cost_only, cost), (qa, qb), (dqa, dqb), (tr["q"][-1], qb)):
        torch.testing.assert_close(x, y, rtol=0, atol=0, equal_nan=True)
    finite = torch.isfinite(cost).double().mean().item()
    print(f"{which} {B}x{S}: finite costs {finite:.5f}")
    assert finite == 1.0 if kind == "joint" else finite > 0.999


@pytest.mark.gpu
def test_host_arrays_and_single_states_match_cuda_tensors():
    import torch

    for variant in ("joint_grav_per_vel", "sliding_xyz_ee_per"):
        B, S = 40, 10
        q, dq, path, pv, pa, kind, kw, frame, off = variant_inputs("ur5", variant, B, S=S)
        c = _ctrl(_cfg("ur5"), kind, kw)
        h = _run(c, kind, q, dq, path, pv, pa, frame, off, effort_weight=1e-3)
        t = lambda a: None if a is None else torch.as_tensor(a, device="cuda")  # noqa: E731
        d = _run(c, kind, t(q), t(dq), t(path), t(pv), t(pa), frame, off, effort_weight=1e-3)
        assert isinstance(h[0], np.ndarray) and isinstance(h[3], np.ndarray)
        assert np.array_equal(h[0], _np(d[0])) and np.array_equal(h[1], _np(d[1])) and np.array_equal(h[3], _np(d[3]))
        for k in ("q", "dq", "u", "x"):
            assert np.array_equal(h[2][k], _np(d[2][k])), k
        tq, tdq = t(q), t(dq)
        _run(c, kind, tq, tdq, t(path), t(pv), t(pa), frame, off)
        assert np.array_equal(_np(tq), q) and np.array_equal(_np(tdq), dq)  # the inputs are left alone
        one = lambda a: None if a is None else a[:, 0]  # noqa: E731
        s = _run(c, kind, q[0], dq[0], one(path), one(pv), one(pa), frame, off)
        b = _run(c, kind, q[:1], dq[:1], one(path), one(pv), one(pa), frame, off)
        assert s[0].shape == (6,) and s[2]["x"].shape == (S, 3) and np.ndim(s[3]) == 0
        assert np.array_equal(s[0], b[0][0]) and np.array_equal(s[2]["u"], b[2]["u"][:, 0]) and s[3] == b[3][0]
        with pytest.raises(ValueError):
            _run(c, kind, q, dq, path[:, :, :2], pv, pa, frame, off)
        with pytest.raises(ValueError):
            _run(c, kind, q, dq, path, None if pv is None else pv[:-1], pa, frame, off)
    sl = _ctrl(_cfg("ur5"), "sliding", dict(kd=8.0, lamb=20.0))
    sl.s = "untouched"
    _run(sl, "sliding", q, dq, path, pv, pa, frame, off)
    assert sl.s == "untouched"


@pytest.mark.gpu
def test_inverse_kinematics_pipeline():
    """generate_path for 1 024 UR5 starts, its position path (a view of one (S, B, n) buffer) into Joint.rollout_path,
    and every 64th trajectory against stepping generate, forward_dynamics and Euler through the public API."""
    import torch

    from abr_control_b200 import controllers
    from abr_control_b200.controllers.path_planners import inverse_kinematics

    rc = _cfg("ur5")
    B, S = 1024, 64
    rng = np.random.default_rng(21)
    q0 = torch.as_tensor(rng.uniform(0, 2 * np.pi, (B, 6)), device="cuda")
    x0 = rc.Tx("EE", q0)
    targets = torch.cat([x0 + torch.as_tensor(rng.uniform(-0.1, 0.1, (B, 3)), device="cuda"),
                         torch.as_tensor(rng.uniform(-np.pi, np.pi, (B, 3)), device="cuda")], 1).contiguous()
    ik = inverse_kinematics.InverseKinematics(rc)
    pos, _ = ik.generate_path(q0, targets, n_timesteps=S, dt=0.01)
    path = pos.permute(1, 0, 2)
    assert path.is_contiguous()
    j = controllers.Joint(rc, kp=300, kv=20)
    dq0 = torch.zeros_like(q0)
    qf, dqf, tr, cost = j.rollout_path(q0, dq0, path, dt=DT, effort_weight=1e-4)
    sel = torch.arange(0, B, 64, device="cuda")
    qs, dqs = q0[sel].clone(), dq0[sel].clone()
    cs = torch.zeros(len(sel), dtype=torch.float64, device="cuda")
    for t in range(S):
        p = path[t, sel].contiguous()
        u = j.generate(qs, dqs, p)
        d = (p - qs + np.pi) % (2 * np.pi) - np.pi
        cs += (d ** 2).sum(-1) + 1e-4 * (u ** 2).sum(-1)
        dqs = dqs + rc.forward_dynamics(qs, dqs, u) * DT
        qs = qs + dqs * DT
    eq, ec = (qf[sel] - qs).abs().max().item(), ((cost[sel] - cs).abs() / cs).max().item()
    print(f"IK pipeline {B}x{S}: stepped public API q {eq:.2e}, cost {ec:.2e}")
    assert eq < 1e-9 and ec < 1e-9


@pytest.mark.gpu
@pytest.mark.parametrize("ortho", [True, False])
@pytest.mark.parametrize("n", [1, 2, 3, 4, 5, 6, 7])
def test_random_chains_vs_oracle(n, ortho):
    """Joint and joint-mode Sliding on random chains of 1-7 joints, orthonormal and sheared frames, over 12 steps."""
    import test_generic_chains as gc

    desc = gc.random_chain(n, ortho, 300 + 10 * n + ortho)
    rng = np.random.default_rng(n + 77)
    B, S = 16, 12
    q, dq = rng.uniform(0, 2 * np.pi, (B, n)), rng.uniform(-1, 1, (B, n))
    path = q[None] + (np.arange(S) / S)[:, None, None] * rng.normal(size=(B, n))[None] * 0.3
    pv = rng.normal(size=(S, B, n)) * 0.2
    rc = _cfg(desc)
    for kind, kw in (("joint", dict(kp=100, kv=15)), ("sliding", dict(kd=5.0, lamb=10.0, cartesian=False))):
        ref = oracle_ctrl_rollout(desc, kind, kw, q, dq, path, DT, pv, None if kind == "joint" else pv, EFFORT)
        qf, dqf, tr, cost = _run(_ctrl(rc, kind, kw), kind, q, dq, path, pv, None if kind == "joint" else pv, "EE",
                                 None, dt=DT, effort_weight=EFFORT)
        tp.assert_matches_oracle(dict(tr, cost=cost), ref, 0, f"rand{n} {ortho} {kind}")
