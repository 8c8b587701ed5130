"""Path-following rollouts (``OSC.rollout_path``, ``abrb_osc_rollout_path_*``, ``rollout_kernel<..., RolloutPathArgs>``).

Semantics, for t = 0 .. S-1 (include/abrb.h):
    x_t = control point at q_t;  u_t = generate(q_t, dq_t, p_t, v_t);  ddq = M^-1 (u_t + g - C dq_t);
    dq_{t+1} = dq_t + ddq dt;  q_{t+1} = q_t + dq_{t+1} dt;  cost += |x_t - p_t[:3]|^2 + effort_weight |u_t|^2

CPU part: the NumPy stepping of that definition (``oracle_rollout_path``, on ``osc_oracle.OSC`` and
``rbd_oracle.ChainOracle``) against the stepped loop the fixed-target rollout tests write inline; the kernel's per-step
body (``rollout_step``) and path addressing (``path_row``), run on the host through tests/hostsim/pathsim.cpp (TEST
INFRASTRUCTURE, never loaded by the package), against that oracle; argument checking of the C entry points.
GPU part: the kernel against ``rollout``, against stepping the public API, against the oracle, indexing properties
and full-size runs.
"""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import cases
from abr_control_b200 import _abi
from oracle import osc_oracle as oo
from oracle import rbd_oracle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
T, F = True, False


# ---------------------------------------------------------------------------------------------- the definition
def oracle_rollout_path(arm, osc_kw, q, dq, path, dt, path_velocity=None, null=(), ref_frame="EE", xyz_offset=None,
                        effort_weight=0.0, ierr=None):
    """NumPy stepping of the path-following rollout, float64.  ``path`` / ``path_velocity``: (S, 6) shared or
    (S, B, 6) per trajectory.  ``ierr``: (B, 6) integrator start rows (ki != 0).
    -> dict(q, dq, u: (S, B, n); x: (S, B, 3); cost: (B,); q_final, dq_final; ierr: (B, 6) or None)"""
    q, dq = np.array(q, dtype=np.float64), np.array(dq, dtype=np.float64)
    B, n = q.shape
    S = path.shape[0]
    P = np.broadcast_to(path[:, None, :], (S, B, 6)) if path.ndim == 2 else path
    V = None
    if path_velocity is not None:
        V = np.broadcast_to(path_velocity[:, None, :], (S, B, 6)) if path_velocity.ndim == 2 else path_velocity
    ch = rbd_oracle.ChainOracle(arm)
    rc = oo.RobotOracle(arm, "fp64")
    refs = []
    for b in range(B):
        nulls = [oo.NULL_KINDS[k](rc, **kw) for k, kw in null] or None
        o = oo.OSC(rc, null_controllers=nulls, **osc_kw)
        if ierr is not None:
            o.err_sum = np.array(ierr[b], dtype=np.float64)
        refs.append(o)
    kw = {"ref_frame": ref_frame}
    xo = None if xyz_offset is None else np.asarray(xyz_offset, dtype=np.float64)
    if xo is not None:
        kw["xyz_offset"] = xo
    out = {k: np.zeros((S, B, 3 if k == "x" else n)) for k in ("q", "dq", "u", "x")}
    cost = np.zeros(B)
    for t in range(S):
        x = ch.Tx(ref_frame, q, xo)
        u = np.array([refs[b].generate(q[b], dq[b], np.array(P[t, b]),
                                       target_velocity=None if V is None else np.array(V[t, b]), **kw)
                      for b in range(B)])
        rhs = u + ch.g(q) - np.einsum("bij,bj->bi", ch.C(q, dq), dq)
        ddq = np.linalg.solve(ch.M(q), rhs[..., None])[..., 0]
        dq = dq + ddq * dt
        q = q + dq * dt
        cost += np.sum((x - P[t, :, :3]) ** 2, axis=1) + effort_weight * np.sum(u ** 2, axis=1)
        out["q"][t], out["dq"][t], out["u"][t], out["x"][t] = q, dq, u, x
    out.update(cost=cost, q_final=q, dq_final=dq,
               ierr=None if ierr is None else np.array([r.err_sum for r in refs]))
    return out


def smooth_path(arm, q, S, seed, per_trajectory=True, velocity=False):
    """A straight line from each start state's end effector (a shared path starts from trajectory 0's) towards a
    random point 0.1 away, a fixed random orientation; a velocity along the line with every fourth row all zero."""
    rng = np.random.default_rng(seed)
    ch = rbd_oracle.ChainOracle(arm)
    x0 = ch.Tx("EE", q)
    B = len(q)
    starts = x0 if per_trajectory else x0[:1]
    d = rng.normal(size=starts.shape)
    d *= 0.1 / np.linalg.norm(d, axis=1, keepdims=True)
    s = (np.arange(S) / S)[:, None, None]
    pos = starts[None] + s * d[None]                                        # (S, B', 3)
    ori = np.broadcast_to(rng.uniform(-np.pi, np.pi, (1, len(starts), 3)), pos.shape)
    path = np.concatenate([pos, ori], axis=2)
    vel = np.concatenate([np.broadcast_to(d[None] * 3.0, pos.shape), rng.uniform(-0.5, 0.5, pos.shape)], axis=2)
    vel[::4] = 0.0
    if not per_trajectory:
        path, vel = path[:, 0], vel[:, 0]
    path = np.ascontiguousarray(path)
    return path, (np.ascontiguousarray(vel) if velocity else None)


# the host-shim / oracle cases: (arm, OSC kwargs, secondary controllers, path velocity?)
CASES = {
    "ur5_xyz": ("ur5", dict(kp=10, use_C=True), (), False),
    "ur5_6dof_C_ki": ("ur5", dict(kp=10, ki=0.2, ctrlr_dof=[T] * 6, use_C=True), (), False),
    "jaco2_xyz_pv_damping": ("jaco2", dict(kp=20), (("Damping", dict(kv=5)),), True),
    "threejoint_cfg1": ("threejoint", dict(kp=20, use_C=True, ctrlr_dof=[T, T, F, F, F, F]),
                        (("Damping", dict(kv=10)),
                         ("RestingConfig", dict(kp=50, kv=float(np.sqrt(50)), rest_angles=[np.pi / 4, np.pi, None]))),
                        False),
}
STEPS, DT, EFFORT = 32, 1e-3, 1e-4


def case_inputs(name, B, per_trajectory, seed=0):
    arm, osc_kw, null, has_pv = CASES[name]
    q, dq, _, _ = cases.states(arm, B)
    dq = dq * 0.1
    path, pv = smooth_path(arm, q, STEPS, seed + len(name), per_trajectory, velocity=has_pv)
    ierr = np.random.default_rng(seed + 1).uniform(-0.05, 0.05, (B, 6)) if osc_kw.get("ki") else None
    return arm, osc_kw, null, q, dq, path, pv, ierr


_ORACLE = {}


def oracle_for(name, B, per_trajectory):
    key = (name, B, per_trajectory)
    if key not in _ORACLE:
        arm, osc_kw, null, q, dq, path, pv, ierr = case_inputs(name, B, per_trajectory)
        _ORACLE[key] = oracle_rollout_path(arm, osc_kw, q, dq, path, DT, pv, null=null, effort_weight=EFFORT, ierr=ierr)
    return _ORACLE[key]


# fp64 bounds of test_rollout_vs_oracle_stepped_loop (each step's u on the oracle's own state history); fp32 bounds of
# the fp32 parity tests, scaled by the row's magnitude
TOL = {0: dict(u=1e-6, q=1e-8, dq=1e-6, x=1e-8, cost=1e-8), 1: dict(u=2e-3, q=2e-4, dq=2e-2, x=2e-4, cost=2e-3)}


def assert_matches_oracle(got, ref, f32, what=""):
    tol = TOL[f32]
    S = ref["u"].shape[0]
    for t in range(S):
        assert np.abs(got["u"][t] - ref["u"][t]).max() < tol["u"] * max(1.0, np.abs(ref["u"][t]).max()), (what, "u", t)
        assert np.abs(got["q"][t] - ref["q"][t]).max() < tol["q"], (what, "q", t)
        assert np.abs(got["dq"][t] - ref["dq"][t]).max() < tol["dq"] * max(1.0, np.abs(ref["dq"][t]).max()), (what, "dq", t)
        assert np.abs(got["x"][t] - ref["x"][t]).max() < tol["x"], (what, "x", t)
    rel = np.abs(got["cost"] - ref["cost"]) / np.maximum(1e-12, np.abs(ref["cost"]))
    assert rel.max() < tol["cost"], (what, "cost", rel.max())


# ---------------------------------------------------------------------------------------------- 1. oracle
def test_oracle_constant_path_equals_stepped_loop():
    """A constant path without velocity is the fixed-target rollout: the inline loop of
    test_rollout_vs_oracle_stepped_loop, stepped here the same way; the cost is the sum of the oracle's own x and u."""
    osc_kw = dict(kp=10, ki=0.2, ctrlr_dof=[T] * 6, use_C=True)
    Bq, steps, dt = 8, 12, 1e-3
    q, dq, target, _ = cases.states("ur5", Bq)
    dq = dq * 0.1
    ch = rbd_oracle.ChainOracle("ur5")
    refs = [oo.OSC(oo.RobotOracle("ur5", "fp64"), **osc_kw) for _ in range(Bq)]
    qs, dqs = q.copy(), dq.copy()
    us, qt, dqt = [], [], []
    for t in range(steps):
        u = np.array([refs[b].generate(qs[b], dqs[b], target[b]) for b in range(Bq)])
        rhs = u + ch.g(qs) - np.einsum("bij,bj->bi", ch.C(qs, dqs), dqs)
        ddq = np.linalg.solve(ch.M(qs), rhs[..., None])[..., 0]
        dqs = dqs + ddq * dt
        qs = qs + dqs * dt
        us.append(u), qt.append(qs), dqt.append(dqs)
    path = np.ascontiguousarray(np.broadcast_to(target[None], (steps, Bq, 6)))
    o = oracle_rollout_path("ur5", osc_kw, q, dq, path, dt, effort_weight=0.01, ierr=np.zeros((Bq, 6)))
    assert np.array_equal(o["u"], np.array(us)) and np.array_equal(o["q"], np.array(qt))
    assert np.array_equal(o["dq"], np.array(dqt)) and np.array_equal(o["q_final"], qs)
    assert np.array_equal(o["ierr"], np.array([r.err_sum for r in refs]))
    # x_t is the state before step t
    xs = np.concatenate([ch.Tx("EE", q)[None], np.array([ch.Tx("EE", qq) for qq in qt[:-1]])])
    assert np.array_equal(o["x"], xs)
    cost = np.zeros(Bq)
    for t in range(steps):
        cost += np.sum((o["x"][t] - target[:, :3]) ** 2, axis=1) + 0.01 * np.sum(o["u"][t] ** 2, axis=1)
    assert np.array_equal(o["cost"], cost)


# ---------------------------------------------------------------------------------------------- 2. host shim
@pytest.fixture(scope="module")
def pathsim(tmp_path_factory):
    src = os.path.join(ROOT, "tests", "hostsim", "pathsim.cpp")
    so = str(tmp_path_factory.mktemp("pathsim") / "_pathsim.so")
    subprocess.run(["g++", "-O1", "-std=c++17", "-shared", "-fPIC", "-x", "c++", src, "-o", so], check=True)
    return C.CDLL(so)


def _p(a):
    return a.ctypes.data_as(C.c_void_p) if a is not None else None


def shim_rollout_path(ps, arm, osc_kw, null, q, dq, path, pv, ierr, f32=0, general=0, ref_frame="EE", xoff=None):
    cd = _abi.chain_desc_from_dict(_abi.load_arm_json(arm))
    n, B = cd.n_joints, len(q)
    p = _abi.osc_params(n, null=[_abi.null_params(k, n, **kw) for k, kw in null], **osc_kw)
    S = path.shape[0]
    q, dq = np.array(q, dtype=np.float64), np.array(dq, dtype=np.float64)
    out = {k: np.zeros((S, B, 3 if k == "x" else n)) for k in ("q", "dq", "u", "x")}
    cost = np.zeros(B)
    ie = None if ierr is None else np.array(ierr, dtype=np.float64)
    xo = None if xoff is None else (C.c_double * 3)(*xoff)
    picked = ps.ps_rollout_path(
        C.byref(cd), C.byref(p), f32, general, ps.hs_frame_id(n, ref_frame.encode()), xo, _p(q), _p(dq),
        _p(np.ascontiguousarray(path)), 6 if path.ndim == 3 else 0, _p(pv), 0 if pv is None or pv.ndim == 2 else 6,
        STEPS if S == STEPS else S, C.c_double(DT), C.c_double(EFFORT), _p(out["q"]), _p(out["dq"]), _p(out["u"]),
        _p(out["x"]), _p(cost), _p(ie), C.c_int64(B))
    assert picked in (0, 1)
    out.update(cost=cost, q_final=q, dq_final=dq, ierr=ie, plain=picked == 1)
    return out


# which instantiation rollout_path_go picks for each case
PLAIN = {"ur5_xyz": True, "ur5_6dof_C_ki": False, "jaco2_xyz_pv_damping": False, "threejoint_cfg1": False}


@pytest.mark.parametrize("layout", ["per_trajectory", "shared"])
@pytest.mark.parametrize("f32", [0, 1])
@pytest.mark.parametrize("name", list(CASES))
def test_host_step_vs_oracle(pathsim, name, f32, layout):
    B = 24
    per = layout == "per_trajectory"
    arm, osc_kw, null, q, dq, path, pv, ierr = case_inputs(name, B, per)
    ref = oracle_for(name, B, per)
    got = shim_rollout_path(pathsim, arm, osc_kw, null, q, dq, path, pv, ierr, f32=f32)
    assert got["plain"] == PLAIN[name]
    assert_matches_oracle(got, ref, f32, name)
    assert np.abs(got["q_final"] - ref["q_final"]).max() < TOL[f32]["q"]
    if ierr is not None:
        assert np.abs(got["ierr"] - ref["ierr"]).max() < 1e-9 * (1 if not f32 else 1e5)


def test_host_plain_matches_general_bit_for_bit(pathsim):
    """Without FMA contraction the plain instantiation of the step computes exactly what the general one does."""
    arm, osc_kw, null, q, dq, path, pv, ierr = case_inputs("ur5_xyz", 16, True)
    for f32 in (0, 1):
        a = shim_rollout_path(pathsim, arm, osc_kw, null, q, dq, path, pv, ierr, f32=f32)
        b = shim_rollout_path(pathsim, arm, osc_kw, null, q, dq, path, pv, ierr, f32=f32, general=1)
        assert a["plain"] and not b["plain"]
        for k in ("q", "dq", "u", "x", "cost"):
            assert np.array_equal(a[k], b[k]), k


def test_host_xyz_offset_and_frame(pathsim):
    """x_t is the control point of ref_frame + xyz_offset, and the cost is measured there."""
    arm, osc_kw = "ur5", dict(kp=10, use_C=True)
    q, dq, _, _ = cases.states(arm, 16)
    dq = dq * 0.1
    path, _ = smooth_path(arm, q, STEPS, 3)
    off = [0.02, -0.03, 0.05]
    for frame in ("EE", "link4"):
        got = shim_rollout_path(pathsim, arm, osc_kw, (), q, dq, path, None, None, ref_frame=frame, xoff=off)
        ref = oracle_rollout_path(arm, osc_kw, q, dq, path, DT, ref_frame=frame, xyz_offset=off, effort_weight=EFFORT)
        assert got["plain"] == (frame == "EE")
        assert_matches_oracle(got, ref, 0, frame)


# ---------------------------------------------------------------------------------------------- 3. ABI checks
def _abi_args(**over):
    a = dict(c=None, frame=0, xoff=None, q=None, dq=None, path=None, ps=0, pv=None, pvs=0, steps=4, dt=1e-3, ew=0.0,
             qt=None, dqt=None, ut=None, xt=None, cost=None, ie=None, B=8, stream=None)
    a.update(over)
    return [a[k] for k in ("c", "frame", "xoff", "q", "dq", "path", "ps", "pv", "pvs", "steps", "dt", "ew", "qt", "dqt",
                           "ut", "xt", "cost", "ie", "B", "stream")]


@pytest.fixture(scope="module")
def native():
    """A UR5 controller handle with ki == 0 and one with ki != 0, host buffers to point at."""
    from abr_control_b200 import _lib

    lib = _lib.lib()
    cd = _abi.chain_desc_from_dict(_abi.load_arm_json("ur5"))
    m = C.c_void_p()
    _lib.check(lib.abrb_model_create(C.byref(cd), C.byref(m)))
    hs = []
    for ki in (0.0, 0.3):
        p = _abi.osc_params(6, kp=10, ki=ki)
        h = C.c_void_p()
        _lib.check(lib.abrb_osc_create(m, C.byref(p), C.byref(h)))
        hs.append(h)
    buf = np.zeros(4096)
    yield lib, hs[0], hs[1], buf
    for h in hs:
        lib.abrb_osc_destroy(h)
    lib.abrb_model_destroy(m)


@pytest.mark.parametrize("fn", ["abrb_osc_rollout_path_f64", "abrb_osc_rollout_path_f32"])
def test_abi_rejects_bad_arguments_before_any_device_work(native, fn):
    lib, h, hki, buf = native
    f = getattr(lib, fn)
    p = buf.ctypes.data
    ok = dict(c=h, q=p, dq=p, path=p)
    bad = [
        (dict(c=None), _abi.EINVAL, "controller"),
        (dict(q=None), _abi.EINVAL, "NULL q"),
        (dict(dq=None), _abi.EINVAL, "NULL dq"),
        (dict(path=None), _abi.EINVAL, "path"),
        (dict(ps=3), _abi.EINVAL, "path_stride"),
        (dict(pvs=12, pv=p), _abi.EINVAL, "pv_stride"),
        (dict(steps=-1), _abi.EINVAL, "steps"),
        (dict(B=-1), _abi.EINVAL, "B < 0"),
        (dict(ew=-1.0), _abi.EINVAL, "effort_weight"),
        (dict(ew=float("nan")), _abi.EINVAL, "effort_weight"),
        (dict(ew=float("inf")), _abi.EINVAL, "effort_weight"),
        (dict(ie=p), _abi.EINVAL, "integrated_error"),
        (dict(c=hki), _abi.EINVAL, "integrated_error"),
        (dict(q=p + 1), _abi.EINVAL, "misaligned pointer (q)"),
        (dict(path=p + 2), _abi.EINVAL, "misaligned pointer (path)"),
        (dict(cost=p + 1), _abi.EINVAL, "misaligned pointer (cost)"),
        (dict(xt=p + 2), _abi.EINVAL, "misaligned pointer (x_traj)"),
        (dict(frame=99), _abi.EFRAME, "frame"),
        (dict(frame=-1), _abi.EFRAME, "frame"),
    ]
    for over, code, word in bad:
        rc = f(*_abi_args(**{**ok, **over}))
        assert rc == code, (over, rc)
        msg = lib.abrb_last_error().decode()
        assert msg.startswith("abrb_osc_rollout_path") and word in msg, (over, msg)
    # B == 0 is a no-op whatever the pointers; a NULL path is fine without steps
    assert f(*_abi_args(**{**ok, "B": 0, "q": None, "dq": None, "path": None})) == 0


def test_signatures_cover_the_new_entry_points():
    from abr_control_b200 import _lib

    for fn in ("abrb_osc_rollout_path_f64", "abrb_osc_rollout_path_f32"):
        res, args = _lib.SIGNATURES[fn]
        assert len(args) == 20 and args[11] is C.c_double and args[18] is C.c_int64
    with open(os.path.join(ROOT, "include", "abrb.h")) as fh:
        hdr = fh.read()
    assert "int abrb_osc_rollout_path_f64(" in hdr and "int abrb_osc_rollout_path_f32(" in hdr


# ============================================================================================== GPU
def _cfg(arm, dtype=np.float64):
    import abr_control_b200.arms as arms

    return getattr(arms, arm).Config(dtype=dtype)


def _ctrl(rc, osc_kw, null=()):
    from abr_control_b200 import controllers

    nulls = [getattr(controllers, k)(rc, **kw) for k, kw in null] or None
    return controllers.OSC(rc, null_controllers=nulls, **osc_kw)


def _np(x):
    return x.cpu().numpy() if hasattr(x, "cpu") else np.asarray(x)


# ---------------------------------------------------------------------------------------------- 4. = rollout
@pytest.mark.gpu
@pytest.mark.parametrize("osc_kw", [dict(kp=10, ctrlr_dof=[T] * 6, use_C=True), dict(kp=10)], ids=["plain", "general"])
def test_constant_path_reproduces_rollout(osc_kw):
    """A shared path whose every row is the target, no velocity: the same closed loop as rollout.  The records agree to
    1e-12 relative; where the compiler emitted the same arithmetic for both instantiations they are bit-identical."""
    import torch

    rc = _cfg("ur5")
    c = _ctrl(rc, osc_kw)
    q, dq, target, _ = cases.states("ur5", 96)
    q, dq = torch.as_tensor(q, device="cuda"), torch.as_tensor(0.1 * dq, device="cuda")
    tg = torch.as_tensor(target[0], device="cuda")
    S = 24
    qf, dqf, tr = c.rollout(q, dq, tg, steps=S, dt=DT)
    qg, dqg, tp, cost = c.rollout_path(q, dq, tg[None].expand(S, 6).contiguous(), dt=DT)
    for k in ("q", "dq", "u"):
        a, b = tr[k].double(), tp[k].double()
        rel = ((a - b).abs() / a.abs().clamp_min(1.0)).max().item()
        print(f"{osc_kw}: {k} max rel diff {rel:.2e}, bit-identical {torch.equal(a, b)}")
        assert rel <= 1e-12, (k, rel)
    assert torch.equal(qf, tr["q"][-1]) and torch.equal(qg, tp["q"][-1]) and torch.equal(dqg, tp["dq"][-1])
    assert torch.isfinite(cost).all()


# ---------------------------------------------------------------------------------------------- 5. = public API stepped
@pytest.mark.gpu
@pytest.mark.parametrize("offset", [None, [0.03, -0.02, 0.05]], ids=["no_offset", "offset"])
def test_per_step_semantics_vs_stepping_the_public_api(offset):
    rc = _cfg("ur5")
    c = _ctrl(rc, dict(kp=10))
    B, S = 64, 16
    q, dq, _, _ = cases.states("ur5", B)
    dq = 0.1 * dq
    path, pv = smooth_path("ur5", q, S, 11, per_trajectory=True, velocity=True)
    pv[:, ::5] = 0.0  # whole trajectories without velocity, besides every fourth step of every trajectory
    ew = 1e-3
    qf, dqf, tr, cost = c.rollout_path(q, dq, path, dt=DT, path_velocity=pv, xyz_offset=offset, effort_weight=ew)
    assert tr["x"].shape == (S, B, 3) and tr["u"].shape == (S, B, 6) and cost.shape == (B,)
    qs, dqs = q.copy(), dq.copy()
    for t in range(S):
        x = rc.Tx("EE", qs, x=offset)
        assert np.abs(tr["x"][t] - x).max() < 1e-12, t
        u = c.generate(qs, dqs, path[t], target_velocity=pv[t], xyz_offset=offset)
        d = rc.eval(qs, dqs, want=("M", "g", "C"))
        rhs = u + d["g"] - np.einsum("bij,bj->bi", d["C"], dqs)
        ddq = np.linalg.solve(d["M"], rhs[..., None])[..., 0]
        dqs = dqs + ddq * DT
        qs = qs + dqs * DT
        assert np.abs(tr["u"][t] - u).max() < 1e-7 * max(1.0, np.abs(u).max()), t
    assert np.abs(qf - qs).max() < 1e-9 and np.abs(dqf - dqs).max() < 1e-7
    ref = np.zeros(B)
    for t in range(S):
        ref += np.sum((tr["x"][t] - path[t, :, :3]) ** 2, axis=1) + ew * np.sum(tr["u"][t] ** 2, axis=1)
    assert (np.abs(cost - ref) / ref).max() <= 1e-12


# ---------------------------------------------------------------------------------------------- 6. = oracle
@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_device_vs_oracle(name):
    B = 48
    per = name != "ur5_6dof_C_ki"  # one case on a shared path
    arm, osc_kw, null, q, dq, path, pv, ierr = case_inputs(name, B, per)
    ref = oracle_for(name, B, per)
    rc = _cfg(arm)
    c = _ctrl(rc, osc_kw, null)
    buf = None
    if ierr is not None:  # the rollout starts from the controller's (B, 6) integrator rows of CUDA calls
        import torch

        c.generate(*(torch.as_tensor(a, device="cuda") for a in (q, dq, path[0])))
        buf = next(iter(c.integrated_error_batch.values()))
        buf.copy_(torch.as_tensor(ierr, device="cuda"))
    qf, dqf, tr, cost = c.rollout_path(q, dq, path, dt=DT, path_velocity=pv, effort_weight=EFFORT)
    assert_matches_oracle(dict(tr, cost=cost), ref, 0, name)
    if buf is not None:
        assert np.abs(buf.cpu().numpy() - ref["ierr"]).max() < 1e-9


@pytest.mark.gpu
def test_device_fp32_jaco2_vs_oracle():
    B = 48
    arm, osc_kw, null, q, dq, path, pv, ierr = case_inputs("jaco2_xyz_pv_damping", B, True)
    ref = oracle_for("jaco2_xyz_pv_damping", B, True)
    c = _ctrl(_cfg(arm, np.float32), osc_kw, null)
    f = np.float32
    qf, dqf, tr, cost = c.rollout_path(q.astype(f), dq.astype(f), path.astype(f), dt=DT, path_velocity=pv.astype(f),
                                       effort_weight=EFFORT)
    assert tr["u"].dtype == np.float32 and cost.dtype == np.float32
    assert_matches_oracle(dict(tr, cost=cost), ref, 1, "jaco2 fp32")


# ---------------------------------------------------------------------------------------------- 7. indexing
@pytest.mark.gpu
def test_step_indexing_trajectory_permutation_and_shared_layout():
    import torch

    rc = _cfg("ur5")
    c = _ctrl(rc, dict(kp=10))
    B, S, t0 = 80, 12, 5
    q, dq, _, _ = cases.states("ur5", B)
    q, dq = torch.as_tensor(q, device="cuda"), torch.as_tensor(0.1 * dq, device="cuda")
    path, pv = smooth_path("ur5", q.cpu().numpy(), S, 21, per_trajectory=True, velocity=True)
    path, pv = torch.as_tensor(path, device="cuda"), torch.as_tensor(pv, device="cuda")
    kw = dict(dt=DT, path_velocity=pv, effort_weight=1e-3)
    _, _, a, ca = c.rollout_path(q, dq, path, **kw)
    p2 = path.clone()
    p2[t0, :, :3] += 0.05
    _, _, b, cb = c.rollout_path(q, dq, p2, **kw)
    for k in ("q", "dq", "u", "x"):
        assert torch.equal(a[k][:t0], b[k][:t0]), k
    # u_t, q_{t+1}, dq_{t+1} of step t0 see the changed row; x_{t0} is the state before it
    for k in ("q", "dq", "u"):
        assert (a[k][t0] != b[k][t0]).any(dim=-1).all(), k
    assert torch.equal(a["x"][t0], b["x"][t0]) and (a["x"][t0 + 1] != b["x"][t0 + 1]).any(dim=-1).all()
    assert (ca != cb).all()
    # permuting trajectories together with their path and velocity columns permutes every output
    perm = torch.randperm(B, device="cuda")
    qp, dqp, tp, cp = c.rollout_path(q[perm].contiguous(), dq[perm].contiguous(), path[:, perm].contiguous(), dt=DT,
                                     path_velocity=pv[:, perm].contiguous(), effort_weight=1e-3)
    for k in ("q", "dq", "u", "x"):
        assert torch.equal(tp[k], a[k][:, perm]), k
    assert torch.equal(cp, ca[perm])
    # a shared path and velocity equal the same tiled to (S, B, 6), bit for bit
    sp, sv = path[:, 0].contiguous(), pv[:, 0].contiguous()
    _, _, s1, c1 = c.rollout_path(q, dq, sp, dt=DT, path_velocity=sv)
    _, _, s2, c2 = c.rollout_path(q, dq, sp[:, None].expand(S, B, 6).contiguous(), dt=DT,
                                  path_velocity=sv[:, None].expand(S, B, 6).contiguous())
    for k in ("q", "dq", "u", "x"):
        assert torch.equal(s1[k], s2[k]), k
    assert torch.equal(c1, c2)
    # no steps: the state is left as it is, the cost is zero
    q0, dq0, tz, cz = c.rollout_path(q, dq, path[:0], dt=DT)
    assert torch.equal(q0, q) and torch.equal(dq0, dq) and tz["u"].shape == (0, B, 6) and torch.equal(cz, torch.zeros_like(cz))


# ---------------------------------------------------------------------------------------------- 8. full size
def _stepped_reference(rc, osc_kw, q, dq, path, pv, ew, steps):
    """Batched stepping of the public API (generate + eval + solve + Euler) on the device, float64."""
    import torch

    c = _ctrl(rc, osc_kw)
    q, dq = q.clone(), dq.clone()
    us, xs, cost = [], [], torch.zeros(q.shape[0], dtype=q.dtype, device=q.device)
    for t in range(steps):
        x = rc.Tx("EE", q)
        u = c.generate(q, dq, path[t], target_velocity=None if pv is None else pv[t])
        d = rc.eval(q, dq, want=("M", "g", "C"))
        ddq = torch.linalg.solve(d["M"], (u + d["g"] - torch.bmm(d["C"], dq[..., None])[..., 0])[..., None])[..., 0]
        dq = dq + ddq * DT
        q = q + dq * DT
        cost += ((x - path[t][..., :3]) ** 2).sum(-1) + ew * (u ** 2).sum(-1)
        us.append(u), xs.append(x)
    ie = next(iter(c.integrated_error_batch.values())) if c.ki != 0 else None
    return q, dq, torch.stack(us), torch.stack(xs), cost, ie


@pytest.mark.gpu
@pytest.mark.parametrize("B,S,osc_kw", [(4096, 128, dict(kp=10)), (140000, 8, dict(kp=10, ctrlr_dof=[T] * 6, use_C=True)),
                                         (4096, 32, dict(kp=10, ki=0.3, ctrlr_dof=[T] * 6, use_C=True))],
                         ids=["cfg4_4096x128", "plain_140000x8", "ki_4096x32"])
def test_full_size_cost_only_and_stepped_reference(B, S, osc_kw):
    import torch

    rc = _cfg("ur5")
    rng = np.random.default_rng(B + S)
    q = torch.as_tensor(rng.uniform(0, 2 * np.pi, (B, 6)), device="cuda")
    dq = torch.as_tensor(rng.uniform(-0.5, 0.5, (B, 6)), device="cuda")
    x0 = rc.Tx("EE", q)
    ramp = torch.linspace(0, 1, S, device="cuda", dtype=torch.float64)[:, None, None]
    end = torch.as_tensor(rng.uniform(-0.1, 0.1, (B, 3)), device="cuda")
    path = torch.cat([x0[None] + ramp * end[None], torch.as_tensor(rng.uniform(-1, 1, (1, B, 3)), device="cuda").expand(S, B, 3)], -1)
    path = path.contiguous()
    ew = 1e-4
    c1, c2 = _ctrl(rc, osc_kw), _ctrl(rc, osc_kw)
    qa, dqa, _, cost_only = c1.rollout_path(q, dq, path, dt=DT, record=(), effort_weight=ew)
    qb, dqb, tr, cost = c2.rollout_path(q, dq, path, dt=DT, effort_weight=ew)
    assert torch.equal(cost_only, cost) and torch.equal(qa, qb) and torch.equal(dqa, dqb)
    sel = torch.arange(0, B, 64, device="cuda")
    qs, dqs, us, xs, cs, ie = _stepped_reference(rc, osc_kw, q[sel].contiguous(), dq[sel].contiguous(),
                                                 path[:, sel].contiguous(), None, ew, S)
    err_u = ((tr["u"][:, sel] - us).abs().amax(-1) / us.abs().amax(-1).clamp_min(1.0)).max().item()
    err_x = (tr["x"][:, sel] - xs).abs().max().item()
    err_q, err_dq = (qb[sel] - qs).abs().max().item(), (dqb[sel] - dqs).abs().max().item()
    err_c = ((cost[sel] - cs).abs() / cs).max().item()
    print(f"{B}x{S} {osc_kw}: u {err_u:.2e} x {err_x:.2e} q {err_q:.2e} dq {err_dq:.2e} cost {err_c:.2e}")
    assert err_u < 1e-6 and err_x < 1e-8 and err_q < 1e-8 and err_dq < 1e-6 and err_c < 1e-8
    if ie is not None:
        mine = next(iter(c2.integrated_error_batch.values()))
        assert (mine[sel] - ie).abs().max().item() < 1e-9
        assert torch.equal(mine, next(iter(c1.integrated_error_batch.values())))


# ---------------------------------------------------------------------------------------------- 9. input forms
@pytest.mark.gpu
def test_host_arrays_and_single_state_match_cuda_tensors():
    import torch

    rc = _cfg("ur5")
    c = _ctrl(rc, dict(kp=10))
    B, S = 40, 10
    q, dq, _, _ = cases.states("ur5", B)
    dq = 0.1 * dq
    path, pv = smooth_path("ur5", q, S, 31, per_trajectory=True, velocity=True)
    h = c.rollout_path(q, dq, path, dt=DT, path_velocity=pv, effort_weight=1e-3)
    d = c.rollout_path(*(torch.as_tensor(a, device="cuda") for a in (q, dq, path)), dt=DT,
                       path_velocity=torch.as_tensor(pv, device="cuda"), effort_weight=1e-3)
    assert isinstance(h[0], np.ndarray) and isinstance(h[3], np.ndarray)
    assert np.array_equal(h[0], _np(d[0])) and np.array_equal(h[1], _np(d[1])) and np.array_equal(h[3], _np(d[3]))
    for k in ("q", "dq", "u", "x"):
        assert np.array_equal(h[2][k], _np(d[2][k])), k
    # one state with an (S, 6) path equals row 0 of the batched call with the same path shared
    s = c.rollout_path(q[0], dq[0], path[:, 0], dt=DT, path_velocity=pv[:, 0])
    b = c.rollout_path(q[:1], dq[:1], path[:, 0], dt=DT, path_velocity=pv[:, 0])
    assert s[0].shape == (6,) and s[2]["x"].shape == (S, 3) and np.ndim(s[3]) == 0
    assert np.array_equal(s[0], b[0][0]) and np.array_equal(s[2]["u"], b[2]["u"][:, 0]) and s[3] == b[3][0]
