"""The plant on its own: forward and inverse dynamics and open-loop plant rollouts (``BaseConfig.forward_dynamics``,
``inverse_dynamics``, ``simulate``; ``abrb_forward_dynamics_*``, ``abrb_inverse_dynamics_*``, ``abrb_plant_rollout_*``).

Semantics (include/abrb.h):
    forward   ddq = M^-1 (u + g - C dq)          inverse   u = M ddq + C dq - g
    rollout   tau_t = u_t (or u_t - g(q_t));  x_t = control point at q_t;  ddq = M^-1 (tau_t + g - C dq_t);
              dq_{t+1} = dq_t + ddq dt;  q_{t+1} = q_t + dq_{t+1} dt;  cost += |x_t - p_t[:3]|^2 + w |tau_t|^2

CPU part: the NumPy definition (``oracle_simulate``, on ``rbd_oracle.ChainOracle``) against the kernels' per-state code
run on the host through tests/hostsim/plantsim.cpp (TEST INFRASTRUCTURE, never loaded by the package); the replay of a
closed-loop rollout's torques (tests/hostsim/pathsim.cpp) bit for bit; the round trip; the energy balance; argument
checking of the C entry points.
GPU part: the kernels against the oracle, the replay of ``OSC.rollout_path`` / ``OSC.rollout``, the single-step
dynamics against ``eval`` + solve, layout and indexing properties, full-size runs and the input forms.
"""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import cases
from abr_control_b200 import _abi
from oracle import rbd_oracle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
T, F = True, False
ARMS = ("ur5", "jaco2", "threejoint", "twojoint")
STEPS, DT, EFFORT = 24, 1e-3, 1e-4


# ---------------------------------------------------------------------------------------------- the definition
def oracle_simulate(arm, q, dq, u, dt, path=None, effort_weight=0.0, compensate_gravity=False, ref_frame="EE",
                    xyz_offset=None):
    """NumPy stepping of the plant rollout, float64.  ``u``: (S, n) shared or (S, B, n); ``path``: None, (S, 6) or
    (S, B, 6).  -> dict(q, dq, u (the applied tau), x: (S, B, .); cost: (B,); q_final, dq_final)"""
    q, dq = np.array(q, dtype=np.float64), np.array(dq, dtype=np.float64)
    B, n = q.shape
    S = u.shape[0]
    U = np.broadcast_to(u[:, None, :], (S, B, n)) if u.ndim == 2 else u
    P = None if path is None else (np.broadcast_to(path[:, None, :], (S, B, 6)) if path.ndim == 2 else path)
    ch = rbd_oracle.ChainOracle(arm)
    xo = None if xyz_offset is None else np.asarray(xyz_offset, dtype=np.float64)
    out = {k: np.zeros((S, B, 3 if k == "x" else n)) for k in ("q", "dq", "u", "x")}
    cost = np.zeros(B)
    for t in range(S):
        x = ch.Tx(ref_frame, q, xo)
        g = ch.g(q)
        tau = U[t] - g if compensate_gravity else np.array(U[t])
        rhs = tau + g - np.einsum("bij,bj->bi", ch.C(q, dq), dq)
        ddq = np.linalg.solve(ch.M(q), rhs[..., None])[..., 0]
        dq = dq + ddq * dt
        q = q + dq * dt
        if P is not None:
            cost += np.sum((x - P[t, :, :3]) ** 2, axis=1)
        cost += effort_weight * np.sum(tau ** 2, axis=1)
        out["q"][t], out["dq"][t], out["u"][t], out["x"][t] = q, dq, tau, x
    out.update(cost=cost, q_final=q, dq_final=dq)
    return out


def oracle_forward(arm, q, dq, u):
    ch = rbd_oracle.ChainOracle(arm)
    rhs = u + ch.g(q) - np.einsum("bij,bj->bi", ch.C(q, dq), dq)
    return np.linalg.solve(ch.M(q), rhs[..., None])[..., 0]


def oracle_inverse(arm, q, dq, ddq):
    ch = rbd_oracle.ChainOracle(arm)
    return np.einsum("bij,bj->bi", ch.M(q), ddq) + np.einsum("bij,bj->bi", ch.C(q, dq), dq) - ch.g(q)


# the rollout variants of the host and device checks: (torque layout, path layout, compensate_gravity, frame, offset)
VARIANTS = {
    "per_u_no_path": ("per", None, F, "EE", None),
    "shared_u_shared_path_comp": ("shared", "shared", T, "EE", None),
    "per_u_per_path_offset_frame": ("per", "per", F, "mid", [0.02, -0.03, 0.05]),
    "shared_u_per_path_comp_offset": ("shared", "per", T, "EE", [0.01, 0.02, -0.04]),
}


def variant_inputs(arm, variant, B, S=STEPS, seed=0):
    """Start states (dq scaled down), a torque sequence about the start's gravity hold (or residual torques with
    compensation), a straight-line path from the start's control point."""
    ulay, play, comp, frame, off = VARIANTS[variant]
    frame = cases.ARMS[arm]["mid"] if frame == "mid" else frame
    q, dq, _, _ = cases.states(arm, B)
    dq = 0.2 * dq
    n = q.shape[1]
    rng = np.random.default_rng(seed + cases.hash_name(arm + variant))
    ch = rbd_oracle.ChainOracle(arm)
    hold = np.zeros((B, n)) if comp else -ch.g(q)
    scale = 1.0 + 0.1 * np.abs(hold).max()
    if ulay == "per":
        u = hold[None] + scale * rng.normal(size=(S, B, n))
    else:
        u = hold[0][None] + scale * rng.normal(size=(S, n))
    path = None
    if play is not None:
        x0 = ch.Tx(frame, q, off)
        starts = x0 if play == "per" else x0[:1]
        d = rng.normal(size=starts.shape)
        d *= 0.05 / np.linalg.norm(d, axis=1, keepdims=True)
        s = (np.arange(S) / S)[:, None, None]
        pos = starts[None] + s * d[None]
        path = np.concatenate([pos, rng.uniform(-np.pi, np.pi, pos.shape)], axis=2)
        if play == "shared":
            path = path[:, 0]
        path = np.ascontiguousarray(path)
    return q, dq, np.ascontiguousarray(u), path, comp, frame, off


_ORACLE = {}


def oracle_for(arm, variant, B):
    key = (arm, variant, B)
    if key not in _ORACLE:
        q, dq, u, path, comp, frame, off = variant_inputs(arm, variant, B)
        _ORACLE[key] = oracle_simulate(arm, q, dq, u, DT, path, EFFORT, comp, frame, off)
    return _ORACLE[key]


# fp64 bounds of test_rollout_path.TOL (u: the applied torque, relative to its row's magnitude); fp32 bounds likewise
TOL = {0: dict(u=1e-9, q=1e-8, dq=1e-6, x=1e-8, cost=1e-8), 1: dict(u=2e-3, q=2e-4, dq=2e-2, x=2e-4, cost=2e-3)}


def assert_matches_oracle(got, ref, f32, what=""):
    tol = TOL[f32]
    for t in range(ref["u"].shape[0]):
        assert np.abs(got["u"][t] - ref["u"][t]).max() < tol["u"] * max(1.0, np.abs(ref["u"][t]).max()), (what, "u", t)
        assert np.abs(got["q"][t] - ref["q"][t]).max() < tol["q"], (what, "q", t)
        assert np.abs(got["dq"][t] - ref["dq"][t]).max() < tol["dq"] * max(1.0, np.abs(ref["dq"][t]).max()), (what, "dq", t)
        assert np.abs(got["x"][t] - ref["x"][t]).max() < tol["x"], (what, "x", t)
    rel = np.abs(got["cost"] - ref["cost"]) / np.maximum(1e-12, np.abs(ref["cost"]))
    assert rel.max() < tol["cost"], (what, "cost", rel.max())


def test_oracle_matches_its_own_terms():
    """One step of the oracle by hand: tau, x before the update, the Euler order, the cost with and without a path."""
    q, dq, u, path, _, _, _ = variant_inputs("ur5", "per_u_per_path_offset_frame", 4, S=1)
    ch = rbd_oracle.ChainOracle("ur5")
    o = oracle_simulate("ur5", q, dq, u, 0.01, path, 0.5, True, "link3", [0.1, 0, 0])
    g = ch.g(q)
    ddq = oracle_forward("ur5", q, dq, u[0] - g)
    assert np.array_equal(o["u"][0], u[0] - g) and np.allclose(o["dq"][0], dq + 0.01 * ddq, rtol=0, atol=1e-12)
    assert np.allclose(o["q"][0], q + 0.01 * o["dq"][0], rtol=0, atol=1e-15)
    x = ch.Tx("link3", q, [0.1, 0, 0])
    assert np.array_equal(o["x"][0], x)
    assert np.allclose(o["cost"], np.sum((x - path[0, :, :3]) ** 2, 1) + 0.5 * np.sum((u[0] - g) ** 2, 1), rtol=1e-14)
    o2 = oracle_simulate("ur5", q, dq, u, 0.01, None, 0.5)
    assert np.allclose(o2["cost"], 0.5 * np.sum(u[0] ** 2, 1), rtol=1e-14)


# ---------------------------------------------------------------------------------------------- host shims
def _build(tmp_path_factory, name):
    src = os.path.join(ROOT, "tests", "hostsim", f"{name}.cpp")
    so = str(tmp_path_factory.mktemp(name) / f"_{name}.so")
    subprocess.run(["g++", "-O1", "-std=c++17", "-shared", "-fPIC", "-x", "c++", src, "-o", so], check=True)
    return C.CDLL(so)


@pytest.fixture(scope="module")
def plantsim(tmp_path_factory):
    return _build(tmp_path_factory, "plantsim")


@pytest.fixture(scope="module")
def pathsim(tmp_path_factory):
    return _build(tmp_path_factory, "pathsim")


def _p(a):
    return a.ctypes.data_as(C.c_void_p) if a is not None else None


def _desc(arm):
    return _abi.chain_desc_from_dict(_abi.load_arm_json(arm))


def shim_simulate(ps, arm, q, dq, u, path, comp, frame="EE", xoff=None, f32=0, dt=DT, effort=EFFORT):
    cd = _desc(arm)
    n, B = cd.n_joints, len(q)
    S = u.shape[0]
    q, dq = np.array(q, dtype=np.float64), np.array(dq, dtype=np.float64)
    out = {k: np.zeros((S, B, 3 if k == "x" else n)) for k in ("q", "dq", "u", "x")}
    cost = np.zeros(B)
    xo = None if xoff is None else (C.c_double * 3)(*xoff)
    rc = ps.pl_rollout(C.byref(cd), f32, ps.hs_frame_id(n, frame.encode()), xo, _p(q), _p(dq),
                       _p(np.ascontiguousarray(u, dtype=np.float64)), n if u.ndim == 3 else 0, int(comp),
                       _p(None if path is None else np.ascontiguousarray(path, dtype=np.float64)),
                       0 if path is None or path.ndim == 2 else 6, S, C.c_double(dt), C.c_double(effort), _p(out["q"]),
                       _p(out["dq"]), _p(out["u"]), _p(out["x"]), _p(cost), C.c_int64(B))
    assert rc == 0
    out.update(cost=cost, q_final=q, dq_final=dq)
    return out


def shim_dynamics(ps, arm, kind, q, dq, x, f32=0):
    cd = _desc(arm)
    q, dq, x = (np.ascontiguousarray(a, dtype=np.float64) for a in (q, dq, x))
    out = np.zeros_like(q)
    assert ps.pl_dynamics(C.byref(cd), f32, kind, _p(q), _p(dq), _p(x), C.c_int64(len(q)), _p(out)) == 0
    return out


@pytest.mark.parametrize("f32", [0, 1])
@pytest.mark.parametrize("variant", list(VARIANTS))
@pytest.mark.parametrize("arm", ARMS)
def test_host_rollout_vs_oracle(plantsim, arm, variant, f32):
    B = 12
    q, dq, u, path, comp, frame, off = variant_inputs(arm, variant, B)
    ref = oracle_for(arm, variant, B)
    got = shim_simulate(plantsim, arm, q, dq, u, path, comp, frame, off, f32=f32)
    assert_matches_oracle(got, ref, f32, f"{arm} {variant}")
    assert np.abs(got["q_final"] - ref["q_final"]).max() < TOL[f32]["q"]


@pytest.mark.parametrize("f32", [0, 1])
@pytest.mark.parametrize("arm", ARMS)
def test_host_dynamics_vs_oracle(plantsim, arm, f32):
    """Forward and inverse dynamics against M, g, C of the oracle (fp64: 1e-9 relative to the row; fp32: 2e-3)."""
    q, dq, _, _ = cases.states(arm, 24)
    rng = np.random.default_rng(7)
    u = rng.normal(size=q.shape) * 5
    a = rng.normal(size=q.shape) * 3
    tol = 2e-3 if f32 else 1e-9
    ddq = shim_dynamics(plantsim, arm, 0, q, dq, u, f32)
    ref = oracle_forward(arm, q, dq, u)
    assert (np.abs(ddq - ref).max(1) / np.maximum(1.0, np.abs(ref).max(1))).max() < tol * (30 if f32 else 1)
    uu = shim_dynamics(plantsim, arm, 1, q, dq, a, f32)
    ref = oracle_inverse(arm, q, dq, a)
    assert (np.abs(uu - ref).max(1) / np.maximum(1.0, np.abs(ref).max(1))).max() < tol


# the closed-loop cases whose torques are replayed: (arm, OSC kwargs, secondary controllers, general instantiation?)
REPLAY = {
    "ur5_plain": ("ur5", dict(kp=10, ctrlr_dof=[T] * 6, use_C=True), (), 0),
    "ur5_general": ("ur5", dict(kp=10, ctrlr_dof=[T] * 6, use_C=True), (), 1),
    "jaco2_xyz_damping": ("jaco2", dict(kp=20), (("Damping", dict(kv=5)),), 0),
}


@pytest.mark.parametrize("f32", [0, 1])
@pytest.mark.parametrize("name", list(REPLAY))
def test_host_replay_of_closed_loop_torques_is_bit_identical(plantsim, pathsim, name, f32):
    """The u_traj of a path-following OSC rollout (rollout_step, pathsim.cpp), fed into the plant rollout from the same
    state with the same path and effort weight, reproduces the closed loop's q, dq, x and cost exactly: the plant of
    both is the same sequence of operations, and the host compiler contracts nothing into FMAs."""
    arm, osc_kw, null, general = REPLAY[name]
    cd = _desc(arm)
    n, B, S = cd.n_joints, 10, STEPS
    q, dq, _, _ = cases.states(arm, B)
    dq = 0.2 * dq
    q, dq = np.array(q), np.array(dq)
    _, _, _, path, _, _, _ = variant_inputs(arm, "shared_u_per_path_comp_offset", B)  # a path near the EE
    p =_abi.osc_params(n, null=[_abi.null_params(k, n, **kw) for k, kw in null], **osc_kw)
    cl = {k: np.zeros((S, B, 3 if k == "x" else n)) for k in ("q", "dq", "u", "x")}
    ccost = np.zeros(B)
    qc, dqc = q.copy(), dq.copy()
    picked = pathsim.ps_rollout_path(C.byref(cd), C.byref(p), f32, general, pathsim.hs_frame_id(n, b"EE"), None, _p(qc),
                                     _p(dqc), _p(path), 6, None, 0, S, C.c_double(DT), C.c_double(EFFORT), _p(cl["q"]),
                                     _p(cl["dq"]), _p(cl["u"]), _p(cl["x"]), _p(ccost), None, C.c_int64(B))
    assert picked == (1 if name == "ur5_plain" else 0)
    got = shim_simulate(plantsim, arm, q, dq, cl["u"], path, False, f32=f32)
    for k in ("q", "dq", "u", "x"):
        assert np.array_equal(got[k], cl[k]), k
    assert np.array_equal(got["cost"], ccost) and np.array_equal(got["q_final"], qc) and np.array_equal(got["dq_final"], dqc)


@pytest.mark.parametrize("f32", [0, 1])
@pytest.mark.parametrize("arm", ARMS)
def test_host_round_trip(plantsim, arm, f32):
    """forward_dynamics(q, dq, inverse_dynamics(q, dq, a)) == a to within cond(M) times the precision's epsilon
    (times 50 for the solve's and the products' rounding)."""
    q, dq, _, _ = cases.states(arm, 24)
    a = np.random.default_rng(3).normal(size=q.shape) * 4
    u = shim_dynamics(plantsim, arm, 1, q, dq, a, f32)
    back = shim_dynamics(plantsim, arm, 0, q, dq, u, f32)
    eps = np.finfo(np.float32 if f32 else np.float64).eps
    cond = np.linalg.cond(rbd_oracle.ChainOracle(arm).M(q))
    scale = np.maximum(np.abs(a).max(1), np.abs(u).max(1) / np.linalg.norm(rbd_oracle.ChainOracle(arm).M(q), 2, axis=(1, 2)))
    err = np.abs(back - a).max(1)
    assert (err <= 50 * eps * cond * scale).all(), (err / (eps * cond * scale)).max()


def _energy(ch, q, dq):
    """E = 1/2 dq^T M dq + V,  V = -sum_l m_l gravity . p_l over the links' centres of mass (the link frames)."""
    kin = 0.5 * np.einsum("bi,bij,bj->b", dq, ch.M(q), dq)
    V = 0.0
    for l in range(ch.n_links):
        V = V - ch.Tx(f"link{l}", q) @ (ch.W[l, :3] * ch.gravity[:3])
    return kin + V


@pytest.mark.parametrize("arm", ["ur5", "jaco2"])
def test_host_energy_balance_converges_first_order(plantsim, arm):
    """Without compensation the energy change E_S - E_0 equals the work sum_t tau_t . dq_{t+1} dt up to the integrator's
    error, which halves with dt (semi-implicit Euler is first order).  Independent of the oracle's g and C: a wrong sign
    of either breaks the balance."""
    ch = rbd_oracle.ChainOracle(arm)
    B, Ttot = 8, 0.2
    q, dq, _, _ = cases.states(arm, B)
    dq = 0.3 * dq
    rng = np.random.default_rng(5)
    u0 = rng.normal(size=q.shape) * 2.0  # constant torque per trajectory, so both step sizes see the same signal
    mism = []
    for dt in (2e-3, 1e-3):
        S = int(round(Ttot / dt))
        u = np.ascontiguousarray(np.broadcast_to(u0[None], (S, B, q.shape[1])))
        o = shim_simulate(plantsim, arm, q, dq, u, None, False, dt=dt, effort=0.0)
        work = np.einsum("tbi,tbi->b", o["u"], o["dq"]) * dt
        mism.append(np.abs(_energy(ch, o["q_final"], o["dq_final"]) - _energy(ch, q, dq) - work))
    ratio = mism[0] / mism[1]
    print(arm, "mismatch", mism[0], mism[1], "ratio", ratio)
    assert (mism[1] < 0.05 * np.abs(_energy(ch, q, dq)).max()).all()
    assert np.median(ratio) > 1.7 and np.median(ratio) < 2.4 and ratio.min() > 1.2 and ratio.max() < 3.5, ratio


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


def _plant_args(**over):
    a = dict(m=None, frame=0, xoff=None, q=None, dq=None, u=None, us=0, comp=0, path=None, ps=0, steps=4, dt=1e-3,
             ew=0.0, qt=None, dqt=None, ut=None, xt=None, cost=None, B=8, stream=None)
    a.update(over)
    return [a[k] for k in ("m", "frame", "xoff", "q", "dq", "u", "us", "comp", "path", "ps", "steps", "dt", "ew", "qt",
                           "dqt", "ut", "xt", "cost", "B", "stream")]


@pytest.mark.parametrize("fn", ["abrb_plant_rollout_f64", "abrb_plant_rollout_f32"])
def test_abi_plant_rollout_rejects_bad_arguments_before_any_device_work(native, fn):
    lib, m, buf = native
    f = getattr(lib, fn)
    p = buf.ctypes.data
    ok = dict(m=m, q=p, dq=p, u=p)
    bad = [
        (dict(m=None), _abi.EINVAL, "model"),
        (dict(q=None), _abi.EINVAL, "NULL q"),
        (dict(dq=None), _abi.EINVAL, "NULL dq"),
        (dict(u=None), _abi.EINVAL, "NULL u"),
        (dict(us=3), _abi.EINVAL, "u_stride"),
        (dict(us=6 * 8), _abi.EINVAL, "u_stride"),
        (dict(ps=3, path=p), _abi.EINVAL, "path_stride"),
        (dict(steps=-1), _abi.EINVAL, "steps"),
        (dict(B=-1), _abi.EINVAL, "B < 0"),
        (dict(ew=-1.0), _abi.EINVAL, "effort_weight"),
        (dict(ew=float("nan")), _abi.EINVAL, "effort_weight"),
        (dict(ew=float("inf")), _abi.EINVAL, "effort_weight"),
        (dict(q=p + 1), _abi.EINVAL, "misaligned pointer (q)"),
        (dict(u=p + 2), _abi.EINVAL, "misaligned pointer (u)"),
        (dict(path=p + 2), _abi.EINVAL, "misaligned pointer (path)"),
        (dict(cost=p + 1), _abi.EINVAL, "misaligned pointer (cost)"),
        (dict(xt=p + 2), _abi.EINVAL, "misaligned pointer (x_traj)"),
        (dict(ut=p + 1), _abi.EINVAL, "misaligned pointer (u_traj)"),
        (dict(frame=99), _abi.EFRAME, "frame"),
        (dict(frame=-1), _abi.EFRAME, "frame"),
    ]
    for over, code, word in bad:
        rc = f(*_plant_args(**{**ok, **over}))
        assert rc == code, (over, rc)
        msg = lib.abrb_last_error().decode()
        assert msg.startswith("abrb_plant_rollout") and word in msg, (over, msg)
    # B == 0 is a no-op whatever the pointers; a NULL u is fine without steps (the call then needs a device)
    assert f(*_plant_args(**{**ok, "B": 0, "q": None, "dq": None, "u": None})) == 0


@pytest.mark.parametrize("fn", ["abrb_forward_dynamics_f64", "abrb_forward_dynamics_f32", "abrb_inverse_dynamics_f64",
                                "abrb_inverse_dynamics_f32"])
def test_abi_dynamics_rejects_bad_arguments_before_any_device_work(native, fn):
    lib, m, buf = native
    f = getattr(lib, fn)
    p = buf.ctypes.data
    inn, out = ("u", "ddq") if "forward" in fn else ("ddq", "u")
    ok = dict(m=m, q=p, dq=p, i=p, o=p, B=8)
    bad = [
        (dict(m=None), "NULL model"),
        (dict(q=None), "NULL q"),
        (dict(dq=None), "NULL dq"),
        (dict(i=None), f"NULL {inn}"),
        (dict(o=None), f"NULL {out}"),
        (dict(B=-1), "B < 0"),
        (dict(q=p + 1), "misaligned pointer (q)"),
        (dict(i=p + 2), f"misaligned pointer ({inn})"),
        (dict(o=p + 1), f"misaligned pointer ({out})"),
    ]
    who = fn.rsplit("_", 1)[0]
    for over, word in bad:
        a = {**ok, **over}
        rc = f(a["m"], a["q"], a["dq"], a["i"], a["o"], a["B"], None)
        assert rc == _abi.EINVAL, (over, rc)
        msg = lib.abrb_last_error().decode()
        assert msg.startswith(who) and word in msg, (over, msg)
    assert f(m, None, None, None, None, 0, None) == 0


def test_abi_valid_calls_without_a_device_fail_with_ecuda(native):
    lib, m, buf = native
    if lib.abrb_device_count() > 0:
        pytest.skip("a CUDA device is present")
    p = buf.ctypes.data
    for fn in ("abrb_forward_dynamics_f64", "abrb_inverse_dynamics_f32"):
        assert getattr(lib, fn)(m, p, p, p, p, 4, None) == _abi.ECUDA
    for fn in ("abrb_plant_rollout_f64", "abrb_plant_rollout_f32"):
        assert getattr(lib, fn)(*_plant_args(m=m, q=p, dq=p, u=p, steps=3)) == _abi.ECUDA
        assert getattr(lib, fn)(*_plant_args(m=m, q=p, dq=p, steps=0, cost=p)) == _abi.ECUDA
    assert "no CUDA device" in lib.abrb_last_error().decode()


def test_signatures_cover_the_new_entry_points():
    from abr_control_b200 import _lib

    for fn in ("abrb_plant_rollout_f64", "abrb_plant_rollout_f32"):
        res, args = _lib.SIGNATURES[fn]
        assert len(args) == 20 and args[11] is C.c_double and args[12] is C.c_double and args[18] is C.c_int64
    for fn in ("abrb_forward_dynamics_f64", "abrb_forward_dynamics_f32", "abrb_inverse_dynamics_f64",
               "abrb_inverse_dynamics_f32"):
        res, args = _lib.SIGNATURES[fn]
        assert len(args) == 7 and args[5] is C.c_int64
    with open(os.path.join(ROOT, "include", "abrb.h")) as fh:
        hdr = fh.read()
    for fn in ("abrb_plant_rollout", "abrb_forward_dynamics", "abrb_inverse_dynamics"):
        assert f"int {fn}_f64(" in hdr and f"int {fn}_f32(" in hdr


# ============================================================================================== GPU
def _cfg(arm, dtype=np.float64):
    import abr_control_b200.arms as arms

    return getattr(arms, arm).Config(dtype=dtype)


def _np(x):
    return x.cpu().numpy() if hasattr(x, "cpu") else np.asarray(x)


# ---------------------------------------------------------------------------------------------- 6. = oracle
@pytest.mark.gpu
@pytest.mark.parametrize("variant", list(VARIANTS))
@pytest.mark.parametrize("arm", ARMS)
def test_device_rollout_vs_oracle(arm, variant):
    B = 12
    q, dq, u, path, comp, frame, off = variant_inputs(arm, variant, B)
    ref = oracle_for(arm, variant, B)
    rc = _cfg(arm)
    qf, dqf, tr, cost = rc.simulate(q, dq, u, dt=DT, path=path, effort_weight=EFFORT, compensate_gravity=comp,
                                    ref_frame=frame, xyz_offset=off)
    assert_matches_oracle(dict(tr, cost=cost), ref, 0, f"{arm} {variant}")
    f = np.float32
    rc32 = _cfg(arm, f)
    qf, dqf, tr, cost = rc32.simulate(q.astype(f), dq.astype(f), u.astype(f), dt=DT,
                                      path=None if path is None else path.astype(f), effort_weight=EFFORT,
                                      compensate_gravity=comp, ref_frame=frame, xyz_offset=off)
    assert tr["u"].dtype == np.float32 and cost.dtype == np.float32
    assert_matches_oracle(dict(tr, cost=cost), ref, 1, f"{arm} {variant} fp32")


@pytest.mark.gpu
@pytest.mark.parametrize("arm", ARMS)
def test_device_dynamics_vs_oracle(arm):
    q, dq, _, _ = cases.states(arm, 40)
    rng = np.random.default_rng(7)
    u, a = rng.normal(size=q.shape) * 5, rng.normal(size=q.shape) * 3
    rc = _cfg(arm)
    ref = oracle_forward(arm, q, dq, u)
    got = rc.forward_dynamics(q, dq, u)
    assert (np.abs(got - ref).max(1) / np.maximum(1.0, np.abs(ref).max(1))).max() < 1e-9
    ref = oracle_inverse(arm, q, dq, a)
    got = rc.inverse_dynamics(q, dq, a)
    assert (np.abs(got - ref).max(1) / np.maximum(1.0, np.abs(ref).max(1))).max() < 1e-9


# ---------------------------------------------------------------------------------------------- 7. replay
def _mpc_inputs(B, S, seed):
    import torch

    rc = _cfg("ur5")
    rng = np.random.default_rng(seed)
    q = torch.as_tensor(rng.uniform(0, 2 * np.pi, (B, 6)), device="cuda")
    dq = torch.as_tensor(rng.uniform(-0.5, 0.5, (B, 6)), device="cuda")
    x0 = rc.Tx("EE", q)
    ramp = torch.linspace(0, 1, S, device="cuda", dtype=torch.float64)[:, None, None]
    end = torch.as_tensor(rng.uniform(-0.1, 0.1, (B, 3)), device="cuda")
    ori = torch.as_tensor(rng.uniform(-1, 1, (1, B, 3)), device="cuda").expand(S, B, 3)
    path = torch.cat([x0[None] + ramp * end[None], ori], -1).contiguous()
    return rc, q, dq, path


@pytest.mark.gpu
@pytest.mark.parametrize("osc_kw", [dict(kp=10, ctrlr_dof=[T] * 6, use_C=True), dict(kp=10)], ids=["plain", "kp10"])
def test_device_replay_of_osc_rollouts(osc_kw):
    """OSC.rollout_path's recorded u through simulate with the same path and effort weight gives back its q, dq, x and
    cost; OSC.rollout's u without a path gives back its q and dq.  Bit-identity is not required, since nvcc may contract
    the plant's arithmetic into FMAs differently in the two kernels; on an H100 80GB HBM3 with CUDA 12.9 every
    difference was 0 for both controllers."""
    import torch

    from abr_control_b200 import controllers

    B, S, ew = 4096, 128, 1e-4
    rc, q, dq, path = _mpc_inputs(B, S, 11)
    c = controllers.OSC(rc, **osc_kw)
    qf, dqf, tr, cost = c.rollout_path(q, dq, path, dt=DT, effort_weight=ew)
    qs, dqs, ts, cs = rc.simulate(q, dq, tr["u"], dt=DT, path=path, effort_weight=ew)
    errs = dict(q=(ts["q"] - tr["q"]).abs().max().item(), dq=(ts["dq"] - tr["dq"]).abs().max().item(),
                x=(ts["x"] - tr["x"]).abs().max().item(), cost=((cs - cost).abs() / cost).max().item(),
                u=(ts["u"] - tr["u"]).abs().max().item())
    print(f"replay rollout_path {osc_kw}: " + ", ".join(f"{k} {v:.2e}" for k, v in errs.items()))
    assert errs["u"] == 0.0
    assert errs["q"] < 1e-9 and errs["x"] < 1e-9 and errs["dq"] < 1e-7 and errs["cost"] < 1e-9, errs
    assert torch.equal(qs, ts["q"][-1]) and torch.equal(dqs, ts["dq"][-1])
    target = path[-1]
    qf, dqf, tr = c.rollout(q, dq, target, steps=S, dt=DT)
    qs, dqs, ts, cs = rc.simulate(q, dq, tr["u"], dt=DT, record=("q", "dq"))
    eq, edq = (ts["q"] - tr["q"]).abs().max().item(), (ts["dq"] - tr["dq"]).abs().max().item()
    print(f"replay rollout {osc_kw}: q {eq:.2e}, dq {edq:.2e}")
    assert eq < 1e-9 and edq < 1e-7
    assert torch.equal(cs, torch.zeros_like(cs))


# ---------------------------------------------------------------------------------------------- 8. single step
@pytest.mark.gpu
@pytest.mark.parametrize("dtype", ["float64", "float32"])
def test_single_step_dynamics_at_65536_states(dtype):
    import torch

    rc = _cfg("ur5")
    B = 65536
    gen = torch.Generator(device="cuda").manual_seed(3)
    td = getattr(torch, dtype)
    q = (torch.rand((B, 6), device="cuda", generator=gen, dtype=torch.float64) * 2 * np.pi).to(td)
    dq = (torch.rand((B, 6), device="cuda", generator=gen, dtype=torch.float64) * 2 - 1).to(td)
    u = (torch.randn((B, 6), device="cuda", generator=gen, dtype=torch.float64) * 5).to(td)
    d = rc.eval(q.double(), dq.double(), want=("M", "g", "C"))
    cdq = torch.bmm(d["C"], dq.double()[..., None])[..., 0]
    ref = torch.linalg.solve(d["M"], (u.double() + d["g"] - cdq)[..., None])[..., 0]
    got = rc.forward_dynamics(q, dq, u)
    assert got.dtype == td and got.shape == (B, 6)
    rel = ((got.double() - ref).abs().amax(1) / ref.abs().amax(1).clamp_min(1.0))
    cond = torch.linalg.cond(d["M"])
    tol = (1e-13 if dtype == "float64" else 2e-6) * cond
    print(f"forward {dtype}: max rel {rel.max().item():.2e}, max rel / cond(M) {(rel / cond).max().item():.2e}")
    assert (rel <= tol).all()
    uu = rc.inverse_dynamics(q, dq, ref.to(td))
    refu = torch.bmm(d["M"], ref.to(td).double()[..., None])[..., 0] + cdq - d["g"]
    relu = ((uu.double() - refu).abs().amax(1) / refu.abs().amax(1).clamp_min(1.0)).max().item()
    print(f"inverse {dtype}: max rel {relu:.2e}")
    assert relu < (1e-12 if dtype == "float64" else 1e-4)


# ---------------------------------------------------------------------------------------------- 9. layout, indexing
@pytest.mark.gpu
def test_layouts_permutation_and_records_are_bit_identical():
    import torch

    rc = _cfg("ur5")
    B, S = 96, 16
    q, dq, u, path, _, _, _ = variant_inputs("ur5", "shared_u_per_path_comp_offset", B, S=S)
    q, dq, u, path = (torch.as_tensor(a, device="cuda") for a in (q, dq, u, path))
    kw = dict(dt=DT, effort_weight=1e-3, compensate_gravity=True)
    # a shared (S, n) sequence equals the same tiled to (S, B, n); a shared path equals the same tiled
    _, _, a, ca = rc.simulate(q, dq, u, path=path, **kw)
    _, _, b, cb = rc.simulate(q, dq, u[:, None].expand(S, B, 6).contiguous(), path=path, **kw)
    for k in ("q", "dq", "u", "x"):
        assert torch.equal(a[k], b[k]), k
    assert torch.equal(ca, cb)
    sp = path[:, 0].contiguous()
    _, _, a, ca = rc.simulate(q, dq, u, path=sp, **kw)
    _, _, b, cb = rc.simulate(q, dq, u, path=sp[:, None].expand(S, B, 6).contiguous(), **kw)
    for k in ("q", "dq", "u", "x"):
        assert torch.equal(a[k], b[k]), k
    assert torch.equal(ca, cb)
    # per-trajectory torques: permuting trajectories with their torque and path columns permutes every output
    up = u[:, None].expand(S, B, 6) + 0.1 * torch.randn((S, B, 6), device="cuda", dtype=torch.float64)
    up = up.contiguous()
    qa, dqa, a, ca = rc.simulate(q, dq, up, path=path, **kw)
    perm = torch.randperm(B, device="cuda")
    qp, dqp, p, cp = rc.simulate(q[perm].contiguous(), dq[perm].contiguous(), up[:, perm].contiguous(),
                                 path=path[:, perm].contiguous(), **kw)
    for k in ("q", "dq", "u", "x"):
        assert torch.equal(p[k], a[k][:, perm]), k
    assert torch.equal(cp, ca[perm]) and torch.equal(qp, qa[perm]) and torch.equal(dqp, dqa[perm])
    # step indexing: changing u_t changes q_{t+1}.. (records t on) and leaves x_t and everything before alone
    t0 = 5
    u2 = up.clone()
    u2[t0] += 1.0
    _, _, c2, _ = rc.simulate(q, dq, u2, path=path, **kw)
    for k in ("q", "dq", "u", "x"):
        assert torch.equal(c2[k][:t0], a[k][:t0]), k
    assert torch.equal(c2["x"][t0], a["x"][t0]) and (c2["x"][t0 + 1] != a["x"][t0 + 1]).any(-1).all()
    assert (c2["dq"][t0] != a["dq"][t0]).any(-1).all()
    # no steps: the state is left as it is, the cost is zero
    q0, dq0, tz, cz = rc.simulate(q, dq, up[:0], path=path[:0], **kw)
    assert torch.equal(q0, q) and torch.equal(dq0, dq) and tz["u"].shape == (0, B, 6) and torch.equal(cz, torch.zeros_like(cz))


@pytest.mark.gpu
@pytest.mark.parametrize("B,S", [(4096, 128), (140000, 8)])
def test_full_size_cost_only_equals_full_records(B, S):
    import torch

    rc, q, dq, path = _mpc_inputs(B, S, B + S)
    gen = torch.Generator(device="cuda").manual_seed(B)
    u = torch.randn((S, B, 6), device="cuda", generator=gen, dtype=torch.float64)
    kw = dict(dt=DT, path=path, effort_weight=1e-4, compensate_gravity=True)
    qa, dqa, _, cost_only = rc.simulate(q, dq, u, record=(), **kw)
    qb, dqb, tr, cost = rc.simulate(q, dq, u, **kw)
    assert torch.equal(cost_only, cost) and torch.equal(qa, qb) and torch.equal(dqa, dqb)
    assert torch.equal(tr["q"][-1], qb) and torch.isfinite(cost).all()
    # a sample of trajectories against stepping forward_dynamics and Tx through the public API
    sel = torch.arange(0, B, max(1, B // 64), device="cuda")
    qs, dqs, cs = q[sel].clone(), dq[sel].clone(), torch.zeros(len(sel), dtype=q.dtype, device="cuda")
    for t in range(S):
        x = rc.Tx("EE", qs)
        tau = u[t, sel] - rc.eval(qs, want=("g",))["g"]
        dqs = dqs + rc.forward_dynamics(qs, dqs, tau) * DT
        qs = qs + dqs * DT
        cs += ((x - path[t, sel, :3]) ** 2).sum(-1) + 1e-4 * (tau ** 2).sum(-1)
    eq, ec = (qb[sel] - qs).abs().max().item(), ((cost[sel] - cs).abs() / cs).max().item()
    print(f"{B}x{S}: stepped public API q {eq:.2e}, cost {ec:.2e}")
    assert eq < 1e-9 and ec < 1e-9


# ---------------------------------------------------------------------------------------------- 10. input forms
@pytest.mark.gpu
def test_host_arrays_and_single_states_match_cuda_tensors():
    import torch

    rc = _cfg("ur5")
    B, S = 40, 10
    q, dq, u, path, _, _, _ = variant_inputs("ur5", "per_u_per_path_offset_frame", B, S=S)
    h = rc.simulate(q, dq, u, path=path, effort_weight=1e-3)
    d = rc.simulate(*(torch.as_tensor(a, device="cuda") for a in (q, dq, u)), path=torch.as_tensor(path, device="cuda"),
                    effort_weight=1e-3)
    assert isinstance(h[0], np.ndarray) and isinstance(h[3], np.ndarray)
    assert np.array_equal(h[0], _np(d[0])) and np.array_equal(h[1], _np(d[1])) and np.array_equal(h[3], _np(d[3]))
    for k in ("q", "dq", "u", "x"):
        assert np.array_equal(h[2][k], _np(d[2][k])), k
    s = rc.simulate(q[0], dq[0], u[:, 0], path=path[:, 0])
    b = rc.simulate(q[:1], dq[:1], u[:, 0], path=path[:, 0])
    assert s[0].shape == (6,) and s[2]["x"].shape == (S, 3) and np.ndim(s[3]) == 0
    assert np.array_equal(s[0], b[0][0]) and np.array_equal(s[2]["u"], b[2]["u"][:, 0]) and s[3] == b[3][0]
    for fn in (rc.forward_dynamics, rc.inverse_dynamics):
        hh = fn(q, dq, u[0])
        dd = fn(*(torch.as_tensor(a, device="cuda") for a in (q, dq, u[0])))
        assert isinstance(hh, np.ndarray) and np.array_equal(hh, _np(dd))
        one = fn(q[3], dq[3], u[0, 3])
        assert one.shape == (6,) and np.array_equal(one, hh[3])
    with pytest.raises(ValueError):
        rc.forward_dynamics(q, dq, u[0, :5])
    with pytest.raises(ValueError):
        rc.simulate(q, dq, u[:, :5])
    with pytest.raises(ValueError):
        rc.simulate(q, dq, u, path=path[:-1])
