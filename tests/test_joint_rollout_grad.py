"""Gradients of the Joint closed loop: ``Joint.rollout_path`` through ``torch.autograd``
(``abrb_joint_rollout_path_vjp_*``).

Semantics (include/abrb.h, DESIGN.md S3.6): the adjoint recursion over the recorded states of
``abrb_joint_rollout_path_*`` gives the cotangents of the start state, the path and path velocity rows (per trajectory)
and the gains (per trajectory).  The wrap of ``path - q`` passes the tangent through unchanged.

CPU part: the kernel's per-lane function (abrb_grad.cuh) runs on the host through tests/hostsim/jointgradsim.cpp (TEST
INFRASTRUCTURE, never loaded by the package): a dot-product test against a forward-mode dual rollout of
``ctrl_rollout_step``, central differences of the NumPy oracle, bit-identical values of the phased dual step, edge
cases, argument checking of the C entry points and the Python rejections.  GPU part: the kernel against the shim,
gradcheck, a full-size run, shared paths, bit identities, the gains and a small path optimisation.
"""
import ctypes as C
import os

import numpy as np
import pytest

from abr_control_b200 import _abi
from test_ctrl_rollout import DT, EFFORT, MID, _desc, oracle_ctrl_rollout, shim_rollout, wrap
from test_generic_chains import random_chain
from test_plant import _build, _p
from test_plant_grad import random_cotangents

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ARMS = ("ur5", "jaco2", "threejoint", "twojoint")
CHAINS = ARMS + ("rand7_shear",)
# (path layout, path velocity?, account_for_gravity, frame, offset)
VARIANTS = {
    "per_grav": ("per", False, True, "EE", None),
    "per_vel_nograv_mid_offset": ("per", True, False, "mid", [0.02, -0.03, 0.05]),
    "shared_vel_grav": ("shared", True, True, "EE", None),
    "shared_nograv_offset": ("shared", False, False, "EE", [0.0, 0.04, -0.02]),
}
KP, KV = 120.0, 15.0
KEYS = ("cost", "qf", "dqf", "q", "dq", "u", "x")


@pytest.fixture(scope="module")
def jg(tmp_path_factory):
    return _build(tmp_path_factory, "jointgradsim")


def _arm(name):
    """an arm name, or the descriptor dict of a random sheared 7-joint chain"""
    return random_chain(7, False, seed=107) if name == "rand7_shear" else name


def _frame(name, frame):
    return MID.get(name, "EE") if frame == "mid" else frame


def joint_inputs(name, variant, B, S, seed=0):
    """starts on the arm's range and a path that wanders within 0.4 rad of them: |wrap(path - q)| stays far from pi"""
    layout, vel, grav, frame, off = VARIANTS[variant]
    n = _desc(_arm(name)).n_joints
    rng = np.random.default_rng(seed)
    q = rng.uniform(-2.0, 2.0, (B, n))
    dq = rng.uniform(-0.5, 0.5, (B, n))
    steps = np.cumsum(rng.normal(scale=0.03, size=(S, B, n)), axis=0)
    path = q[None] + np.clip(steps, -0.4, 0.4) + 0.1
    pv = rng.normal(scale=0.5, size=(S, B, n)) if vel else None
    if layout == "shared":
        path, pv = path[:, 0], None if pv is None else pv[:, 0]
    return q, dq, path, pv, grav, _frame(name, frame), off


def _stride(a, n):
    return 0 if a is None or a.ndim == 2 else n


def _arr(a):
    return None if a is None else np.ascontiguousarray(a, dtype=np.float64)


def forward(jg, name, q, dq, path, pv, grav, frame, off, kp=KP, kv=KV):
    return shim_rollout(jg, _arm(name), "joint", dict(kp=kp, kv=kv, account_for_gravity=grav), q, dq, path, pv,
                        frame=frame, xoff=off)


def shim_vjp(jg, name, q0, dq0, path, pv, grav, frame, off, q_traj, dq_traj, cot, kp=KP, kv=KV, f32=0,
             want=("path", "pv", "gains")):
    cd = _desc(_arm(name))
    n, B = cd.n_joints, len(q0)
    S = path.shape[0]
    g_path = np.zeros((S, B, n)) if "path" in want else None
    g_pv = np.zeros((S, B, n)) if "pv" in want and pv is not None else None
    g_gains = np.zeros((B, 2)) if "gains" in want else None
    gq0, gdq0 = np.zeros((B, n)), np.zeros((B, n))
    xo = None if off is None else (C.c_double * 3)(*off)
    c = [_arr(cot.get(k)) for k in KEYS]
    rc = jg.jg_rollout_vjp(C.byref(cd), f32, C.c_double(kp), C.c_double(kv), int(grav), jg.hs_frame_id(n, frame.encode()),
                           xo, _p(_arr(q0)), _p(_arr(dq0)), _p(_arr(path)), _stride(path, n), _p(_arr(pv)),
                           _stride(pv, n), S, C.c_double(DT), C.c_double(EFFORT), _p(_arr(q_traj)), _p(_arr(dq_traj)),
                           *[_p(a) for a in c], _p(g_path), _p(g_pv), _p(g_gains), _p(gq0), _p(gdq0), C.c_int64(B))
    assert rc == 0
    return dict(path=g_path, pv=g_pv, gains=g_gains, q0=gq0, dq0=gdq0)


def shim_jvp(jg, name, q0, dq0, path, pv, grav, frame, off, tan, phased=0, kp=KP, kv=KV):
    """tan: dict(a, b, path, pv, kp, kv) -> dict of record values and tangents"""
    cd = _desc(_arm(name))
    n, B = cd.n_joints, len(q0)
    S = path.shape[0]
    o = {k: np.zeros((S, B, 3 if k == "x" else n)) for k in ("q", "dq", "u", "x")}
    t = {k: np.zeros_like(o[k]) for k in o}
    cost, t_cost = np.zeros(B), np.zeros(B)
    t_qf, t_dqf = np.zeros((B, n)), np.zeros((B, n))
    xo = None if off is None else (C.c_double * 3)(*off)
    rc = jg.jg_rollout_jvp(C.byref(cd), 0, phased, C.c_double(kp), C.c_double(kv), int(grav),
                           jg.hs_frame_id(n, frame.encode()), xo, _p(_arr(q0)), _p(_arr(dq0)), _p(_arr(path)),
                           _stride(path, n), _p(_arr(pv)), _stride(pv, n), S, C.c_double(DT), C.c_double(EFFORT),
                           _p(_arr(tan["a"])), _p(_arr(tan["b"])), _p(_arr(tan["path"])), _p(_arr(tan["pv"])),
                           C.c_double(tan["kp"]), C.c_double(tan["kv"]), *[_p(o[k]) for k in ("q", "dq", "u", "x")],
                           _p(cost), *[_p(t[k]) for k in ("q", "dq", "u", "x")], _p(t_cost), _p(t_qf), _p(t_dqf),
                           C.c_int64(B))
    assert rc == 0
    o["cost"] = cost
    t.update(cost=t_cost, qf=t_qf, dqf=t_dqf)
    return o, t


def random_tangents(rng, q, path, pv):
    return dict(a=rng.normal(size=q.shape), b=rng.normal(size=q.shape), path=rng.normal(size=path.shape),
                pv=None if pv is None else rng.normal(size=pv.shape), kp=float(rng.normal()), kv=float(rng.normal()))


def pair(g, tan, path, pv):
    """<g, tangent> over every differentiable input; a shared path's gradient is the sum over B"""
    red = lambda x, ref: x if ref.ndim == 3 else x.sum(1)  # noqa: E731
    s = np.sum(g["q0"] * tan["a"]) + np.sum(g["dq0"] * tan["b"]) + np.sum(red(g["path"], path) * tan["path"])
    if pv is not None:
        s += np.sum(red(g["pv"], pv) * tan["pv"])
    return s + g["gains"][:, 0].sum() * tan["kp"] + g["gains"][:, 1].sum() * tan["kv"]


# ---------------------------------------------------------------------------------------------- host
@pytest.mark.parametrize("variant", list(VARIANTS))
@pytest.mark.parametrize("name", CHAINS)
def test_host_adjoint_dot_product(jg, name, variant):
    """<J^T v, w> from the lane loop equals <v, J w> from a dual rollout of ctrl_rollout_step, with random cotangents
    on every output and record, within 1e-11 relative."""
    B, S = 4, 7
    q, dq, path, pv, grav, frame, off = joint_inputs(name, variant, B, S, seed=3)
    fw = forward(jg, name, q, dq, path, pv, grav, frame, off)
    n = q.shape[1]
    rng = np.random.default_rng(11)
    cot = random_cotangents(rng, S, B, n)
    g = shim_vjp(jg, name, q, dq, path, pv, grav, frame, off, fw["q"], fw["dq"], cot)
    tan = random_tangents(rng, q, path, pv)
    _, t = shim_jvp(jg, name, q, dq, path, pv, grav, frame, off, tan)
    lhs = pair(g, tan, path, pv)
    rhs = sum(np.sum(cot[k] * t[k]) for k in KEYS)
    assert abs(lhs - rhs) < 1e-11 * max(abs(lhs), abs(rhs)), (lhs, rhs)


@pytest.mark.parametrize("name", ARMS)
def test_host_gradient_vs_central_differences_of_the_oracle(jg, name):
    """S = 16: the gradient of cost + w.q_final + wx.x along each input group (q0, dq0, path, path velocity, kp, kv)
    against central differences of oracle_ctrl_rollout, within 1e-6 relative."""
    B, S = 2, 16
    q, dq, path, pv, grav, frame, off = joint_inputs(name, "per_vel_nograv_mid_offset", B, S, seed=5)
    grav = True
    n = q.shape[1]
    rng = np.random.default_rng(21)
    w, wx = rng.normal(size=(B, n)), rng.normal(size=(S, B, 3))
    fw = forward(jg, name, q, dq, path, pv, grav, frame, off)
    pre = np.concatenate([q[None], fw["q"][:-1]])
    assert np.abs(wrap(path - pre)).max() < np.pi - 1e-3
    g = shim_vjp(jg, name, q, dq, path, pv, grav, frame, off, fw["q"], fw["dq"], dict(cost=np.ones(B), qf=w, x=wx))

    def f(qq, dd, pp, vv, kp, kv):
        o = oracle_ctrl_rollout(name, "joint", dict(kp=kp, kv=kv, account_for_gravity=grav), qq, dd, pp, DT, vv,
                                effort_weight=EFFORT, ref_frame=frame, offset=off)
        return np.sum(o["cost"]) + np.sum(w * o["q_final"]) + np.sum(wx * o["x"])

    zero = dict(a=np.zeros_like(q), b=np.zeros_like(q), path=np.zeros_like(path), pv=np.zeros_like(pv), kp=0.0, kv=0.0)
    for key in ("a", "b", "path", "pv", "kp", "kv"):
        tan = dict(zero)
        tan[key] = float(rng.normal()) if key in ("kp", "kv") else rng.normal(size=zero[key].shape)
        h = 1e-5 * (10.0 if key in ("kp", "kv") else 1.0)
        args = lambda s: (q + s * tan["a"], dq + s * tan["b"], path + s * tan["path"], pv + s * tan["pv"],  # noqa
                          KP + s * tan["kp"], KV + s * tan["kv"])
        fd = (f(*args(h)) - f(*args(-h))) / (2 * h)
        an = pair(g, tan, path, pv)
        assert abs(fd - an) <= 1e-6 * max(1.0, abs(an)), (key, fd, an)


@pytest.mark.parametrize("variant", list(VARIANTS))
@pytest.mark.parametrize("name", CHAINS)
def test_host_dual_step_values_are_the_forward_records_bit_for_bit(jg, name, variant):
    """The values of the phased dual step joint_vjp_lane runs (and of ctrl_rollout_step on Dual) equal the forward
    shim's records u, x, q, dq and the cost bit for bit; both give the same tangents."""
    B, S = 3, 9
    q, dq, path, pv, grav, frame, off = joint_inputs(name, variant, B, S, seed=7)
    fw = forward(jg, name, q, dq, path, pv, grav, frame, off)
    tan = random_tangents(np.random.default_rng(2), q, path, pv)
    o1, t1 = shim_jvp(jg, name, q, dq, path, pv, grav, frame, off, tan, phased=1)
    o0, t0 = shim_jvp(jg, name, q, dq, path, pv, grav, frame, off, tan, phased=0)
    for o in (o0, o1):
        for k in ("q", "dq", "u", "x", "cost"):
            assert np.array_equal(o[k], fw[k]), k
    for k in t0:
        np.testing.assert_allclose(t1[k], t0[k], rtol=1e-13, atol=1e-13 * max(1.0, np.abs(t0[k]).max()))


def test_host_zero_steps_zero_cotangents_and_optional_outputs(jg):
    name, variant = "ur5", "per_vel_nograv_mid_offset"
    B, n = 3, 6
    rng = np.random.default_rng(4)
    q, dq, path, pv, grav, frame, off = joint_inputs(name, variant, B, 5, seed=1)
    # steps = 0: the start-state cotangents are those of the final state, the gains get zero
    cot = random_cotangents(rng, 0, B, n)
    e = np.zeros((0, B, n))
    g = shim_vjp(jg, name, q, dq, e, e, grav, frame, off, e, e, cot)
    assert np.array_equal(g["q0"], cot["qf"]) and np.array_equal(g["dq0"], cot["dqf"])
    assert np.array_equal(g["gains"], np.zeros((B, 2)))
    # zero cotangents: zero gradients
    fw = forward(jg, name, q, dq, path, pv, grav, frame, off)
    S = path.shape[0]
    zero = {k: np.zeros_like(v) for k, v in random_cotangents(rng, S, B, n).items()}
    g = shim_vjp(jg, name, q, dq, path, pv, grav, frame, off, fw["q"], fw["dq"], zero)
    assert all(not np.any(v) for v in g.values())
    g = shim_vjp(jg, name, q, dq, path, pv, grav, frame, off, fw["q"], fw["dq"], {})
    assert all(not np.any(v) for v in g.values())
    # a missing g_path, g_path_velocity or g_gains changes no other output
    cot = random_cotangents(rng, S, B, n)
    full = shim_vjp(jg, name, q, dq, path, pv, grav, frame, off, fw["q"], fw["dq"], cot)
    for want in (("pv", "gains"), ("path", "pv"), ("path", "gains"), ()):
        part = shim_vjp(jg, name, q, dq, path, pv, grav, frame, off, fw["q"], fw["dq"], cot, want=want)
        for k, v in part.items():
            assert (v is None) == (k in ("path", "pv", "gains") and k not in want), (want, k)
            if v is not None:
                assert np.array_equal(v, full[k]), (want, k)


def test_host_fp32_lanes_follow_fp64(jg):
    name, variant = "ur5", "per_vel_nograv_mid_offset"
    B, S, n = 3, 6, 6
    q, dq, path, pv, grav, frame, off = joint_inputs(name, variant, B, S, seed=2)
    fw = forward(jg, name, q, dq, path, pv, grav, frame, off)
    cot = random_cotangents(np.random.default_rng(3), S, B, n)
    g64 = shim_vjp(jg, name, q, dq, path, pv, grav, frame, off, fw["q"], fw["dq"], cot)
    g32 = shim_vjp(jg, name, q, dq, path, pv, grav, frame, off, fw["q"], fw["dq"], cot, f32=1)
    for k in g64:
        scale = max(1.0, np.abs(g64[k]).max())
        assert np.abs(g32[k] - g64[k]).max() < 1e-3 * scale, k


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


VJP_FNS = ["abrb_joint_rollout_path_vjp_f64", "abrb_joint_rollout_path_vjp_f32"]
_VJP_KEYS = ("m", "kp", "kv", "grav", "frame", "xoff", "q0", "dq0", "path", "ps", "pv", "pvs", "steps", "dt", "ew",
             "qt", "dqt", "gc", "gq", "gdq", "gqt", "gdqt", "gut", "gxt", "gp", "gpv", "gg", "gq0", "gdq0", "B",
             "stream")


def _vjp_args(**over):
    a = {k: None for k in _VJP_KEYS}
    a.update(kp=10.0, kv=3.0, grav=1, frame=0, ps=0, pvs=0, steps=4, dt=1e-3, ew=0.0, B=8)
    a.update(over)
    return [a[k] for k in _VJP_KEYS]


@pytest.mark.parametrize("fn", VJP_FNS)
def test_abi_vjp_rejects_bad_arguments_before_any_device_work(native, fn):
    lib, m, buf = native
    f = getattr(lib, fn)
    p = buf.ctypes.data
    ok = dict(m=m, q0=p, dq0=p, path=p, qt=p, dqt=p, gq0=p, gdq0=p)
    bad = [
        (dict(m=None), _abi.EINVAL, "model"),
        (dict(q0=None), _abi.EINVAL, "NULL q0"),
        (dict(dq0=None), _abi.EINVAL, "NULL dq0"),
        (dict(gq0=None), _abi.EINVAL, "NULL gq0"),
        (dict(gdq0=None), _abi.EINVAL, "NULL gdq0"),
        (dict(path=None), _abi.EINVAL, "NULL path"),
        (dict(qt=None), _abi.EINVAL, "NULL q_traj"),
        (dict(dqt=None), _abi.EINVAL, "NULL dq_traj"),
        (dict(gpv=p), _abi.EINVAL, "g_path_velocity without path_velocity"),
        (dict(ps=3), _abi.EINVAL, "path_stride"),
        (dict(pv=p, pvs=2), _abi.EINVAL, "pv_stride"),
        (dict(steps=-1), _abi.EINVAL, "steps"),
        (dict(B=-1), _abi.EINVAL, "B < 0"),
        (dict(ew=-1.0), _abi.EINVAL, "effort_weight"),
        (dict(ew=float("nan")), _abi.EINVAL, "effort_weight"),
        (dict(q0=p + 1), _abi.EINVAL, "misaligned pointer (q0)"),
        (dict(path=p + 2), _abi.EINVAL, "misaligned pointer (path)"),
        (dict(gc=p + 1), _abi.EINVAL, "misaligned pointer (g_cost)"),
        (dict(gxt=p + 2), _abi.EINVAL, "misaligned pointer (g_x_traj)"),
        (dict(gp=p + 1), _abi.EINVAL, "misaligned pointer (g_path)"),
        (dict(gg=p + 2), _abi.EINVAL, "misaligned pointer (g_gains)"),
        (dict(gdq0=p + 1), _abi.EINVAL, "misaligned pointer (gdq0)"),
        (dict(frame=99), _abi.EFRAME, "frame"),
        (dict(frame=-1), _abi.EFRAME, "frame"),
    ]
    for over, code, word in bad:
        rc = f(*_vjp_args(**{**ok, **over}))
        assert rc == code, (over, rc)
        msg = lib.abrb_last_error().decode()
        assert msg.startswith("abrb_joint_rollout_path_vjp") and word in msg, (over, msg)
    # no path or records are needed for steps == 0; B == 0 is a no-op whatever the pointers
    assert f(*_vjp_args(**{**ok, "B": 0, "q0": None, "dq0": None, "path": None, "gq0": None})) == 0
    if lib.abrb_device_count() == 0:
        assert f(*_vjp_args(**{**ok, "steps": 0, "path": None, "qt": None, "dqt": None})) == _abi.ECUDA
        assert f(*_vjp_args(**{**ok, "ps": 6, "pv": p, "pvs": 6, "gpv": p, "gp": p, "gg": p})) == _abi.ECUDA
        assert "no CUDA device" in lib.abrb_last_error().decode()


def test_signatures_and_header_cover_the_vjp_entry_points():
    from abr_control_b200 import _lib

    for fn in VJP_FNS:
        res, args = _lib.SIGNATURES[fn]
        assert res is C.c_int and len(args) == len(_VJP_KEYS)
        assert args[1] is C.c_double and args[2] is C.c_double and args[3] is C.c_int and args[4] is C.c_int
        assert args[12] is C.c_int and args[13] is C.c_double and args[14] is C.c_double
        assert all(a is C.c_void_p for a in args[15:29]) and args[-2] is C.c_int64
    with open(os.path.join(ROOT, "include", "abrb.h")) as fh:
        hdr = fh.read()
    for fn in VJP_FNS:
        assert f"int {fn}(" in hdr


# ---------------------------------------------------------------------------------------------- Python checks
def test_python_rejects_cpu_and_integer_tensors_that_require_grad():
    torch = pytest.importorskip("torch")
    import abr_control_b200.arms as arms
    from abr_control_b200 import controllers

    rc = arms.ur5.Config()
    ctrl = controllers.Joint(rc, kp=50.0, kv=5.0)
    q = np.zeros((2, 6))
    path = np.zeros((3, 6))
    with pytest.raises(ValueError, match="float32 or float64 CUDA tensors"):
        ctrl.rollout_path(q, q, torch.zeros(3, 6, dtype=torch.float64, requires_grad=True))
    with pytest.raises(ValueError, match="float32 or float64 CUDA tensors"):
        ctrl.rollout_path(torch.zeros(2, 6, requires_grad=True), q, path)
    with pytest.raises(ValueError, match="float32 or float64 CUDA tensors"):
        controllers.Joint(rc, kp=torch.tensor(4.0, requires_grad=True)).rollout_path(q, q, path)


def test_python_numpy_and_value_only_calls_do_not_take_the_autograd_path(monkeypatch):
    torch = pytest.importorskip("torch")
    import abr_control_b200.arms as arms
    from abr_control_b200 import controllers
    from abr_control_b200.controllers import _batch

    def boom(*a, **k):
        raise AssertionError("autograd path taken")

    import abr_control_b200.controllers._ctrl_autograd as ca

    monkeypatch.setattr(ca, "joint_rollout_path", boom)
    monkeypatch.setattr(_batch, "ctrl_rollout", lambda *a, **k: "value")
    rc = arms.ur5.Config()
    q, path = np.zeros((2, 6)), np.zeros((3, 6))
    assert controllers.Joint(rc, kp=50.0).rollout_path(q, q, path) == "value"
    with torch.no_grad():
        assert controllers.Joint(rc, kp=50.0).rollout_path(q, q, torch.zeros(3, 6, requires_grad=True)) == "value"
    assert not _batch.wants_grad(q, path, 3.0, torch.zeros(3))


# ============================================================================================== GPU
def _dev():
    import torch

    return torch.device("cuda")


def _ctrl(name, kp=KP, kv=KV, grav=True, dtype=np.float64):
    import abr_control_b200.arms as arms
    from abr_control_b200 import controllers
    from abr_control_b200.arms.base_config import BaseConfig

    a = _arm(name)
    rc = BaseConfig(a, dtype=dtype) if isinstance(a, dict) else getattr(arms, a).Config(dtype=dtype)
    return controllers.Joint(rc, kp=kp, kv=kv, account_for_gravity=grav)


def _t(a, dtype=None, grad=False):
    import torch

    if a is None:
        return None
    t = torch.as_tensor(np.asarray(a), device=_dev()).to(dtype or torch.float64)
    return t.requires_grad_(grad)


def device_grads(name, q, dq, path, pv, grav, frame, off, cot, dtype=None, kp=KP, kv=KV):
    """gradients of <cot, outputs> through Joint.rollout_path on the device -> dict like shim_vjp's (gains summed)"""
    import torch

    dtype = dtype or torch.float64
    kpt, kvt = _t(kp, dtype, True), _t(kv, dtype, True)
    c = _ctrl(name, kpt, kvt, grav)
    qt, dqt, pt, vt = _t(q, dtype, True), _t(dq, dtype, True), _t(path, dtype, True), _t(pv, dtype, pv is not None)
    qf, dqf, tr, cost = c.rollout_path(qt, dqt, pt, dt=DT, path_velocity=vt, ref_frame=frame, xyz_offset=off,
                                       effort_weight=EFFORT)
    out = dict(cost=cost, qf=qf, dqf=dqf, **tr)
    loss = sum((out[k] * _t(cot[k], dtype)).sum() for k in KEYS if cot.get(k) is not None)
    ins = [qt, dqt, pt, kpt, kvt] + ([vt] if vt is not None else [])
    gr = torch.autograd.grad(loss, ins)
    res = dict(q0=gr[0], dq0=gr[1], path=gr[2], kp=gr[3], kv=gr[4], pv=gr[5] if vt is not None else None)
    return {k: None if v is None else v.double().cpu().numpy() for k, v in res.items()}


def _close(a, b, tol):
    scale = max(1.0, np.abs(b).max())
    return np.abs(a - b).max() <= tol * scale, np.abs(a - b).max() / scale


@pytest.mark.gpu
@pytest.mark.parametrize("f32", [False, True])
@pytest.mark.parametrize("name", CHAINS)
def test_device_vs_shim(jg, name, f32):
    """every input's gradient against the shim (fp64 1e-11, fp32 5e-3 of the largest entry); B spans a second pass
    of the grid-stride loop"""
    import torch

    variant = "per_vel_nograv_mid_offset" if name in ("ur5", "rand7_shear") else "shared_vel_grav"
    S = 6
    B = 132 * 16 * 4 + 37 if name == "ur5" and not f32 else 70
    q, dq, path, pv, grav, frame, off = joint_inputs(name, variant, B, S, seed=8)
    n = q.shape[1]
    cot = random_cotangents(np.random.default_rng(12), S, B, n)
    got = device_grads(name, q, dq, path, pv, grav, frame, off, cot, torch.float32 if f32 else torch.float64)
    rows = np.r_[0:20, B - 20:B] if B > 1000 else np.arange(B)
    sub = lambda a: a if a.ndim == 2 else a[:, rows]  # noqa: E731
    fw = forward(jg, name, q[rows], dq[rows], sub(path), sub(pv) if pv is not None else None, grav, frame, off)
    csub = {k: (v[rows] if k in ("cost", "qf", "dqf") else v[:, rows]) for k, v in cot.items()}
    ref = shim_vjp(jg, name, q[rows], dq[rows], sub(path), sub(pv) if pv is not None else None, grav, frame, off,
                   fw["q"], fw["dq"], csub)
    tol = 5e-3 if f32 else 1e-11
    for k in ("q0", "dq0"):
        ok, err = _close(got[k][rows], ref[k], tol)
        assert ok, (k, err)
    if path.ndim == 3:
        for k in ("path", "pv"):
            ok, err = _close(got[k][:, rows], ref[k], tol)
            assert ok, (k, err)
    if B == len(rows):
        red = (lambda x: x) if path.ndim == 3 else (lambda x: x.sum(1))
        for k in ("path", "pv"):
            ok, err = _close(got[k], red(ref[k]), tol)
            assert ok, (k, err)
        for i, k in enumerate(("kp", "kv")):
            ok, err = _close(np.atleast_1d(got[k]), np.atleast_1d(ref["gains"][:, i].sum()), tol)
            assert ok, (k, err)


@pytest.mark.gpu
def test_gradcheck_every_input():
    import torch

    c = _ctrl("ur5", _t(40.0, grad=True), _t(6.0, grad=True))
    q, dq, path, pv, grav, frame, off = joint_inputs("ur5", "per_vel_nograv_mid_offset", 3, 5, seed=1)
    ins = [_t(a, grad=True) for a in (q, dq, path, pv)]

    def fn(qq, dd, pp, vv, kp, kv):
        c.kp, c.kv = kp, kv
        qf, dqf, tr, cost = c.rollout_path(qq, dd, pp, path_velocity=vv, ref_frame=frame, xyz_offset=off,
                                           effort_weight=EFFORT)
        return cost, qf, dqf, tr["x"], tr["u"]

    assert torch.autograd.gradcheck(fn, ins + [_t(40.0, grad=True), _t(6.0, grad=True)], eps=1e-6, atol=1e-5,
                                    rtol=1e-4)


@pytest.mark.gpu
def test_full_size_ur5_against_shim_and_fp32(jg):
    """4096 UR5 trajectories x 128 steps, per-trajectory path and velocity: fp64 against the shim on 12 sampled rows
    (1e-10), fp32 against the device fp64 gradient (median 1e-5, p99 1e-4 relative to each row's largest entry;
    an H100 gave 1.1e-6 and 2.5e-6)."""
    import torch

    jg_lib = jg

    B, S, name = 4096, 128, "ur5"
    q, dq, path, pv, grav, frame, off = joint_inputs(name, "per_vel_nograv_mid_offset", B, S, seed=31)
    n = q.shape[1]
    cot = dict(cost=np.ones(B), x=np.random.default_rng(5).normal(size=(S, B, 3)))
    g64 = device_grads(name, q, dq, path, pv, grav, frame, off, cot)
    g32 = device_grads(name, q, dq, path, pv, grav, frame, off, cot, torch.float32)
    rows = np.random.default_rng(0).choice(B, 12, replace=False)
    fw = forward(jg_lib, name, q[rows], dq[rows], path[:, rows], pv[:, rows], grav, frame, off)
    ref = shim_vjp(jg_lib, name, q[rows], dq[rows], path[:, rows], pv[:, rows], grav, frame, off, fw["q"], fw["dq"],
                   dict(cost=np.ones(len(rows)), x=cot["x"][:, rows]))
    for k in ("q0", "dq0"):
        assert _close(g64[k][rows], ref[k], 1e-10)[0], k
    for k in ("path", "pv"):
        assert _close(g64[k][:, rows], ref[k], 1e-10)[0], k
    for k in ("path", "pv"):
        a, b = g32[k].transpose(1, 0, 2).reshape(B, -1), g64[k].transpose(1, 0, 2).reshape(B, -1)
        rel = np.abs(a - b).max(1) / np.maximum(1e-30, np.abs(b).max(1))
        print(k, "fp32 median", np.median(rel), "p99", np.percentile(rel, 99))
        assert np.median(rel) < 1e-5 and np.percentile(rel, 99) < 1e-4, k


@pytest.mark.gpu
def test_shared_path_gradient_is_the_sum_of_the_broadcast_one():
    import torch

    B, S = 300, 12
    q, dq, path, pv, grav, frame, off = joint_inputs("jaco2", "shared_vel_grav", B, S, seed=4)
    cot = random_cotangents(np.random.default_rng(6), S, B, 6)
    gs = device_grads("jaco2", q, dq, path, pv, grav, frame, off, cot)
    tile = lambda a: np.ascontiguousarray(np.broadcast_to(a[:, None], (S, B, a.shape[-1])))  # noqa: E731
    gt = device_grads("jaco2", q, dq, tile(path), tile(pv), grav, frame, off, cot)
    for k in ("path", "pv"):
        np.testing.assert_allclose(gs[k], gt[k].sum(1), rtol=1e-12, atol=1e-12 * np.abs(gs[k]).max())
    for k in ("q0", "dq0", "kp", "kv"):
        np.testing.assert_allclose(gs[k], gt[k], rtol=1e-12, atol=1e-12 * max(1.0, np.abs(gs[k]).max()))
    del torch


@pytest.mark.gpu
def test_permuted_and_tiled_batches_and_forward_values_are_bit_identical():
    import torch

    B, S = 257, 10
    q, dq, path, pv, grav, frame, off = joint_inputs("ur5", "per_vel_nograv_mid_offset", B, S, seed=9)
    cot = random_cotangents(np.random.default_rng(7), S, B, 6, which=("cost", "qf", "x"))
    g = device_grads("ur5", q, dq, path, pv, grav, frame, off, cot)
    perm = np.random.default_rng(1).permutation(B)
    cp = {k: (None if v is None else (v[perm] if k in ("cost", "qf", "dqf") else v[:, perm])) for k, v in cot.items()}
    gp = device_grads("ur5", q[perm], dq[perm], path[:, perm], pv[:, perm], grav, frame, off, cp)
    for k in ("q0", "dq0"):
        assert np.array_equal(gp[k], g[k][perm]), k
    for k in ("path", "pv"):
        assert np.array_equal(gp[k], g[k][:, perm]), k
    tl = lambda a, ax: np.concatenate([a, a], axis=ax)  # noqa: E731
    ct = {k: (None if v is None else tl(v, 0 if k in ("cost", "qf", "dqf") else 1)) for k, v in cot.items()}
    g2 = device_grads("ur5", tl(q, 0), tl(dq, 0), tl(path, 1), tl(pv, 1), grav, frame, off, ct)
    assert np.array_equal(g2["q0"][:B], g["q0"]) and np.array_equal(g2["q0"][B:], g["q0"])
    assert np.array_equal(g2["path"][:, B:], g["path"])
    # the forward outputs under grad are those of a value-only call
    c = _ctrl("ur5", _t(KP, grad=True), _t(KV), grav)
    qt = _t(q, grad=True)
    outs = c.rollout_path(qt, _t(dq), _t(path, grad=True), path_velocity=_t(pv), ref_frame=frame, xyz_offset=off)
    with torch.no_grad():
        ref = _ctrl("ur5", KP, KV, grav).rollout_path(_t(q), _t(dq), _t(path), path_velocity=_t(pv), ref_frame=frame,
                                                       xyz_offset=off)
    for a, b in zip((outs[0], outs[1], outs[3]), (ref[0], ref[1], ref[3])):
        assert torch.equal(a.detach(), b)
    for k in ref[2]:
        assert torch.equal(outs[2][k].detach(), ref[2][k]), k


@pytest.mark.gpu
def test_gain_gradients_against_central_differences_of_device_rollouts():
    import torch

    B, S = 64, 40
    q, dq, path, pv, grav, frame, off = joint_inputs("ur5", "per_grav", B, S, seed=10)
    cot = dict(cost=np.ones(B))
    g = device_grads("ur5", q, dq, path, pv, grav, frame, off, cot)

    def f(kp, kv):
        with torch.no_grad():
            return _ctrl("ur5", kp, kv, grav).rollout_path(_t(q), _t(dq), _t(path), dt=DT, ref_frame=frame,
                                                            xyz_offset=off, effort_weight=EFFORT)[3].sum().item()

    h = 1e-4
    for k, fd in (("kp", (f(KP + h, KV) - f(KP - h, KV)) / (2 * h)), ("kv", (f(KP, KV + h) - f(KP, KV - h)) / (2 * h))):
        assert abs(fd - float(g[k])) <= 1e-6 * max(1.0, abs(fd)), (k, fd, g[k])


@pytest.mark.gpu
def test_tensor_kp_with_the_default_kv_keeps_sqrt_kp_in_the_graph():
    """Joint(rc, kp=<0-d tensor>) sets kv = sqrt(kp): d cost/d kp = g_kp + g_kv / (2 sqrt(kp))"""
    import torch

    B, S = 32, 20
    q, dq, path, pv, grav, frame, off = joint_inputs("ur5", "per_grav", B, S, seed=12)
    g = device_grads("ur5", q, dq, path, pv, grav, frame, off, dict(cost=np.ones(B)), kp=KP, kv=np.sqrt(KP))
    kp = _t(KP, grad=True)
    c = _ctrl("ur5", kp, None, grav)
    cost = c.rollout_path(_t(q), _t(dq), _t(path), dt=DT, ref_frame=frame, xyz_offset=off, effort_weight=EFFORT)[3]
    (gk,) = torch.autograd.grad(cost.sum(), [kp])
    want = float(g["kp"]) + float(g["kv"]) / (2 * np.sqrt(KP))
    assert abs(gk.item() - want) <= 1e-12 * max(1.0, abs(want)), (gk.item(), want)


# Adam on the joint path from InverseKinematics.generate_path, through the closed loop, so that the tracked end
# effector follows the Cartesian track the plan was made for (the forward kinematics of the planned path): the PD loop
# lags behind the plan, and the refined path leads it.  On an H100 the 80 steps cut the loss to 0.25 of its start.
ADAM_STEPS, ADAM_LR, ADAM_FACTOR = 80, 5e-3, 0.5


@pytest.mark.gpu
def test_adam_on_the_ik_path_lowers_the_cartesian_tracking_loss():
    import torch

    from abr_control_b200 import controllers
    from abr_control_b200.controllers.path_planners import inverse_kinematics

    c = _ctrl("ur5", 300.0, 35.0)
    rc = c.robot_config
    B, S = 16, 80
    rng = np.random.default_rng(3)
    q0 = torch.as_tensor(rng.uniform(-1.0, 1.0, (B, 6)) + np.array([0, -1.2, 1.4, 0, 0.6, 0]), device=_dev())
    x0 = rc.Tx("EE", q0)
    targets = torch.cat([x0 + torch.as_tensor(rng.uniform(-0.1, 0.1, (B, 3)), device=_dev()),
                         torch.as_tensor(rng.uniform(-np.pi, np.pi, (B, 3)), device=_dev())], 1).contiguous()
    pos, _ = inverse_kinematics.InverseKinematics(rc).generate_path(q0, targets, n_timesteps=S, dt=0.01)
    plan = pos.permute(1, 0, 2).contiguous()
    x_ref = rc.Tx("EE", plan.reshape(-1, 6)).reshape(S, B, 3)
    dq0 = torch.zeros_like(q0)
    path = plan.clone().requires_grad_()

    def loss_of(p):
        _, _, tr, _ = c.rollout_path(q0, dq0, p, record=("x",))
        return ((tr["x"] - x_ref) ** 2).sum()

    opt = torch.optim.Adam([path], lr=ADAM_LR)
    first = None
    for _ in range(ADAM_STEPS):
        opt.zero_grad()
        loss = loss_of(path)
        first = loss.item() if first is None else first
        loss.backward()
        opt.step()
    with torch.no_grad():
        last = loss_of(path).item()
    print(f"Adam on the IK path: loss {first:.4e} -> {last:.4e} ({last / first:.3f})")
    assert last < ADAM_FACTOR * first, (first, last)
