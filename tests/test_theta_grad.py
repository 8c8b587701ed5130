"""Gradients with respect to the link inertias theta (``link_inertia[1:]`` flattened): ``simulate``,
``forward_dynamics`` and ``inverse_dynamics`` with ``theta=``, and ``abrb_plant_rollout_theta_vjp_*``.

Semantics (include/abrb.h, DESIGN.md S3.8): per trajectory,
``g_theta = sum_t [-Y(q_t, dq_t, ddq_t)^T w_t + c_g Y(q_t, 0, 0)^T gu_t]``, ``w_t = gu_t - 2 e gc tau_t - gr_t``.

CPU part: the kernel's per-state function (abrb_theta.cuh) runs on the host through tests/hostsim/thetasim.cpp (TEST
INFRASTRUCTURE, never loaded by the package), fed by the host adjoint of abrb_plant_rollout_vjp_*, against central
differences of the NumPy plant over theta and against a forward-mode dual rollout whose chain carries a theta
tangent; argument checking of the C entry points and of the Python methods.  GPU part: the kernel against the shim,
gradcheck, full size, bit identities, and output-error identification end to end.
"""
import ctypes as C
import os

import numpy as np
import pytest

from abr_control_b200 import _abi
from oracle import ident_oracle, rbd_oracle
from test_generic_chains import random_chain
from test_identification import perturbed, sinusoid_paths, with_theta
from test_plant import _build, _p, oracle_simulate
from test_plant_grad import random_cotangents, shim_vjp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ARMS = ("ur5", "jaco2", "threejoint", "twojoint")
RANDOM = tuple(f"rand{n}_{'ortho' if o else 'shear'}" for n in range(1, 8) for o in (True, False))
DT = 1e-3
# the rollout variants: (shared u, path, compensate_gravity, effort weight, cotangents given)
ALL = ("cost", "qf", "dqf", "q", "dq", "u", "x")
CASES = {
    "comp_path_effort_records": (False, True, True, 1e-2, ALL),
    "plain_path_effort_records": (False, True, False, 1e-2, ALL),
    "comp_final_state_only": (False, False, True, 0.0, ("qf", "dqf")),
    "plain_final_state_only": (False, False, False, 0.0, ("qf", "dqf")),
    "shared_u_comp_cost_and_torques": (True, True, True, 1e-2, ("cost", "u")),
}


def _chain(name):
    if name.startswith("rand"):
        n, kind = name[4:].split("_")
        return random_chain(int(n), kind == "ortho", seed=7 * int(n) + (kind == "ortho"))
    return _abi.load_arm_json(name)


@pytest.fixture(scope="module")
def thetasim(tmp_path_factory):
    return _build(tmp_path_factory, "thetasim")


def case_inputs(desc, case, B, S, seed):
    """start states, torques about the gravity hold (residual torques with compensation) and a path near the start"""
    shared, with_path, comp, effort, which = CASES[case]
    n = desc["n_joints"]
    ch = rbd_oracle.ChainOracle(desc)
    rng = np.random.default_rng(seed)
    q = rng.uniform(-np.pi, np.pi, (B, n))
    dq = rng.uniform(-0.5, 0.5, (B, n))
    hold = np.zeros((B, n)) if comp else -ch.g(q)
    scale = 1.0 + 0.1 * np.abs(hold).max()
    u = (hold[0][None] + scale * rng.normal(size=(S, n))) if shared else (hold[None] + scale * rng.normal(size=(S, B, n)))
    path = None
    if with_path:
        x0 = ch.Tx("EE", q)
        path = np.concatenate([x0[None] + 0.05 * rng.normal(size=(S, B, 3)), np.zeros((S, B, 3))], axis=2)
        path = np.ascontiguousarray(path[:, 0] if shared else path)
    cot = random_cotangents(rng, S, B, n, which)
    return q, dq, np.ascontiguousarray(u), path, comp, effort, cot


def shim_theta_vjp(ts, desc, q0, dq0, u, comp, effort, q_traj, dq_traj, gu, g_cost, g_u, f32=0):
    cd = _abi.chain_desc_from_dict(desc)
    n, B, S = cd.n_joints, len(q0), u.shape[0]
    out = np.zeros((B, 6 * n))
    c = lambda a: None if a is None else np.ascontiguousarray(a, dtype=np.float64)  # noqa: E731
    rc = ts.th_rollout_theta_vjp(C.byref(cd), f32, _p(c(q0)), _p(c(dq0)), _p(c(u)), n if u.ndim == 3 else 0, int(comp),
                                 S, C.c_double(effort), _p(c(q_traj)), _p(c(dq_traj)), _p(c(gu)), _p(c(g_cost)),
                                 _p(c(g_u)), _p(out), C.c_int64(B))
    assert rc == 0
    return out


def shim_theta_jvp(ts, desc, q0, dq0, u, path, comp, effort, v):
    cd = _abi.chain_desc_from_dict(desc)
    n, B, S = cd.n_joints, len(q0), u.shape[0]
    t = {k: np.zeros((S, B, 3 if k == "x" else n)) for k in ("q", "dq", "u", "x")}
    t.update(cost=np.zeros(B), qf=np.zeros((B, n)), dqf=np.zeros((B, n)))
    rc = ts.th_rollout_theta_jvp(C.byref(cd), 0, ts.hs_frame_id(n, b"EE"), None, _p(np.ascontiguousarray(q0)),
                                 _p(np.ascontiguousarray(dq0)), _p(u), n if u.ndim == 3 else 0, int(comp),
                                 _p(path), 0 if path is None or path.ndim == 2 else 6, S, C.c_double(DT),
                                 C.c_double(effort), _p(np.ascontiguousarray(v, dtype=np.float64)),
                                 *[_p(t[k]) for k in ("q", "dq", "u", "x", "cost", "qf", "dqf")], C.c_int64(B))
    assert rc == 0
    return t


def host_theta_grad(ts, desc, q, dq, u, path, comp, effort, cot, f32=0):
    """(B, 6n) per-trajectory gradient: the host adjoint for gu, then the host theta pass"""
    cd = _abi.chain_desc_from_dict(desc)
    fw = oracle_simulate(desc, q, dq, u, DT, path, effort, comp)
    gu, _, _ = shim_vjp(ts, cd, q, dq, u, path, comp, "EE", None, fw["q"], fw["dq"], cot, f32=f32, effort=effort)
    return shim_theta_vjp(ts, desc, q, dq, u, comp, effort, fw["q"], fw["dq"], gu, cot["cost"], cot["u"], f32), fw


def _loss(o, cot):
    """per-trajectory pairing of the rollout's outputs with the cotangents"""
    keys = dict(cost="cost", qf="q_final", dqf="dq_final", q="q", dq="dq", u="u", x="x")
    B = len(o["cost"])
    total = np.zeros(B)
    for k, c in cot.items():
        if c is None:
            continue
        v = c * o[keys[k]]
        total += v if v.ndim == 1 else (v.sum(-1) if v.ndim == 2 else v.sum((0, 2)))
    return total


# ---------------------------------------------------------------------------------------------- host
@pytest.mark.parametrize("case", list(CASES))
@pytest.mark.parametrize("name", ARMS + RANDOM)
def test_host_theta_gradient_vs_central_differences(thetasim, name, case):
    """every entry of every trajectory's row against central differences of the NumPy plant over theta +- h e_p, within
    1e-6 of the row's largest entry plus the differences' own rounding, 1e3 eps |loss| / h"""
    desc = _chain(name)
    n, B, S = desc["n_joints"], 3, 6
    q, dq, u, path, comp, effort, cot = case_inputs(desc, case, B, S, 11)
    got, _ = host_theta_grad(thetasim, desc, q, dq, u, path, comp, effort, cot)
    th = ident_oracle.theta(desc)
    fd = np.zeros((B, 6 * n))
    rnd = 1e3 * np.finfo(np.float64).eps * np.abs(_loss(oracle_simulate(desc, q, dq, u, DT, path, effort, comp), cot))
    for p in range(6 * n):
        h = 1e-6 * max(1.0, abs(th[p]))
        e = np.zeros(6 * n)
        e[p] = h
        lp = _loss(oracle_simulate(with_theta(desc, th + e), q, dq, u, DT, path, effort, comp), cot)
        lm = _loss(oracle_simulate(with_theta(desc, th - e), q, dq, u, DT, path, effort, comp), cot)
        fd[:, p] = (lp - lm) / (2 * h)
    tol = 1e-6 * np.abs(fd).max(1, keepdims=True) + rnd[:, None] / 1e-6
    assert np.all(np.abs(got - fd) <= tol), (name, case, (np.abs(got - fd) / tol).max())


@pytest.mark.parametrize("case", list(CASES))
@pytest.mark.parametrize("name", ARMS + RANDOM)
def test_host_theta_gradient_dot_product(thetasim, name, case):
    """<g_theta, v> equals the tangent of a dual rollout of the phased plant step along v (inertial constants only)
    paired with the same cotangents, within 1e-12 of the larger side's magnitude before cancellation plus 1e-14 of the
    paired outputs' own magnitude (the rounding of the rollout where theta's effect is tiny)"""
    desc = _chain(name)
    n, B, S = desc["n_joints"], 4, 7
    q, dq, u, path, comp, effort, cot = case_inputs(desc, case, B, S, 12)
    got, fw = host_theta_grad(thetasim, desc, q, dq, u, path, comp, effort, cot)
    v = np.random.default_rng(13).normal(size=6 * n) * np.maximum(np.abs(ident_oracle.theta(desc)), 1e-3)
    t = shim_theta_jvp(thetasim, desc, q, dq, u, path, comp, effort, v)
    lhs = float(np.sum(got @ v))
    rhs = float(sum(np.sum(cot[k] * t[k]) for k in cot if cot[k] is not None))
    scale = max(float(np.sum(np.abs(got) @ np.abs(v))),
                float(sum(np.sum(np.abs(cot[k] * t[k])) for k in cot if cot[k] is not None)))
    size = float(np.sum(np.abs(_loss({k: np.abs(x) for k, x in fw.items()}, {k: None if c is None else np.abs(c)
                                                                            for k, c in cot.items()}))))
    assert abs(lhs - rhs) <= 1e-12 * scale + 1e-14 * size, (name, case, lhs, rhs, scale, size)


@pytest.mark.parametrize("name", ("ur5", "rand7_shear", "rand2_ortho"))
def test_host_fp32_theta_gradient_vs_fp64(thetasim, name):
    """the fp32 instantiation (fp32 adjoint and theta pass) within 2e-3 of the fp64 row's largest entry"""
    desc = _chain(name)
    q, dq, u, path, comp, effort, cot = case_inputs(desc, "comp_path_effort_records", 4, 16, 14)
    g64, _ = host_theta_grad(thetasim, desc, q, dq, u, path, comp, effort, cot)
    g32, _ = host_theta_grad(thetasim, desc, q, dq, u, path, comp, effort, cot, f32=1)
    assert np.all(np.abs(g32 - g64) <= 2e-3 * np.abs(g64).max(1, keepdims=True))


def test_host_recorded_final_state_does_not_enter(thetasim):
    """ddq_t is recomputed from the state before step t and its torque: the last recorded state (after the last step)
    never enters, so changing it leaves every row bit-identical"""
    desc = _chain("ur5")
    q, dq, u, path, comp, effort, cot = case_inputs(desc, "comp_path_effort_records", 3, 5, 15)
    fw = oracle_simulate(desc, q, dq, u, DT, path, effort, comp)
    gu, _, _ = shim_vjp(thetasim, _abi.chain_desc_from_dict(desc), q, dq, u, path, comp, "EE", None, fw["q"], fw["dq"],
                        cot, effort=effort)
    ref = shim_theta_vjp(thetasim, desc, q, dq, u, comp, effort, fw["q"], fw["dq"], gu, cot["cost"], cot["u"])
    qt, dqt = fw["q"].copy(), fw["dq"].copy()
    qt[-1] += 0.3
    dqt[-1] -= 2.0
    got = shim_theta_vjp(thetasim, desc, q, dq, u, comp, effort, qt, dqt, gu, cot["cost"], cot["u"])
    assert np.array_equal(got, ref)
    # and the state before a step does enter
    dqt = fw["dq"].copy()
    dqt[1] += 0.1
    assert not np.array_equal(shim_theta_vjp(thetasim, desc, q, dq, u, comp, effort, fw["q"], dqt, gu, cot["cost"],
                                             cot["u"]), ref)


def test_host_zero_steps_give_zeros(thetasim):
    desc = _chain("jaco2")
    q = np.ones((2, 6))
    z = np.zeros((0, 2, 6))
    assert np.array_equal(shim_theta_vjp(thetasim, desc, q, q, z, True, 0.1, z, z, z, None, None), np.zeros((2, 36)))


# ---------------------------------------------------------------------------------------------- ABI and Python
@pytest.fixture(scope="module")
def native():
    from abr_control_b200 import _lib

    lib = _lib.lib()
    cd = _abi.chain_desc_from_dict(_abi.load_arm_json("ur5"))
    m = C.c_void_p()
    _lib.check(lib.abrb_model_create(C.byref(cd), C.byref(m)))
    yield lib, m, np.zeros(4096)
    lib.abrb_model_destroy(m)


FNS = ["abrb_plant_rollout_theta_vjp_f64", "abrb_plant_rollout_theta_vjp_f32"]
_KEYS = ("m", "q0", "dq0", "u", "us", "comp", "steps", "ew", "qt", "dqt", "gu", "gc", "gut", "gth", "B", "stream")


def _args(**over):
    a = {k: None for k in _KEYS}
    a.update(us=0, comp=0, steps=4, ew=0.0, B=8)
    a.update(over)
    return [a[k] for k in _KEYS]


@pytest.mark.parametrize("fn", FNS)
def test_abi_rejects_bad_arguments_before_any_device_work(native, fn):
    lib, m, buf = native
    f = getattr(lib, fn)
    p = buf.ctypes.data
    ok = dict(m=m, q0=p, dq0=p, u=p, qt=p, dqt=p, gu=p, gth=p)
    bad = [
        (dict(m=None), "model"),
        (dict(q0=None), "NULL q0"),
        (dict(dq0=None), "NULL dq0"),
        (dict(u=None), "NULL u"),
        (dict(qt=None), "NULL q_traj"),
        (dict(dqt=None), "NULL dq_traj"),
        (dict(gu=None), "NULL gu"),
        (dict(gth=None), "NULL g_theta"),
        (dict(us=3), "u_stride"),
        (dict(steps=-1), "steps"),
        (dict(B=-1), "B < 0"),
        (dict(ew=-1.0), "effort_weight"),
        (dict(ew=float("inf")), "effort_weight"),
        (dict(q0=p + 1), "misaligned pointer (q0)"),
        (dict(dqt=p + 2), "misaligned pointer (dq_traj)"),
        (dict(gc=p + 1), "misaligned pointer (g_cost)"),
        (dict(gut=p + 2), "misaligned pointer (g_u_traj)"),
        (dict(gth=p + 1), "misaligned pointer (g_theta)"),
    ]
    for over, word in bad:
        rc = f(*_args(**{**ok, **over}))
        assert rc == _abi.EINVAL, (over, rc)
        msg = lib.abrb_last_error().decode()
        assert msg.startswith("abrb_plant_rollout_theta_vjp") and word in msg, (over, msg)
    assert f(*_args(m=m, B=0)) == 0  # B == 0 is a no-op whatever the pointers
    if lib.abrb_device_count() <= 0:  # steps == 0 needs no torques, records or gu, but writes zeros on the device
        assert f(*_args(m=m, q0=p, dq0=p, gth=p, steps=0)) == _abi.ECUDA
        assert "no CUDA device" in lib.abrb_last_error().decode()


def test_signatures_and_header_cover_the_theta_vjp():
    from abr_control_b200 import _lib

    with open(os.path.join(ROOT, "include", "abrb.h")) as fh:
        hdr = fh.read()
    for fn in FNS:
        res, args = _lib.SIGNATURES[fn]
        assert res is C.c_int and len(args) == 16 and args[7] is C.c_double and args[14] is C.c_int64
        assert args[4] is C.c_int and args[5] is C.c_int and args[6] is C.c_int
        assert f"int {fn}(" in hdr
        assert getattr(_lib.lib(), fn) is not None


def test_python_theta_argument_checks(monkeypatch):
    torch = pytest.importorskip("torch")
    import abr_control_b200.arms as arms

    rc = arms.ur5.Config()
    x, u = np.zeros((2, 6)), np.zeros((3, 2, 6))
    th = rc.inertial_parameters()
    for bad in (th[:-1], np.full(36, np.inf), th.reshape(6, 6)):
        for call in (lambda t: rc.forward_dynamics(x, x, x, theta=t), lambda t: rc.inverse_dynamics(x, x, x, theta=t),
                     lambda t: rc.simulate(x, x, u, theta=t)):
            with pytest.raises(ValueError, match="36 finite"):
                call(bad)
    for bad in (torch.as_tensor(th), torch.as_tensor(th, dtype=torch.float16)):  # CPU or half tensors
        with pytest.raises(ValueError, match="float32/float64 CUDA tensor"):
            rc.simulate(x, x, u, theta=bad)

    # theta=None never builds a second model
    def no(*a, **k):
        raise AssertionError("with_link_inertia called")

    monkeypatch.setattr(type(rc), "with_link_inertia", no)
    for call in (lambda: rc.forward_dynamics(x, x, x), lambda: rc.inverse_dynamics(x, x, x),
                 lambda: rc.simulate(x, x, u)):
        try:
            call()
        except AssertionError:
            raise
        except Exception:  # no device here: the value path fails later, at the launch
            pass


# ============================================================================================== GPU
def _t(a, dtype=None):
    import torch

    return torch.as_tensor(np.asarray(a, dtype=dtype or np.float64), device="cuda")


def _cfg(desc, dtype=np.float64):
    from abr_control_b200.arms.base_config import BaseConfig

    return BaseConfig(desc, dtype=dtype)


def device_theta_grad(rc, q, dq, u, path, comp, effort, cot, dtype=None):
    """(B, 6n) rows of the kernel for the cotangents cot (host arrays), through the C entry points directly"""
    import torch

    from abr_control_b200 import _lib

    td = torch.float32 if dtype == np.float32 else torch.float64
    T = lambda a: None if a is None else _t(a, dtype).to(td).contiguous()  # noqa: E731
    q0, dq0, uu = T(q), T(dq), T(u)
    with torch.no_grad():
        qf, dqf, tr, cost = rc.simulate(q0, dq0, uu, dt=DT, path=T(path), effort_weight=effort, compensate_gravity=comp)
    B, n = q0.shape
    S = uu.shape[0]
    cc = [T(cot[k]) for k in ("cost", "qf", "dqf", "q", "dq", "u", "x")]
    gu, gq0, gdq0 = torch.empty((S, B, n), dtype=td, device="cuda"), torch.empty_like(q0), torch.empty_like(q0)
    L = _lib.lib()
    f32 = td == torch.float32
    p = lambda t: None if t is None else t.data_ptr()  # noqa: E731
    pth = T(path)
    _lib.check((L.abrb_plant_rollout_vjp_f32 if f32 else L.abrb_plant_rollout_vjp_f64)(
        rc.handle, rc.frame_id("EE"), None, p(q0), p(dq0), p(uu), 0 if uu.dim() == 2 else n, int(comp), p(pth),
        0 if pth is None or pth.dim() == 2 else 6, S, DT, effort, p(tr["q"]), p(tr["dq"]), *[p(c) for c in cc], p(gu),
        p(gq0), p(gdq0), B, torch.cuda.current_stream().cuda_stream))
    gth = torch.empty((B, 6 * n), dtype=td, device="cuda")
    _lib.check((L.abrb_plant_rollout_theta_vjp_f32 if f32 else L.abrb_plant_rollout_theta_vjp_f64)(
        rc.handle, p(q0), p(dq0), p(uu), 0 if uu.dim() == 2 else n, int(comp), S, effort, p(tr["q"]), p(tr["dq"]),
        p(gu), p(cc[0]), p(cc[5]), p(gth), B, torch.cuda.current_stream().cuda_stream))
    return gth, tr


@pytest.mark.gpu
@pytest.mark.parametrize("f32", [0, 1])
@pytest.mark.parametrize("name", ARMS + ("rand1_ortho", "rand2_shear", "rand5_ortho", "rand7_ortho", "rand7_shear"))
def test_device_vs_shim(thetasim, name, f32):
    """fp64 within 1e-10 of the shim's row scale (different summation order over the steps); fp32 within 1e-3 of the
    fp32 shim, both fed the device's own records"""
    desc = _chain(name)
    rc = _cfg(desc)
    for case in ("comp_path_effort_records", "plain_path_effort_records", "shared_u_comp_cost_and_torques"):
        q, dq, u, path, comp, effort, cot = case_inputs(desc, case, 37, 45, 16)
        dt = np.float32 if f32 else np.float64
        got, tr = device_theta_grad(rc, q, dq, u, path, comp, effort, cot, dt)
        h = lambda a: None if a is None else np.asarray(a, dtype=dt).astype(np.float64)  # noqa: E731
        gu, _, _ = shim_vjp(thetasim, _abi.chain_desc_from_dict(desc), h(q), h(dq), h(u), h(path), comp, "EE", None,
                            tr["q"].double().cpu().numpy(), tr["dq"].double().cpu().numpy(),
                            {k: h(v) for k, v in cot.items()}, f32=f32, effort=effort)
        ref = shim_theta_vjp(thetasim, desc, h(q), h(dq), h(u), comp, effort, tr["q"].double().cpu().numpy(),
                             tr["dq"].double().cpu().numpy(), gu, h(cot["cost"]), h(cot["u"]), f32)
        g = got.double().cpu().numpy()
        assert g.shape == ref.shape and got.element_size() == (4 if f32 else 8)
        err = (np.abs(g - ref) / np.abs(ref).max(1, keepdims=True)).max()
        assert err <= (1e-3 if f32 else 1e-10), (name, case, err)


@pytest.mark.gpu
def test_gradcheck_theta_with_state_and_torques():
    import torch

    for name in ("ur5", "rand7_shear"):
        desc = _chain(name)
        rc = _cfg(desc)
        n = desc["n_joints"]
        th = torch.as_tensor(ident_oracle.theta(desc), device="cuda").requires_grad_()
        gen = np.random.default_rng(4)
        q, dq, x = (_t(gen.uniform(-1, 1, (3, n))).requires_grad_() for _ in range(3))
        for fn in (rc.forward_dynamics, rc.inverse_dynamics):
            assert torch.autograd.gradcheck(lambda a, b, c, t: fn(a, b, c, theta=t), (q, dq, x, th), eps=1e-6,
                                            atol=1e-6, rtol=1e-5), (name, fn.__name__)
        S, B = 5, 3
        q0 = _t(gen.uniform(-1, 1, (B, n))).requires_grad_()
        dq0 = _t(gen.uniform(-0.3, 0.3, (B, n))).requires_grad_()
        path = _t(gen.uniform(-0.5, 0.5, (S, B, 6)))
        for comp in (False, True):
            for shared in (False, True):
                u = _t(gen.normal(size=(S, n) if shared else (S, B, n))).requires_grad_()

                def f(qq, dd, uu, tt):
                    qf, dqf, tr, cost = rc.simulate(qq, dd, uu, dt=0.01, path=path, effort_weight=0.01,
                                                    compensate_gravity=comp, theta=tt)
                    return (qf, dqf, cost) + tuple(tr[k] for k in ("q", "dq", "u", "x"))

                assert torch.autograd.gradcheck(f, (q0, dq0, u, th), eps=1e-6, atol=1e-6, rtol=1e-5), (name, comp,
                                                                                                       shared)


def _full_inputs(arm, B, S, seed, dtype=np.float64):
    """the arm's model, start states, a path that moves the control point away from the start, random torques"""
    import torch

    import abr_control_b200.arms as arms

    rc = getattr(arms, arm).Config(dtype=dtype)
    g = torch.Generator(device="cuda").manual_seed(seed)
    q = torch.rand((B, 6), device="cuda", generator=g, dtype=torch.float64) * 2 * np.pi
    dq = torch.rand((B, 6), device="cuda", generator=g, dtype=torch.float64) - 0.5
    x0 = getattr(arms, arm).Config().Tx("EE", q)
    ramp = torch.linspace(0, 1, S, device="cuda", dtype=torch.float64)[:, None, None]
    end = torch.rand((B, 3), device="cuda", generator=g, dtype=torch.float64) * 0.2 - 0.1
    path = torch.cat([x0[None] + ramp * end[None], torch.zeros((S, B, 3), device="cuda", dtype=torch.float64)], -1)
    u = torch.randn((S, B, 6), device="cuda", generator=g, dtype=torch.float64)
    return rc, q, dq, path.contiguous(), u


@pytest.mark.gpu
@pytest.mark.parametrize("arm", ["ur5", "jaco2"])
def test_full_size_theta_gradient(arm):
    """4 096 x 128 with a path, an effort weight and compensate_gravity: theta's gradient against central differences
    along three random directions (1e-6 relative) and against the composed regressor route (1e-12 relative); the fp32
    kernel within 1e-3 of fp64"""
    import torch

    B, S = 4096, 128
    rc, q, dq, path, u = _full_inputs(arm, B, S, 51)
    kw = dict(dt=DT, path=path, effort_weight=1e-4, compensate_gravity=True)
    th0 = torch.as_tensor(rc.inertial_parameters(), device="cuda")
    th = th0.clone().requires_grad_()
    _, _, tr, cost = rc.simulate(q, dq, u, record=("q", "dq", "u"), theta=th, **kw)
    cost.sum().backward()
    gen = torch.Generator(device="cuda").manual_seed(5)
    with torch.no_grad():
        for _ in range(3):
            v = torch.randn(th0.shape, device="cuda", generator=gen, dtype=torch.float64) * th0.abs().clamp_min(1e-3)
            h = 1e-6
            cp = rc.simulate(q, dq, u, record=(), theta=th0 + h * v, **kw)[3].sum()
            cm = rc.simulate(q, dq, u, record=(), theta=th0 - h * v, **kw)[3].sum()
            fd = float((cp - cm) / (2 * h))
            an = float((th.grad * v).sum())
            print(f"{arm}: theta gradient vs central differences {abs(fd - an) / max(1.0, abs(an)):.2e}")
            assert abs(fd - an) < 1e-6 * max(1.0, abs(an)), (fd, an)
    # the composed route: gu from the adjoint, ddq from forward_dynamics, Y from the regressor, contracted by matmul
    with torch.no_grad():
        uu = u.clone().requires_grad_()
        with torch.enable_grad():
            _, _, tr2, c2 = rc.simulate(q, dq, uu, record=("q", "dq", "u"), **kw)
            c2.sum().backward()
        gu = uu.grad
        qp = torch.cat([q[None], tr2["q"][:-1]]).reshape(-1, 6)
        dqp = torch.cat([dq[None], tr2["dq"][:-1]]).reshape(-1, 6)
        tau = tr2["u"].reshape(-1, 6)
        w = gu.reshape(-1, 6) - 2e-4 * tau
        ddq = rc.forward_dynamics(qp, dqp, tau)
        ref = torch.zeros(36, dtype=torch.float64, device="cuda")
        for i in range(0, len(qp), 65536):
            s = slice(i, i + 65536)
            Y = rc.inverse_dynamics_regressor(qp[s], dqp[s], ddq[s])
            Y0 = rc.inverse_dynamics_regressor(qp[s], torch.zeros_like(qp[s]), torch.zeros_like(qp[s]))
            ref += -torch.matmul(w[s][:, None, :], Y)[:, 0].sum(0) + torch.matmul(gu.reshape(-1, 6)[s][:, None, :],
                                                                                  Y0)[:, 0].sum(0)
        rel = float((th.grad - ref).abs().max() / ref.abs().max())
        print(f"{arm}: theta gradient vs composed regressor route {rel:.2e}")
        assert rel < 1e-12
    # fp32
    rc32 = _full_inputs(arm, 1, 1, 0, np.float32)[0]
    th32 = th0.float().clone().requires_grad_()
    _, _, _, c32 = rc32.simulate(q.float(), dq.float(), u.float(), record=(), theta=th32, **dict(kw, path=path.float()))
    c32.sum().backward()
    e32 = float((th32.grad.double() - th.grad).abs().max() / th.grad.abs().max())
    print(f"{arm}: fp32 theta gradient vs fp64 {e32:.2e}")
    assert e32 < 1e-3


@pytest.mark.gpu
def test_theta_gradient_bit_identities():
    import torch

    B, S = 256, 40
    rc, q, dq, path, u = _full_inputs("ur5", B, S, 61)
    kw = dict(dt=DT, effort_weight=1e-3, compensate_gravity=True)
    th0 = torch.as_tensor(rc.inertial_parameters(), device="cuda")

    def rows(qq, dd, uu, pp):
        desc = rc.desc
        cot = dict(cost=np.ones(B), qf=None, dqf=None, q=None, dq=None, u=np.full((S, B, 6), 0.5), x=None)
        g, _ = device_theta_grad(_cfg(desc), qq.cpu().numpy(), dd.cpu().numpy(), uu.cpu().numpy(), pp.cpu().numpy(),
                                 True, 1e-3, cot)
        return g

    r1, r2 = rows(q, dq, u, path), rows(q, dq, u, path)
    assert torch.equal(r1, r2)
    perm = torch.randperm(B, device="cuda")
    assert torch.equal(rows(q[perm], dq[perm], u[:, perm], path[:, perm]), r1[perm])
    # a shared (S, n) sequence gives the rows of its expansion
    us = u[:, 0].contiguous()
    cot = dict(cost=np.ones(B), qf=None, dqf=None, q=None, dq=None, u=None, x=None)
    a, _ = device_theta_grad(rc, q.cpu().numpy(), dq.cpu().numpy(), us.cpu().numpy(), None, True, 1e-3, cot)
    b, _ = device_theta_grad(rc, q.cpu().numpy(), dq.cpu().numpy(), us[:, None].expand(S, B, 6).cpu().numpy(), None,
                             True, 1e-3, cot)
    assert torch.equal(a, b)
    # simulate(theta=) equals with_link_inertia(theta).simulate, and the forward outputs do not depend on grad
    th = th0 * 1.1
    ref = rc.with_link_inertia(th.cpu().numpy()).simulate(q, dq, u, path=path, **kw)
    got = rc.simulate(q, dq, u, path=path, theta=th, **kw)
    got_np = rc.simulate(q, dq, u, path=path, theta=th.cpu().numpy(), **kw)
    out = rc.simulate(q, dq, u, path=path, theta=th.clone().requires_grad_(), **kw)
    for o in (got, got_np, out):
        assert all(torch.equal(o[i], ref[i]) for i in (0, 1, 3))
        assert all(torch.equal(o[2][k], ref[2][k]) for k in ("q", "dq", "u", "x"))
    assert out[3].requires_grad and not got[3].requires_grad
    for kind in ("forward_dynamics", "inverse_dynamics"):
        x = u[0]
        r = getattr(rc.with_link_inertia(th.cpu().numpy()), kind)(q, dq, x)
        assert torch.equal(getattr(rc, kind)(q, dq, x, theta=th), r)
        o = getattr(rc, kind)(q, dq, x, theta=th.clone().requires_grad_())
        assert o.requires_grad and torch.equal(o.detach(), r)


def _windows(q_rec, u_rec, dq_rec, W, S):
    """B windows of S steps starting every S steps of a (T + 1, n) track: starts, torques, targets"""
    import torch

    starts = list(range(0, u_rec.shape[0] - S + 1, S))[:W]
    q0 = torch.stack([q_rec[s] for s in starts])
    dq0 = torch.stack([dq_rec[s] for s in starts])
    u = torch.stack([u_rec[s:s + S] for s in starts], 1).contiguous()
    target = torch.stack([q_rec[s + 1:s + S + 1] for s in starts], 1)
    return q0, dq0, u, target


@pytest.mark.gpu
def test_output_error_identification_end_to_end():
    """Record Joint rollouts of a perturbed UR5, cut them into windows that start at recorded states and replay the
    recorded torques without compensation; fit tied parameters phi (theta = T phi) from the nominal model with LBFGS
    on the position error.  Noise-free: the identifiable projection matches theta* to 1e-6.  With Gaussian noise on
    the recorded positions and the window start velocities free: closer to theta* than the equation-error fit on
    finite-differenced dq and ddq of the same noisy positions."""
    import torch

    import abr_control_b200.arms as arms
    from abr_control_b200 import controllers
    from abr_control_b200.arms import _ident
    from abr_control_b200.arms.base_config import BaseConfig

    nominal, true = arms.ur5.Config(), BaseConfig(perturbed("ur5", 7))
    n, B, T, dt = 6, 4, 1024, 1e-3
    q0, dq0, path, pv = (_t(a) for a in sinusoid_paths(n, B, T, dt, 8))
    _, _, tr, _ = controllers.Joint(true, kp=400.0, kv=40.0).rollout_path(q0, dq0, path, dt=dt, path_velocity=pv,
                                                                          record=("q", "dq", "u"))
    q_rec = torch.cat([q0[None], tr["q"]])  # (T + 1, B, n)
    dq_rec = torch.cat([dq0[None], tr["dq"]])
    th_true = true.inertial_parameters()
    Tm = _t(_ident.tie_matrix(n))
    phi0 = _t(_ident.tied(nominal.inertial_parameters(), n))
    # the identifiable directions, from the exact samples
    qp, dqp = q_rec[:-1].reshape(-1, n), dq_rec[:-1].reshape(-1, n)
    ddq = ((dq_rec[1:] - dq_rec[:-1]) / dt).reshape(-1, n)
    _, info = nominal.identify_link_inertia(qp, dqp, ddq, tr["u"].reshape(-1, n))
    Q = info["basis"]
    Wn, S = 64, 16  # windows per trajectory, steps per window

    def windows(qr, dqr):
        parts = [_windows(qr[:, b], tr["u"][:, b], dqr[:, b], Wn, S) for b in range(B)]
        return tuple(torch.cat([p[i] for p in parts], dim=1 if i in (2, 3) else 0) for i in range(4))

    def fit(qr, dqr, free_start, iters):
        """LBFGS on phi = phi0 + |phi0| s (and, when free_start, on the window start states), loss normalised by its
        start"""
        q0w, dq0w, uw, target = windows(qr, dqr)
        scale = phi0.abs().clamp_min(1e-6)
        s = torch.zeros_like(phi0, requires_grad=True)
        dq_s = torch.zeros_like(dq0w, requires_grad=True)
        q_s = torch.zeros_like(q0w, requires_grad=True)
        params = [s, q_s, dq_s] if free_start else [s]

        def loss_of():
            _, _, trw, _ = nominal.simulate(q0w + sigma * q_s, dq0w + 1e-2 * dq_s, uw, dt=dt, compensate_gravity=False,
                                            record=("q",), theta=Tm @ (phi0 + scale * s))
            return (trw["q"] - target).pow(2).sum()

        with torch.no_grad():
            l0 = float(loss_of())
        opt = torch.optim.LBFGS(params, lr=1, max_iter=iters, tolerance_grad=1e-15, tolerance_change=1e-20,
                                history_size=30, line_search_fn="strong_wolfe")

        def closure():
            opt.zero_grad()
            loss = loss_of() / l0
            loss.backward()
            return loss

        opt.step(closure)
        with torch.no_grad():
            print(f"LBFGS: loss {l0:.3e} -> {float(loss_of()):.3e}")
            return (Tm @ (phi0 + scale * s)).cpu().numpy()

    sigma = 1e-5  # rad, the noise on the recorded positions below
    th = fit(q_rec, dq_rec, False, 200)
    err = np.abs(Q.T @ (th - th_true)).max() / np.abs(th_true).max()
    print(f"output-error fit, noise-free: {err:.2e} of |theta*|")
    assert err <= 1e-6
    # noisy positions
    g = torch.Generator(device="cuda").manual_seed(9)
    q_noisy = q_rec + sigma * torch.randn(q_rec.shape, device="cuda", generator=g, dtype=torch.float64)
    dq_fd = torch.zeros_like(q_noisy)
    dq_fd[1:-1] = (q_noisy[2:] - q_noisy[:-2]) / (2 * dt)
    dq_fd[0], dq_fd[-1] = (q_noisy[1] - q_noisy[0]) / dt, (q_noisy[-1] - q_noisy[-2]) / dt
    th_oe = fit(q_noisy, dq_fd, True, 300)
    ddq_fd = (q_noisy[2:] - 2 * q_noisy[1:-1] + q_noisy[:-2]) / dt ** 2  # at samples 1 .. T - 1
    th_ee, _ = nominal.identify_link_inertia(q_noisy[1:-1].reshape(-1, n), dq_fd[1:-1].reshape(-1, n),
                                             ddq_fd.reshape(-1, n), tr["u"][1:].reshape(-1, n))
    e_oe = np.linalg.norm(Q.T @ (th_oe - th_true)) / np.linalg.norm(Q.T @ th_true)
    e_ee = np.linalg.norm(Q.T @ (th_ee - th_true)) / np.linalg.norm(Q.T @ th_true)
    print(f"noise {sigma:g} rad, windows of {S} steps: output error {e_oe:.3e}, equation error {e_ee:.3e}")
    assert e_oe < e_ee
