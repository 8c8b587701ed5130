"""Derivatives of the plant: ``Config.forward_dynamics_derivatives`` / ``inverse_dynamics_derivatives``
(``abrb_*_dynamics_derivatives_*``) and gradients of ``forward_dynamics``, ``inverse_dynamics`` and ``simulate`` through
``torch.autograd`` (``abrb_plant_rollout_vjp_*``).

Conventions (include/abrb.h): derivative blocks are (B, n, n), element [b, i, j] = d out_i / d in_j; the rollout's
vector-Jacobian product runs the adjoint recursion over the recorded states (DESIGN.md S3.6).

CPU part: the kernels' per-lane functions (abrb_grad.cuh) run on the host through tests/hostsim/gradsim.cpp (TEST
INFRASTRUCTURE, never loaded by the package) against central differences of the NumPy oracle, algebraic identities, a
dot-product test of the adjoint against a forward-mode dual rollout of plant_step, and argument checking of the C entry
points.  GPU part: the kernels against the shim, gradcheck, full-size runs, bit-identity properties and a small
optimisation.
"""
import ctypes as C

import numpy as np
import pytest

import cases
from abr_control_b200 import _abi
from oracle import rbd_oracle
from test_generic_chains import random_chain
from test_plant import (ARMS, DT, EFFORT, VARIANTS, _build, _desc, _p, oracle_forward, oracle_inverse,
                        oracle_simulate, shim_simulate, variant_inputs)

NS = list(range(1, 8))


@pytest.fixture(scope="module")
def gradsim(tmp_path_factory):
    return _build(tmp_path_factory, "gradsim")


@pytest.fixture(scope="module")
def plantsim(tmp_path_factory):
    return _build(tmp_path_factory, "plantsim")


def _chain(name):
    """(descriptor dict, ctypes descriptor) of an arm or of a random chain 'rand<n>_<ortho|shear>'"""
    if name.startswith("rand"):
        n, kind = name[4:].split("_")
        d = random_chain(int(n), kind == "ortho", seed=100 + int(n))
    else:
        d = _abi.load_arm_json(name)
    return d, _abi.chain_desc_from_dict(d)


CHAINS = list(ARMS) + [f"rand{n}_{k}" for n in NS for k in ("ortho", "shear")]


def _states(d, B, seed):
    n = d["n_joints"]
    rng = np.random.default_rng(seed)
    return (rng.uniform(-np.pi, np.pi, (B, n)), rng.uniform(-1, 1, (B, n)), rng.normal(size=(B, n)) * 3)


def shim_jac(gs, cd, kind, q, dq, x, f32=0):
    B, n = q.shape
    q, dq, x = (np.ascontiguousarray(a, dtype=np.float64) for a in (q, dq, x))
    out = [np.zeros((B, n, n)) for _ in range(3)]
    assert gs.gr_dyn_jac(C.byref(cd), f32, kind, _p(q), _p(dq), _p(x), C.c_int64(B), *[_p(o) for o in out]) == 0
    return out


def fd_jac(fn, q, dq, x, h=1e-6):
    """central differences of fn(q, dq, x) (B, n) along every input coordinate -> three (B, n, n) blocks"""
    B, n = q.shape
    out = []
    for which in range(3):
        J = np.zeros((B, n, n))
        for j in range(n):
            args_p = [q.copy(), dq.copy(), x.copy()]
            args_m = [q.copy(), dq.copy(), x.copy()]
            args_p[which][:, j] += h
            args_m[which][:, j] -= h
            J[:, :, j] = (fn(*args_p) - fn(*args_m)) / (2 * h)
        out.append(J)
    return out


def _rel(a, b, scale=None):
    """max over states of |a - b| / scale (default |b|), Frobenius norms per state"""
    scale = np.linalg.norm(b.reshape(len(b), -1), axis=1) if scale is None else scale
    return (np.linalg.norm((a - b).reshape(len(a), -1), axis=1) / np.maximum(1e-12, scale)).max()


def _jnorm(blocks):
    """Frobenius norm of each state's whole Jacobian [d_q | d_dq | d_in]"""
    return np.sqrt(sum(np.sum(np.asarray(b).reshape(len(b), -1) ** 2, axis=1) for b in blocks))


# ---------------------------------------------------------------------------------------------- host: derivatives
@pytest.mark.parametrize("name", CHAINS)
def test_host_dynamics_derivatives_vs_central_differences(gradsim, name):
    """fp64 within 1e-6 relative to the Jacobian's norm (the finite difference's own accuracy); fp32 against fp64
    within 1e-3."""
    d, cd = _chain(name)
    q, dq, x = _states(d, 6, 1)
    for kind, fn in ((0, lambda a, b, c: oracle_forward(d, a, b, c)), (1, lambda a, b, c: oracle_inverse(d, a, b, c))):
        got = shim_jac(gradsim, cd, kind, q, dq, x)
        ref = fd_jac(fn, q, dq, x)
        scale = _jnorm(ref)
        for blk, (g, r) in enumerate(zip(got, ref)):
            assert _rel(g, r, scale) < 1e-6, (name, kind, blk, _rel(g, r, scale))
        got32 = shim_jac(gradsim, cd, kind, q, dq, x, f32=1)
        for blk, (g, r) in enumerate(zip(got32, got)):
            assert _rel(g, r, scale) < 1e-3, (name, kind, blk, _rel(g, r, scale))


@pytest.mark.parametrize("name", CHAINS)
def test_host_derivative_identities(gradsim, name):
    """M d_u = I;  d_ddq = M;  d ddq / d(q, dq) = -M^-1 d u / d(q, dq) at u = inverse_dynamics(q, dq, ddq); each
    within 50 eps cond(M)."""
    d, cd = _chain(name)
    q, dq, a = _states(d, 8, 2)
    ch = rbd_oracle.ChainOracle(d)
    M = ch.M(q)
    eps = np.finfo(np.float64).eps
    cond = np.linalg.cond(M)
    n = q.shape[1]
    iq, idq, iddq = shim_jac(gradsim, cd, 1, q, dq, a)
    assert (np.abs(iddq - M).max((1, 2)) <= 50 * eps * cond * np.abs(M).max((1, 2))).all()
    u = oracle_inverse(d, q, dq, a)
    fq, fdq, fu = shim_jac(gradsim, cd, 0, q, dq, u)
    assert (np.abs(M @ fu - np.eye(n)).max((1, 2)) <= 50 * eps * cond).all()
    for f, i in ((fq, iq), (fdq, idq)):
        want = -np.linalg.solve(M, i)
        scale = np.maximum(1.0, np.abs(want).max((1, 2)))
        assert (np.abs(f - want).max((1, 2)) <= 50 * eps * cond * scale).all(), name


# ---------------------------------------------------------------------------------------------- host: rollout adjoint
def shim_vjp(gs, cd, q0, dq0, u, path, comp, frame, xoff, q_traj, dq_traj, cot, f32=0, dt=DT, effort=EFFORT):
    n, B = cd.n_joints, len(q0)
    S = u.shape[0]
    gu = np.zeros((S, B, n))
    gq0, gdq0 = np.zeros((B, n)), np.zeros((B, n))
    xo = None if xoff is None else (C.c_double * 3)(*xoff)
    c = [None if cot.get(k) is None else np.ascontiguousarray(cot[k]) for k in ("cost", "qf", "dqf", "q", "dq", "u", "x")]
    rc = gs.gr_rollout_vjp(C.byref(cd), f32, gs.hs_frame_id(n, frame.encode()), xo, _p(np.ascontiguousarray(q0)),
                           _p(np.ascontiguousarray(dq0)), _p(np.ascontiguousarray(u)), n if u.ndim == 3 else 0,
                           int(comp), _p(None if path is None else np.ascontiguousarray(path)),
                           0 if path is None or path.ndim == 2 else 6, S, C.c_double(dt), C.c_double(effort),
                           _p(np.ascontiguousarray(q_traj)), _p(np.ascontiguousarray(dq_traj)), *[_p(a) for a in c],
                           _p(gu), _p(gq0), _p(gdq0), C.c_int64(B))
    assert rc == 0
    return gu, gq0, gdq0


def shim_jvp(gs, cd, q0, dq0, u, path, comp, frame, xoff, v, a, b, dt=DT, effort=EFFORT):
    n, B = cd.n_joints, len(q0)
    S = u.shape[0]
    t = {k: np.zeros((S, B, 3 if k == "x" else n)) for k in ("q", "dq", "u", "x")}
    t.update(cost=np.zeros(B), qf=np.zeros((B, n)), dqf=np.zeros((B, n)))
    xo = None if xoff is None else (C.c_double * 3)(*xoff)
    rc = gs.gr_rollout_jvp(C.byref(cd), 0, gs.hs_frame_id(n, frame.encode()), xo, _p(np.ascontiguousarray(q0)),
                           _p(np.ascontiguousarray(dq0)), _p(np.ascontiguousarray(u)), n if u.ndim == 3 else 0,
                           int(comp), _p(None if path is None else np.ascontiguousarray(path)),
                           0 if path is None or path.ndim == 2 else 6, S, C.c_double(dt), C.c_double(effort),
                           _p(np.ascontiguousarray(v)), _p(np.ascontiguousarray(a)), _p(np.ascontiguousarray(b)),
                           *[_p(t[k]) for k in ("q", "dq", "u", "x", "cost", "qf", "dqf")], C.c_int64(B))
    assert rc == 0
    return t


def random_cotangents(rng, S, B, n, which=("cost", "qf", "dqf", "q", "dq", "u", "x")):
    shapes = dict(cost=(B,), qf=(B, n), dqf=(B, n), q=(S, B, n), dq=(S, B, n), u=(S, B, n), x=(S, B, 3))
    return {k: rng.normal(size=shapes[k]) if k in which else None for k in shapes}


def _dot_test(gradsim, plantsim, arm, variant, S, seed=0):
    cd = _desc(arm)
    n, B = cd.n_joints, 5
    q, dq, u, path, comp, frame, off = variant_inputs(arm, variant, B, S=S, seed=seed)
    fw = shim_simulate(plantsim, arm, q, dq, u, path, comp, frame, off)
    rng = np.random.default_rng(seed + 17)
    cot = random_cotangents(rng, S, B, n)
    gu, gq0, gdq0 = shim_vjp(gradsim, cd, q, dq, u, path, comp, frame, off, fw["q"], fw["dq"], cot)
    v = rng.normal(size=u.shape)
    a, b = rng.normal(size=(B, n)), rng.normal(size=(B, n))
    t = shim_jvp(gradsim, cd, q, dq, u, path, comp, frame, off, v, a, b)
    gu_in = gu if u.ndim == 3 else gu.sum(1)
    lhs = np.sum(gu_in * v) + np.sum(gq0 * a) + np.sum(gdq0 * b)
    rhs = sum(np.sum(cot[k] * t[k]) for k in cot)
    return lhs, rhs, max(abs(lhs), abs(rhs), 1e-300)


@pytest.mark.parametrize("variant", list(VARIANTS))
@pytest.mark.parametrize("arm", ARMS)
def test_host_rollout_adjoint_dot_product(gradsim, plantsim, arm, variant):
    """<gu, v> + <gq0, a> + <gdq0, b> equals the tangent of a dual rollout of plant_step along (v, a, b) paired with the
    same random cotangents on every output and record, within 1e-11 relative."""
    lhs, rhs, scale = _dot_test(gradsim, plantsim, arm, variant, S=7)
    assert abs(lhs - rhs) < 1e-11 * scale, (lhs, rhs)


def test_host_rollout_adjoint_zero_steps(gradsim):
    """S = 0: the start-state cotangents are those of the final state, nothing else."""
    cd = _desc("ur5")
    B, n = 3, 6
    rng = np.random.default_rng(4)
    q, dq = rng.normal(size=(B, n)), rng.normal(size=(B, n))
    cot = random_cotangents(rng, 0, B, n)
    gu, gq0, gdq0 = shim_vjp(gradsim, cd, q, dq, np.zeros((0, B, n)), None, False, "EE", None, np.zeros((0, B, n)),
                             np.zeros((0, B, n)), cot)
    assert gu.shape == (0, B, n) and np.array_equal(gq0, cot["qf"]) and np.array_equal(gdq0, cot["dqf"])


@pytest.mark.parametrize("variant", ["per_u_per_path_offset_frame", "shared_u_shared_path_comp"])
def test_host_rollout_gradient_vs_central_differences(gradsim, plantsim, variant):
    """The gradient of the cost (plus a final-state term) against central differences of oracle_simulate along random
    directions of u, q0 and dq0, within 1e-6."""
    arm, S, B = "ur5", 6, 3
    cd = _desc(arm)
    n = cd.n_joints
    q, dq, u, path, comp, frame, off = variant_inputs(arm, variant, B, S=S)
    rng = np.random.default_rng(9)
    w = rng.normal(size=(B, n))

    def f(uu, qq, dd):
        o = oracle_simulate(arm, qq, dd, uu, DT, path, EFFORT, comp, frame, off)
        return np.sum(o["cost"]) + np.sum(w * o["q_final"])

    fw = shim_simulate(plantsim, arm, q, dq, u, path, comp, frame, off)
    cot = dict(cost=np.ones(B), qf=w)
    gu, gq0, gdq0 = shim_vjp(gradsim, cd, q, dq, u, path, comp, frame, off, fw["q"], fw["dq"], cot)
    gu_in = gu if u.ndim == 3 else gu.sum(1)
    for _ in range(3):
        v, a, b = rng.normal(size=u.shape), rng.normal(size=(B, n)), rng.normal(size=(B, n))
        h = 1e-5
        fd = (f(u + h * v, q + h * a, dq + h * b) - f(u - h * v, q - h * a, dq - h * b)) / (2 * h)
        an = np.sum(gu_in * v) + np.sum(gq0 * a) + np.sum(gdq0 * b)
        assert abs(fd - an) < 1e-6 * max(1.0, abs(an)), (fd, an)


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


@pytest.mark.parametrize("fn", ["abrb_forward_dynamics_derivatives_f64", "abrb_forward_dynamics_derivatives_f32",
                                "abrb_inverse_dynamics_derivatives_f64", "abrb_inverse_dynamics_derivatives_f32"])
def test_abi_derivatives_reject_bad_arguments_before_any_device_work(native, fn):
    lib, m, buf = native
    f = getattr(lib, fn)
    p = buf.ctypes.data
    inn, d_in = ("u", "d_u") if "forward" in fn else ("ddq", "d_ddq")
    ok = dict(m=m, q=p, dq=p, i=p, a=p, b=p, c=p, B=8)
    bad = [
        (dict(m=None), "NULL model"),
        (dict(q=None), "NULL q"),
        (dict(dq=None), "NULL dq"),
        (dict(i=None), f"NULL {inn}"),
        (dict(a=None), "NULL d_q"),
        (dict(b=None), "NULL d_dq"),
        (dict(B=-1), "B < 0"),
        (dict(q=p + 1), "misaligned pointer (q)"),
        (dict(i=p + 2), f"misaligned pointer ({inn})"),
        (dict(b=p + 1), "misaligned pointer (d_dq)"),
        (dict(c=p + 2), f"misaligned pointer ({d_in})"),
    ]
    who = fn.rsplit("_", 1)[0]
    for over, word in bad:
        a = {**ok, **over}
        rc = f(a["m"], a["q"], a["dq"], a["i"], a["a"], a["b"], a["c"], a["B"], None)
        assert rc == _abi.EINVAL, (over, rc)
        msg = lib.abrb_last_error().decode()
        assert msg.startswith(who) and word in msg, (over, msg)
    assert f(m, None, None, None, None, None, None, 0, None) == 0


_VJP_KEYS = ("m", "frame", "xoff", "q0", "dq0", "u", "us", "comp", "path", "ps", "steps", "dt", "ew", "qt", "dqt",
             "gc", "gq", "gdq", "gqt", "gdqt", "gut", "gxt", "gu", "gq0", "gdq0", "B", "stream")


def _vjp_args(**over):
    a = {k: None for k in _VJP_KEYS}
    a.update(frame=0, us=0, comp=0, ps=0, steps=4, dt=1e-3, ew=0.0, B=8)
    a.update(over)
    return [a[k] for k in _VJP_KEYS]


@pytest.mark.parametrize("fn", ["abrb_plant_rollout_vjp_f64", "abrb_plant_rollout_vjp_f32"])
def test_abi_rollout_vjp_rejects_bad_arguments_before_any_device_work(native, fn):
    lib, m, buf = native
    f = getattr(lib, fn)
    p = buf.ctypes.data
    ok = dict(m=m, q0=p, dq0=p, u=p, qt=p, dqt=p, gu=p, gq0=p, gdq0=p)
    bad = [
        (dict(m=None), _abi.EINVAL, "model"),
        (dict(q0=None), _abi.EINVAL, "NULL q0"),
        (dict(dq0=None), _abi.EINVAL, "NULL dq0"),
        (dict(u=None), _abi.EINVAL, "NULL u"),
        (dict(qt=None), _abi.EINVAL, "NULL q_traj"),
        (dict(dqt=None), _abi.EINVAL, "NULL dq_traj"),
        (dict(gu=None), _abi.EINVAL, "NULL gu"),
        (dict(gq0=None), _abi.EINVAL, "NULL gq0"),
        (dict(gdq0=None), _abi.EINVAL, "NULL gdq0"),
        (dict(us=3), _abi.EINVAL, "u_stride"),
        (dict(ps=3, path=p), _abi.EINVAL, "path_stride"),
        (dict(steps=-1), _abi.EINVAL, "steps"),
        (dict(B=-1), _abi.EINVAL, "B < 0"),
        (dict(ew=-1.0), _abi.EINVAL, "effort_weight"),
        (dict(ew=float("nan")), _abi.EINVAL, "effort_weight"),
        (dict(q0=p + 1), _abi.EINVAL, "misaligned pointer (q0)"),
        (dict(qt=p + 2), _abi.EINVAL, "misaligned pointer (q_traj)"),
        (dict(gc=p + 1), _abi.EINVAL, "misaligned pointer (g_cost)"),
        (dict(gxt=p + 2), _abi.EINVAL, "misaligned pointer (g_x_traj)"),
        (dict(gu=p + 1), _abi.EINVAL, "misaligned pointer (gu)"),
        (dict(frame=99), _abi.EFRAME, "frame"),
        (dict(frame=-1), _abi.EFRAME, "frame"),
    ]
    for over, code, word in bad:
        rc = f(*_vjp_args(**{**ok, **over}))
        assert rc == code, (over, rc)
        msg = lib.abrb_last_error().decode()
        assert msg.startswith("abrb_plant_rollout_vjp") and word in msg, (over, msg)
    assert f(*_vjp_args(m=m, B=0)) == 0
    if lib.abrb_device_count() == 0:  # without steps the records, u and gu are not needed; the call then needs a device
        assert f(*_vjp_args(m=m, q0=p, dq0=p, gq0=p, gdq0=p, steps=0)) == _abi.ECUDA


def test_signatures_cover_the_derivative_entry_points():
    import os

    from abr_control_b200 import _lib

    for fn in ("abrb_forward_dynamics_derivatives", "abrb_inverse_dynamics_derivatives"):
        for sfx in ("_f64", "_f32"):
            res, args = _lib.SIGNATURES[fn + sfx]
            assert len(args) == 9 and args[7] is C.c_int64
    for sfx in ("_f64", "_f32"):
        res, args = _lib.SIGNATURES["abrb_plant_rollout_vjp" + sfx]
        assert len(args) == 27 and args[11] is C.c_double and args[12] is C.c_double and args[25] is C.c_int64
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    with open(os.path.join(root, "include", "abrb.h")) as fh:
        hdr = fh.read()
    for fn in ("abrb_forward_dynamics_derivatives", "abrb_inverse_dynamics_derivatives", "abrb_plant_rollout_vjp"):
        assert f"int {fn}_f64(" in hdr and f"int {fn}_f32(" in hdr


def test_path_requiring_grad_raises_before_any_device_work():
    torch = pytest.importorskip("torch")
    from abr_control_b200.arms import ur5

    rc = ur5.Config()
    path = torch.zeros((3, 6), dtype=torch.float64, requires_grad=True)
    with pytest.raises(NotImplementedError):
        rc.simulate(np.zeros(6), np.zeros(6), np.zeros((3, 6)), path=path)


# ============================================================================================== GPU
def _cfg_desc(name, dtype=np.float64):
    from abr_control_b200.arms.base_config import BaseConfig

    d, _ = _chain(name)
    return BaseConfig(d, ROBOT_NAME=name, dtype=dtype)


@pytest.mark.gpu
@pytest.mark.parametrize("name", CHAINS)
def test_device_derivatives_vs_shim(gradsim, name):
    """fp64 within 1e-12 relative; fp32 within 1e-4 of the fp32 shim (both blocks of both kinds)."""
    import torch

    d, cd = _chain(name)
    q, dq, x = _states(d, 70, 5)
    rc = _cfg_desc(name)
    for f32 in (0, 1):
        td = torch.float32 if f32 else torch.float64
        tq, tdq, tx = (torch.as_tensor(a, device="cuda", dtype=td) for a in (q, dq, x))
        hq, hdq, hx = (a.cpu().double().numpy() for a in (tq, tdq, tx))
        for kind, fn in ((0, rc.forward_dynamics_derivatives), (1, rc.inverse_dynamics_derivatives)):
            got = fn(tq, tdq, tx)
            ref = shim_jac(gradsim, cd, kind, hq, hdq, hx, f32=f32)
            scale = _jnorm(ref)
            for blk, (g, r) in enumerate(zip(got, ref)):
                assert g.dtype == td and tuple(g.shape) == r.shape
                e = _rel(g.double().cpu().numpy(), r, scale)
                assert e < (1e-4 if f32 else 1e-12), (name, f32, kind, blk, e)


@pytest.mark.gpu
def test_derivatives_input_forms():
    import torch

    rc = _cfg_desc("ur5")
    q, dq, x = _states(_chain("ur5")[0], 5, 3)
    h = rc.forward_dynamics_derivatives(q, dq, x)
    dd = rc.forward_dynamics_derivatives(*(torch.as_tensor(a, device="cuda") for a in (q, dq, x)))
    assert all(isinstance(a, np.ndarray) and np.array_equal(a, b.cpu().numpy()) for a, b in zip(h, dd))
    one = rc.inverse_dynamics_derivatives(q[2], dq[2], x[2])
    assert one[0].shape == (6, 6) and np.array_equal(one[2], rc.inverse_dynamics_derivatives(q, dq, x)[2][2])


@pytest.mark.gpu
def test_gradcheck_dynamics_and_simulate():
    import torch

    for name in ("ur5", "rand7_shear"):
        rc = _cfg_desc(name)
        d, _ = _chain(name)
        n = d["n_joints"]
        q, dq, x = (torch.as_tensor(a, device="cuda").requires_grad_() for a in _states(d, 3, 8))
        assert torch.autograd.gradcheck(lambda a, b, c: rc.forward_dynamics(a, b, c), (q, dq, x), eps=1e-6, atol=1e-6,
                                        rtol=1e-5)
        assert torch.autograd.gradcheck(lambda a, b, c: rc.inverse_dynamics(a, b, c), (q, dq, x), eps=1e-6, atol=1e-6,
                                        rtol=1e-5)
        S, B = 5, 3
        gen = np.random.default_rng(4)
        q0 = torch.as_tensor(gen.uniform(-1, 1, (B, n)), device="cuda").requires_grad_()
        dq0 = torch.as_tensor(gen.uniform(-0.3, 0.3, (B, n)), device="cuda").requires_grad_()
        path = torch.as_tensor(gen.uniform(-0.5, 0.5, (S, B, 6)), device="cuda")
        for shared in (False, True):
            u = torch.as_tensor(gen.normal(size=(S, n) if shared else (S, B, n)), device="cuda").requires_grad_()

            def f(qq, dd, uu):
                qf, dqf, tr, cost = rc.simulate(qq, dd, uu, dt=0.01, path=path, effort_weight=0.01,
                                                compensate_gravity=True, ref_frame="EE", xyz_offset=[0.01, 0.02, 0.0])
                return (qf, dqf, cost) + tuple(tr[k] for k in ("q", "dq", "u", "x"))

            assert torch.autograd.gradcheck(f, (q0, dq0, u), eps=1e-6, atol=1e-6, rtol=1e-5), (name, shared)


def _fullsize_inputs(B, S, seed):
    import torch

    from test_plant import _mpc_inputs

    rc, q, dq, path = _mpc_inputs(B, S, seed)
    gen = torch.Generator(device="cuda").manual_seed(seed)
    u = torch.randn((S, B, 6), device="cuda", generator=gen, dtype=torch.float64)
    return rc, q, dq, path, u


@pytest.mark.gpu
def test_full_size_derivatives_vs_central_differences():
    import torch

    rc = _cfg_desc("ur5")
    B = 65536
    gen = torch.Generator(device="cuda").manual_seed(21)
    q = torch.rand((B, 6), device="cuda", generator=gen, dtype=torch.float64) * 2 * np.pi
    dq = torch.rand((B, 6), device="cuda", generator=gen, dtype=torch.float64) * 2 - 1
    u = torch.randn((B, 6), device="cuda", generator=gen, dtype=torch.float64) * 5
    got = rc.forward_dynamics_derivatives(q, dq, u)
    h = 1e-6
    worst = 0.0
    for blk, base in enumerate((q, dq, u)):
        for j in range(6):
            e = torch.zeros_like(base)
            e[:, j] = h
            args_p, args_m = [q, dq, u], [q, dq, u]
            args_p[blk], args_m[blk] = base + e, base - e
            fd = (rc.forward_dynamics(*args_p) - rc.forward_dynamics(*args_m)) / (2 * h)
            col = got[blk][:, :, j]
            rel = ((col - fd).norm(dim=1) / got[blk].flatten(1).norm(dim=1).clamp_min(1e-12)).max().item()
            worst = max(worst, rel)
    print(f"65536 states: derivatives vs central differences {worst:.2e}")
    assert worst < 1e-6


@pytest.mark.gpu
def test_full_size_rollout_gradient(gradsim):
    """4 096 x 128, per-trajectory u and path: the gradient of the cost against central differences along three random
    directions (1e-6) and against the shim on 64 trajectories (1e-10)."""
    import torch

    B, S = 4096, 128
    rc, q, dq, path, u = _fullsize_inputs(B, S, 31)
    kw = dict(dt=DT, path=path, effort_weight=1e-4, compensate_gravity=True)
    u = u.requires_grad_()
    q0, dq0 = q.clone().requires_grad_(), dq.clone().requires_grad_()
    qf, dqf, tr, cost = rc.simulate(q0, dq0, u, record=(), **kw)
    cost.sum().backward()
    gen = torch.Generator(device="cuda").manual_seed(5)
    with torch.no_grad():
        for _ in range(3):
            v = torch.randn(u.shape, device="cuda", generator=gen, dtype=torch.float64)
            a = torch.randn(q.shape, device="cuda", generator=gen, dtype=torch.float64)
            b = torch.randn(q.shape, device="cuda", generator=gen, dtype=torch.float64)
            h = 1e-6
            cp = rc.simulate(q + h * a, dq + h * b, u + h * v, record=(), **kw)[3]
            cm = rc.simulate(q - h * a, dq - h * b, u - h * v, record=(), **kw)[3]
            fd = ((cp - cm) / (2 * h))
            an = (u.grad * v).sum((0, 2)) + (q0.grad * a).sum(1) + (dq0.grad * b).sum(1)
            rel = ((fd - an).abs() / an.abs().clamp_min(1.0)).max().item()
            print(f"rollout gradient vs central differences: {rel:.2e}")
            assert rel < 1e-6
    sel = np.arange(0, B, B // 64)
    tsel = torch.as_tensor(sel, device="cuda")
    kw_sel = dict(kw, path=path[:, tsel].contiguous())
    with torch.no_grad():
        _, _, trs, _ = rc.simulate(q[tsel], dq[tsel], u[:, tsel].contiguous(), **kw_sel)
    cd = _desc("ur5")
    cot = dict(cost=np.ones(len(sel)))
    hn = lambda t: t.detach().cpu().numpy()
    gu, gq0, gdq0 = shim_vjp(gradsim, cd, hn(q[tsel]), hn(dq[tsel]), hn(u[:, tsel]), hn(path[:, tsel]), True, "EE",
                             None, hn(trs["q"]), hn(trs["dq"]), cot, dt=DT, effort=1e-4)
    for g, r in ((hn(u.grad[:, tsel]), gu), (hn(q0.grad[tsel]), gq0), (hn(dq0.grad[tsel]), gdq0)):
        e = np.abs(g - r).max() / np.abs(r).max()
        assert e < 1e-10, e


@pytest.mark.gpu
def test_rollout_gradient_bit_identities():
    import torch

    B, S = 256, 16
    rc, q, dq, path, u = _fullsize_inputs(B, S, 41)
    kw = dict(dt=DT, effort_weight=1e-3, compensate_gravity=True)

    def grads(qq, dd, uu, pp):
        uu = uu.clone().requires_grad_()
        qq, dd = qq.clone().requires_grad_(), dd.clone().requires_grad_()
        qf, dqf, tr, cost = rc.simulate(qq, dd, uu, path=pp, **kw)
        (cost.sum() + (qf ** 2).sum() + tr["x"].sum() + tr["u"].sum()).backward()
        return uu.grad, qq.grad, dd.grad

    gu, gq, gdq = grads(q, dq, u, path)
    perm = torch.randperm(B, device="cuda")
    pu, pq, pdq = grads(q[perm], dq[perm], u[:, perm], path[:, perm])
    assert torch.equal(pu, gu[:, perm]) and torch.equal(pq, gq[perm]) and torch.equal(pdq, gdq[perm])
    us = u[:, 0]
    su, sq, sdq = grads(q, dq, us, path)
    tu, tq, tdq = grads(q, dq, us[:, None].expand(S, B, 6).contiguous(), path)
    assert su.shape == (S, 6)
    assert (su - tu.sum(1)).abs().max().item() <= 1e-12 * tu.sum(1).abs().max().item()
    assert torch.equal(sq, tq) and torch.equal(sdq, tdq)
    # the forward outputs do not depend on whether a gradient is wanted
    with torch.no_grad():
        ref = rc.simulate(q, dq, u, path=path, **kw)
    out = rc.simulate(q.clone().requires_grad_(), dq, u.clone().requires_grad_(), path=path, **kw)
    assert torch.equal(ref[0], out[0]) and torch.equal(ref[1], out[1]) and torch.equal(ref[3], out[3])
    for k in ("q", "dq", "u", "x"):
        assert torch.equal(ref[2][k], out[2][k]), k
    assert out[3].requires_grad


@pytest.mark.gpu
def test_adam_on_a_torque_plan_halves_the_tracking_cost():
    """50 Adam steps on a UR5 torque plan (gravity-compensated residual torques, shared over 8 starts) tracking a
    reachable path cut the cost below half its start."""
    import torch

    rc = _cfg_desc("ur5")
    B, S, dt = 8, 60, 0.01
    rng = np.random.default_rng(2)
    q0 = torch.as_tensor(rng.uniform(-0.2, 0.2, (B, 6)) + np.array([0, -1.2, 1.2, 0, 0.5, 0]), device="cuda")
    dq0 = torch.zeros_like(q0)
    # a reachable path: the end effector's track under a smooth joint motion
    qs = q0[None] + torch.linspace(0, 1, S, device="cuda", dtype=torch.float64)[:, None, None] * 0.4
    xs = torch.stack([rc.Tx("EE", qs[t]) for t in range(S)])
    path = torch.cat([xs, torch.zeros_like(xs)], -1).contiguous()
    u = torch.zeros((S, 6), device="cuda", dtype=torch.float64, requires_grad=True)
    opt = torch.optim.Adam([u], lr=0.5)
    costs = []
    for _ in range(50):
        opt.zero_grad()
        _, _, _, cost = rc.simulate(q0, dq0, u, dt=dt, path=path, effort_weight=1e-5, compensate_gravity=True,
                                    record=())
        loss = cost.sum()
        loss.backward()
        costs.append(loss.item())
        opt.step()
    print("Adam: cost", costs[0], "->", costs[-1])
    assert costs[-1] < 0.5 * costs[0]
