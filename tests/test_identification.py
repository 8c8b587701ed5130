"""Identification of the link inertias: the inverse-dynamics regressor (``BaseConfig.inverse_dynamics_regressor``,
``abrb_inverse_dynamics_regressor_*``) and the least-squares fit (``BaseConfig.identify_link_inertia``).

Semantics (include/abrb.h, DESIGN.md S3.7): ``u = M ddq + C dq - g = Y(q, dq, ddq) theta`` with theta =
``link_inertia[1:]`` flattened; the fit ties the three mass entries of a link.

CPU part: the kernel's per-state function (abrb_regress.cuh) runs on the host through tests/hostsim/regsim.cpp (TEST
INFRASTRUCTURE, never loaded by the package) against the oracle (oracle/ident_oracle.py: column p is the literal
product-rule inverse dynamics of the chain with unit inertia e_p), against the host instantiation of
``inverse_dynamics_state``, column by column; identification from closed-loop Joint rollouts of perturbed arms;
argument checking of the C entry points and of the Python methods.  GPU part: the kernel against the shim and against
``inverse_dynamics`` at full size, batch edges, bit identities, the input forms, and identification end to end.
"""
import copy
import ctypes as C
import os

import numpy as np
import pytest

from abr_control_b200 import _abi
from oracle import ident_oracle
from test_ctrl_rollout import shim_rollout
from test_generic_chains import random_chain
from test_plant import _build, _p

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ARMS = ("ur5", "jaco2", "threejoint", "twojoint")
RANDOM = tuple(f"rand{n}_{'ortho' if o else 'shear'}" for n in range(1, 8) for o in (True, False))
# bounds relative to the largest regressor entry of the batch (the torque scale of a unit parameter): observed maxima
# are 1.3e-15 (fp64) and 8.8e-7 (fp32), DESIGN.md S5
TOL = {0: 1e-12, 1: 1e-4}


def _chain(name):
    """descriptor dict of an arm or of a random chain 'rand<n>_<ortho|shear>'"""
    if name.startswith("rand"):
        n, kind = name[4:].split("_")
        return random_chain(int(n), kind == "ortho", seed=31 * int(n) + (kind == "ortho"))
    return _abi.load_arm_json(name)


def states(n, B, seed):
    rng = np.random.default_rng(seed)
    return rng.uniform(0, 2 * np.pi, (B, n)), rng.uniform(-5, 5, (B, n)), rng.uniform(-10, 10, (B, n))


@pytest.fixture(scope="module")
def regsim(tmp_path_factory):
    return _build(tmp_path_factory, "regsim")


def shim_regressor(rs, desc, q, dq, ddq, f32=0):
    """(B, n, 6n) from the host instantiation of inverse_dynamics_regressor"""
    cd = _abi.chain_desc_from_dict(desc)
    n, B = cd.n_joints, len(q)
    Yt = np.zeros((B, 6 * n, n))
    q, dq, ddq = (np.ascontiguousarray(a, dtype=np.float64) for a in (q, dq, ddq))
    assert rs.rs_regressor(C.byref(cd), f32, _p(q), _p(dq), _p(ddq), C.c_int64(B), _p(Yt)) == 0
    return Yt.transpose(0, 2, 1)


def shim_inverse(rs, desc, q, dq, ddq, f32=0):
    """inverse_dynamics_state on the host (plantsim's pl_dynamics, kind 1)"""
    cd = _abi.chain_desc_from_dict(desc)
    q, dq, ddq = (np.ascontiguousarray(a, dtype=np.float64) for a in (q, dq, ddq))
    out = np.zeros_like(q)
    assert rs.pl_dynamics(C.byref(cd), f32, 1, _p(q), _p(dq), _p(ddq), C.c_int64(len(q)), _p(out)) == 0
    return out


def with_theta(desc, theta):
    d = copy.deepcopy(desc)
    W = np.asarray(d["link_inertia"], dtype=np.float64)
    W[1:] = np.asarray(theta).reshape(-1, 6)
    d["link_inertia"] = W.tolist()
    return d


# ---------------------------------------------------------------------------------------------- regressor, host
@pytest.mark.parametrize("f32", [0, 1])
@pytest.mark.parametrize("name", ARMS + RANDOM)
def test_host_regressor_vs_oracle(regsim, name, f32):
    desc = _chain(name)
    q, dq, ddq = states(desc["n_joints"], 8, 5)
    ref = ident_oracle.regressor(desc, q, dq, ddq)
    got = shim_regressor(regsim, desc, q, dq, ddq, f32)
    assert np.abs(got - ref).max() <= TOL[f32] * np.abs(ref).max(), (name, np.abs(got - ref).max())


@pytest.mark.parametrize("f32", [0, 1])
@pytest.mark.parametrize("name", ARMS + RANDOM)
def test_host_regressor_times_theta_is_inverse_dynamics(regsim, name, f32):
    desc = _chain(name)
    q, dq, ddq = states(desc["n_joints"], 16, 6)
    Y = shim_regressor(regsim, desc, q, dq, ddq, f32)
    u = shim_inverse(regsim, desc, q, dq, ddq, f32)
    scale = np.abs(Y).max() * np.abs(ident_oracle.theta(desc)).max()
    assert np.abs(Y @ ident_oracle.theta(desc) - u).max() <= TOL[f32] * scale


@pytest.mark.parametrize("name", ("ur5", "jaco2", "rand7_shear", "rand3_ortho"))
def test_host_columns_are_inverse_dynamics_of_unit_inertias(regsim, name):
    """column p == inverse_dynamics_state of the chain whose only inertia constant is parameter p"""
    desc = _chain(name)
    n = desc["n_joints"]
    q, dq, ddq = states(n, 12, 7)
    Y = shim_regressor(regsim, desc, q, dq, ddq)
    scale = np.abs(Y).max()
    for p in range(6 * n):
        col = shim_inverse(regsim, ident_oracle.unit_chain(desc, p), q, dq, ddq)
        assert np.abs(Y[:, :, p] - col).max() <= 1e-12 * scale, p


def test_host_regressor_of_link0_free_and_gravity_free_chain(regsim):
    """link 0's inertia never enters; without gravity the static regressor (dq = ddq = 0) vanishes"""
    desc = _chain("ur5")
    q, dq, ddq = states(6, 8, 8)
    d2 = copy.deepcopy(desc)
    d2["link_inertia"][0] = [9.0, 9.0, 9.0, 1.0, 2.0, 3.0]
    assert np.array_equal(shim_regressor(regsim, desc, q, dq, ddq), shim_regressor(regsim, d2, q, dq, ddq))
    d2["gravity"] = [0.0] * 6
    assert np.abs(shim_regressor(regsim, d2, q, 0 * dq, 0 * ddq)).max() == 0.0


# ---------------------------------------------------------------------------------------------- identification, host
def perturbed(arm, seed):
    """the arm with each link's mass scaled by U(0.5, 1.5) (all three entries alike) and each inertia by U(0.5, 1.5)"""
    d = copy.deepcopy(_abi.load_arm_json(arm))
    rng = np.random.default_rng(seed)
    W = np.asarray(d["link_inertia"], dtype=np.float64)
    W[1:, :3] *= rng.uniform(0.5, 1.5, (len(W) - 1, 1))
    W[1:, 3:] *= rng.uniform(0.5, 1.5, (len(W) - 1, 3))
    d["link_inertia"] = W.tolist()
    return d


def sinusoid_paths(n, B, S, dt, seed):
    """random starts and joint paths of three sinusoids each about them, with their exact velocities"""
    rng = np.random.default_rng(seed)
    q0 = rng.uniform(-np.pi, np.pi, (B, n))
    dq0 = rng.uniform(-1, 1, (B, n))
    t = (np.arange(S) * dt)[:, None, None]
    A, w, ph = rng.uniform(0.3, 1.0, (3, B, n)), rng.uniform(2, 12, (3, B, n)), rng.uniform(0, 2 * np.pi, (3, B, n))
    path = q0[None] + sum(A[i] * np.sin(w[i] * t + ph[i]) for i in range(3))
    pv = sum(A[i] * w[i] * np.cos(w[i] * t + ph[i]) for i in range(3))
    return q0, dq0, path, pv


def samples(q0, dq0, traj, dt):
    """(q, dq, ddq, u), each (S, B, n), of a recorded rollout: the state BEFORE step t and its applied torque"""
    qp = np.concatenate([q0[None], traj["q"][:-1]])
    dqp = np.concatenate([dq0[None], traj["dq"][:-1]])
    return qp, dqp, (traj["dq"] - dqp) / dt, traj["u"]


def reduced_rank(Y, rcond):
    """rank of a stacked (K, n, 6n) regressor with tied masses, by the fit's own rule"""
    from abr_control_b200.arms import _ident

    n = Y.shape[1]
    Yr = (Y @ _ident.tie_matrix(n)).reshape(-1, 4 * n)
    return _ident.solve(Yr.T @ Yr, np.zeros(4 * n), rcond)[1].shape[1]


@pytest.fixture(scope="module")
def ctrlsim(tmp_path_factory):
    return _build(tmp_path_factory, "ctrlsim")


@pytest.mark.parametrize("arm", ("ur5", "jaco2"))
def test_host_identification_is_exact_on_simulated_data(regsim, ctrlsim, arm):
    """Joint drives the perturbed arm along sinusoids; the fit from the nominal model recovers it on the identifiable
    directions, with a residual at rounding level and the same inverse dynamics at held-out states"""
    torch = pytest.importorskip("torch")
    from abr_control_b200.arms import _ident

    true, nominal = perturbed(arm, 1), _abi.load_arm_json(arm)
    n, B, S, dt = true["n_joints"], 32, 256, 1e-3
    q0, dq0, path, pv = sinusoid_paths(n, B, S, dt, 2)
    tr = shim_rollout(ctrlsim, true, "joint", dict(kp=400.0, kv=40.0), q0, dq0, path, pv, dt=dt)
    q, dq, ddq, u = (a.reshape(-1, n) for a in samples(q0, dq0, tr, dt))

    def regress(i0, i1):
        return (torch.from_numpy(shim_regressor(regsim, nominal, q[i0:i1], dq[i0:i1], ddq[i0:i1])),
                torch.from_numpy(np.ascontiguousarray(u[i0:i1])))

    theta, info = _ident.identify(regress, len(q), 1000, ident_oracle.theta(nominal), 1e-10)
    th_true = ident_oracle.theta(true)
    assert info["rms_after"] <= 1e-9 * np.sqrt(np.mean(u ** 2)), info
    assert info["rms_before"] > 1e-2 * np.sqrt(np.mean(u ** 2))
    Q = info["basis"]
    assert Q.shape == (6 * n, info["rank"]) and np.allclose(Q.T @ Q, np.eye(info["rank"]), atol=1e-12)
    assert np.abs(Q.T @ (theta - th_true)).max() <= 1e-9 * np.abs(th_true).max()
    assert info["unidentifiable"] == [3, 4]  # link 1 turns about joint 0's axis only: its I_xx, I_yy never act
    assert np.all(theta.reshape(n, 6)[:, 0] == theta.reshape(n, 6)[:, 2])
    # the rank of the oracle's stacked regressor over every 16th sample
    sub = slice(None, None, 16)
    assert info["rank"] == reduced_rank(ident_oracle.regressor(true, q[sub], dq[sub], ddq[sub]), 1e-10)
    qh, dqh, ah = states(n, 64, 9)
    ref = shim_inverse(regsim, true, qh, dqh, ah)
    got = shim_inverse(regsim, with_theta(nominal, theta), qh, dqh, ah)
    assert np.abs(got - ref).max() <= 1e-8 * max(1.0, np.abs(ref).max())


def test_host_misaligned_samples_fit_worse(regsim, ctrlsim):
    """the sample recipe matters: pairing each state with the torque of the step after it leaves a large residual"""
    torch = pytest.importorskip("torch")
    from abr_control_b200.arms import _ident

    true, nominal = perturbed("ur5", 3), _abi.load_arm_json("ur5")
    n, B, S, dt = 6, 8, 128, 1e-3
    q0, dq0, path, pv = sinusoid_paths(n, B, S, dt, 4)
    tr = shim_rollout(ctrlsim, true, "joint", dict(kp=400.0, kv=40.0), q0, dq0, path, pv, dt=dt)
    q, dq, ddq, u = samples(q0, dq0, tr, dt)
    flat = [a.reshape(-1, n) for a in (q[:-1], dq[:-1], ddq[:-1], u[1:])]

    def regress(i0, i1):
        return (torch.from_numpy(shim_regressor(regsim, nominal, *(a[i0:i1] for a in flat[:3]))),
                torch.from_numpy(np.ascontiguousarray(flat[3][i0:i1])))

    _, info = _ident.identify(regress, len(flat[0]), 1000, ident_oracle.theta(nominal), 1e-10)
    assert info["rms_after"] > 1e-4 * np.sqrt(np.mean(flat[3] ** 2))


def test_solve_drops_zero_columns_and_null_directions():
    from abr_control_b200.arms import _ident

    rng = np.random.default_rng(0)
    A = rng.normal(size=(50, 5)) * np.array([1e3, 1.0, 0.0, 1e-3, 1.0])
    A[:, 4] = A[:, 1] + A[:, 3] * 1e3  # a combination: one null direction besides the zero column
    x_true = np.array([1.0, 2.0, 3.0, 4.0, 5.0])
    b = A @ x_true
    x, directions, zero = _ident.solve(A.T @ A, A.T @ b, 1e-10)
    assert list(np.flatnonzero(zero)) == [2] and directions.shape == (5, 3)
    assert np.abs(A @ x - b).max() <= 1e-9 * np.abs(b).max()
    assert np.allclose(directions.T @ directions, np.eye(3), atol=1e-12)
    assert np.abs(x[2]) == 0.0 and np.abs(A @ (np.eye(5) - directions @ directions.T)).max() < 1e-6 * np.abs(A).max()


def test_tied_masses_and_tie_matrix():
    from abr_control_b200.arms import _ident

    th = np.arange(12.0)
    with pytest.raises(ValueError, match="unequal m_x"):
        _ident.tied(th, 2)
    th = np.array([2, 2, 2, 0.1, 0.2, 0.3, 5, 5, 5, 1, 2, 3.0])
    phi = _ident.tied(th, 2)
    assert np.array_equal(phi, [2, 0.1, 0.2, 0.3, 5, 1, 2, 3]) and np.array_equal(_ident.tie_matrix(2) @ phi, th)


# ---------------------------------------------------------------------------------------------- ABI and Python checks
@pytest.fixture(scope="module")
def native():
    from abr_control_b200 import _lib

    lib = _lib.lib()
    cd = _abi.chain_desc_from_dict(_abi.load_arm_json("ur5"))
    m = C.c_void_p()
    _lib.check(lib.abrb_model_create(C.byref(cd), C.byref(m)))
    yield lib, m, np.zeros(4096)
    lib.abrb_model_destroy(m)


FNS = ["abrb_inverse_dynamics_regressor_f64", "abrb_inverse_dynamics_regressor_f32"]


@pytest.mark.parametrize("fn", FNS)
def test_abi_rejects_bad_arguments_before_any_device_work(native, fn):
    lib, m, buf = native
    f = getattr(lib, fn)
    p = buf.ctypes.data
    ok = dict(m=m, q=p, dq=p, ddq=p, Yt=p, B=8)
    keys = ("m", "q", "dq", "ddq", "Yt", "B")
    bad = [
        (dict(m=None), _abi.EINVAL, "model"),
        (dict(q=None), _abi.EINVAL, "NULL q"),
        (dict(dq=None), _abi.EINVAL, "NULL dq"),
        (dict(ddq=None), _abi.EINVAL, "NULL ddq"),
        (dict(Yt=None), _abi.EINVAL, "NULL Yt"),
        (dict(B=-1), _abi.EINVAL, "B < 0"),
        (dict(q=p + 1), _abi.EINVAL, "misaligned pointer (q)"),
        (dict(dq=p + 2), _abi.EINVAL, "misaligned pointer (dq)"),
        (dict(ddq=p + 1), _abi.EINVAL, "misaligned pointer (ddq)"),
        (dict(Yt=p + 2), _abi.EINVAL, "misaligned pointer (Yt)"),
    ]
    for over, code, word in bad:
        a = {**ok, **over}
        rc = f(*[a[k] for k in keys], None)
        assert rc == code, (over, rc)
        msg = lib.abrb_last_error().decode()
        assert msg.startswith("abrb_inverse_dynamics_regressor") and word in msg, (over, msg)
    assert f(m, None, None, None, None, 0, None) == 0  # B == 0 is a no-op whatever the pointers
    if lib.abrb_device_count() <= 0:
        assert f(*[ok[k] for k in keys], None) == _abi.ECUDA
        assert "no CUDA device" in lib.abrb_last_error().decode()


def test_signatures_and_header_cover_the_regressor():
    from abr_control_b200 import _lib

    with open(os.path.join(ROOT, "include", "abrb.h")) as fh:
        hdr = fh.read()
    for fn in FNS:
        res, args = _lib.SIGNATURES[fn]
        assert res is C.c_int and args == [C.c_void_p] * 5 + [C.c_int64, C.c_void_p]
        assert f"int {fn}(" in hdr


def test_python_parameters_and_argument_checks():
    import abr_control_b200.arms as arms

    rc = arms.ur5.Config()
    th = rc.inertial_parameters()
    W = np.asarray(_abi.load_arm_json("ur5")["link_inertia"])
    assert th.dtype == np.float64 and th.shape == (36,) and np.array_equal(th, W[1:].reshape(-1))
    th2 = th * 1.5
    rc2 = rc.with_link_inertia(th2)
    assert np.array_equal(rc2.inertial_parameters(), th2) and rc2.N_JOINTS == 6 and rc2.dtype == rc.dtype
    assert np.array_equal(rc2.desc["link_inertia"][0], W[0]) and rc2.desc["A"] == rc.desc["A"]
    assert np.array_equal(rc.inertial_parameters(), th)  # the original is untouched
    with pytest.raises(ValueError, match="36 finite"):
        rc.with_link_inertia(th[:-1])
    with pytest.raises(ValueError, match="36 finite"):
        rc.with_link_inertia(np.full(36, np.nan))
    x = np.zeros((4, 6))
    untied = th.copy()
    untied[6] += 0.1
    with pytest.raises(ValueError, match=r"link\(s\) \[2\]"):
        rc.with_link_inertia(untied).identify_link_inertia(x, x, x, x)
    with pytest.raises(ValueError, match="chunk_states"):
        rc.identify_link_inertia(x, x, x, x, chunk_states=0)
    with pytest.raises(ValueError, match=r"\(K, 6\)"):
        rc.identify_link_inertia(x, x, x, np.zeros((3, 6)))
    with pytest.raises(ValueError, match=r"\(K, 6\)"):
        rc.identify_link_inertia(x[:0], x[:0], x[:0], x[:0])


# ============================================================================================== GPU
def _dev():
    import torch

    return torch.device("cuda")


def _t(a, dtype=None):
    import torch

    return torch.as_tensor(np.asarray(a, dtype=dtype or np.float64), device=_dev())


@pytest.mark.gpu
@pytest.mark.parametrize("f32", [0, 1])
@pytest.mark.parametrize("name", ARMS + ("rand1_ortho", "rand2_shear", "rand5_ortho", "rand7_ortho", "rand7_shear"))
def test_device_vs_shim(regsim, name, f32):
    from abr_control_b200.arms.base_config import BaseConfig

    desc = _chain(name)
    q, dq, ddq = states(desc["n_joints"], 300, 10)
    rc = BaseConfig(desc)
    dt = np.float32 if f32 else np.float64
    Y = rc.inverse_dynamics_regressor(_t(q, dt), _t(dq, dt), _t(ddq, dt)).cpu().numpy()
    ref = shim_regressor(regsim, desc, q.astype(dt), dq.astype(dt), ddq.astype(dt), f32)
    assert Y.dtype == dt and Y.shape == ref.shape
    assert np.abs(Y - ref).max() <= TOL[f32] * np.abs(ref).max()


@pytest.mark.gpu
@pytest.mark.parametrize("arm,B", [("ur5", 65536), ("jaco2", 140000)])
def test_device_regressor_times_theta_is_inverse_dynamics_at_full_size(arm, B):
    """140 000 states take a second grid-stride pass on a 132-SM H100 (8 CTAs of 128 per SM)"""
    import torch

    import abr_control_b200.arms as arms

    rc = getattr(arms, arm).Config()
    q, dq, ddq = (_t(a) for a in states(6, B, 11))
    Y = rc.inverse_dynamics_regressor(q, dq, ddq)
    assert Y.shape == (B, 6, 36) and Y.is_cuda and not Y.is_contiguous()
    u = rc.inverse_dynamics(q, dq, ddq)
    th = torch.as_tensor(rc.inertial_parameters(), device=q.device)
    err = (torch.matmul(Y, th) - u).abs().amax(dim=1) / u.abs().amax(dim=1).clamp(min=1.0)
    assert float(err.max()) <= 1e-12


@pytest.mark.gpu
def test_device_columns_are_inverse_dynamics_of_unit_inertias():
    import abr_control_b200.arms as arms

    rc = arms.ur5.Config()
    q, dq, ddq = (_t(a) for a in states(6, 4096, 12))
    Y = rc.inverse_dynamics_regressor(q, dq, ddq)
    scale = float(Y.abs().max())
    for p in range(36):
        e = np.zeros(36)
        e[p] = 1.0
        col = rc.with_link_inertia(e).inverse_dynamics(q, dq, ddq)
        assert float((Y[:, :, p] - col).abs().max()) <= 1e-12 * scale, p


@pytest.mark.gpu
def test_device_batch_edges_and_permutation_bit_identity():
    import torch

    import abr_control_b200.arms as arms

    rc = arms.jaco2.Config()
    q, dq, ddq = (_t(a) for a in states(6, 129, 13))
    full = rc.inverse_dynamics_regressor(q, dq, ddq)
    for B in (0, 1, 31, 33, 129):
        Y = rc.inverse_dynamics_regressor(q[:B], dq[:B], ddq[:B])
        assert Y.shape == (B, 6, 36) and torch.equal(Y, full[:B]), B
    perm = torch.randperm(129, generator=torch.Generator().manual_seed(0)).to(q.device)
    Y = rc.inverse_dynamics_regressor(q[perm], dq[perm], ddq[perm])
    assert torch.equal(Y, full[perm])


@pytest.mark.gpu
@pytest.mark.parametrize("f32", [0, 1])
def test_device_host_arrays_and_single_states_match_cuda_tensors(f32):
    import abr_control_b200.arms as arms

    dt = np.float32 if f32 else np.float64
    rc = arms.ur5.Config(dtype=dt)
    q, dq, ddq = (a.astype(dt) for a in states(6, 40, 14))
    ref = rc.inverse_dynamics_regressor(_t(q, dt), _t(dq, dt), _t(ddq, dt)).cpu().numpy()
    host = rc.inverse_dynamics_regressor(q, dq, ddq)
    assert isinstance(host, np.ndarray) and host.dtype == dt and np.array_equal(host, ref)
    # one NumPy state is evaluated in fp64 whatever the model's precision, as inverse_dynamics does
    one = rc.inverse_dynamics_regressor(q[3], dq[3], ddq[3])
    ref64 = rc.inverse_dynamics_regressor(*(_t(a[3:4]) for a in (q, dq, ddq))).cpu().numpy()[0]
    assert one.shape == (6, 36) and one.dtype == np.float64 and np.array_equal(one, ref64)
    one_t = rc.inverse_dynamics_regressor(_t(q[3], dt), _t(dq[3], dt), _t(ddq[3], dt))
    assert one_t.shape == (6, 36) and np.array_equal(one_t.cpu().numpy(), ref[3])


@pytest.mark.gpu
def test_device_identification_end_to_end():
    """4 096 x 128 Joint rollouts of a perturbed UR5, identified from the nominal model: the identified plant replays
    the recorded torques onto the true track"""
    import torch

    import abr_control_b200.arms as arms
    from abr_control_b200 import controllers
    from abr_control_b200.arms.base_config import BaseConfig

    nominal, true = arms.ur5.Config(), BaseConfig(perturbed("ur5", 5))
    B, S, dt, n = 4096, 128, 1e-3, 6
    q0, dq0, path, pv = (_t(a) for a in sinusoid_paths(n, B, S, dt, 6))
    _, _, tr, _ = controllers.Joint(true, kp=400.0, kv=40.0).rollout_path(q0, dq0, path, dt=dt, path_velocity=pv,
                                                                          record=("q", "dq", "u"))
    qp = torch.cat([q0[None], tr["q"][:-1]])
    dqp = torch.cat([dq0[None], tr["dq"][:-1]])
    ddq = (tr["dq"] - dqp) / dt
    theta, info = nominal.identify_link_inertia(*(a.reshape(-1, n) for a in (qp, dqp, ddq, tr["u"])),
                                                chunk_states=100000)
    u_rms = float(tr["u"].pow(2).mean().sqrt())
    assert info["rms_after"] <= 1e-9 * u_rms and info["rms_before"] > 1e-2 * u_rms, info
    th_true = true.inertial_parameters()
    assert np.abs(info["basis"].T @ (theta - th_true)).max() <= 1e-9 * np.abs(th_true).max()
    ident = nominal.with_link_inertia(theta)
    _, _, rep, _ = ident.simulate(q0, dq0, tr["u"], dt=dt, record=("q",))
    assert float((rep["q"] - tr["q"]).abs().max()) <= 1e-8
    # the same samples as host arrays, in float32 on an fp32 model: accumulated in fp64 all the same
    rc32 = arms.ur5.Config(dtype=np.float32)
    th32, info32 = rc32.identify_link_inertia(*(a.reshape(-1, n)[:65536].cpu().numpy() for a in (qp, dqp, ddq, tr["u"])))
    assert info32["rank"] == info["rank"] and info32["rms_after"] <= 1e-5 * u_rms
