"""Joint, Floating, Sliding and InverseKinematics on the device at full size against the batched fp64 reference.

`ctrl_kernel` (Joint.generate, Floating.generate), `sliding_kernel` (Sliding.generate) and `ik_kernel`
(InverseKinematics.generate_path) are grid-stride loops over one state (or trajectory) per thread, launched with
`grid_for(B, 8)` CTAs of 128 threads: on a 132-SM H100 one pass covers 1 056 x 128 = 135 168 states, so B = 140 000
takes a second pass and B = 135 169 a second pass of one state.  This module checks those batch sizes and the odd ones
around a warp or a CTA, that a state's result does not depend on where it sits in the batch (permuted and tiled batches
give bit-identical rows), every Sliding frame of UR5 and Jaco2 with and without an offset, every Joint / Floating flag,
chains of one and two joints, and the singular home poses.

The reference is oracle/ctrl_batch.py (pinned to the per-state oracles by tests/test_ctrl_batch.py).  Inputs are rounded
to fp32 once, so the same fp64 reference serves both types.  The large batches are tilings and permutations of a set of
distinct states, and their references the same tilings of the set's reference.

Error measure: rel err = max|du| / max|u_ref| per state (Joint: over the larger of its terms, which can cancel).
fp64: <= 1e-9 on states whose pseudo-inverses keep no relative singular value below 1e-5 (`smin`; for IK method 2 the
inverse of the damped solve's amplification).  fp32: max(1e-4, 1e4 eps32 / smin) on every state with smin above the
fp32 cut-off plus a decade (1e-5), and bounds on the median and p99 of the well-conditioned states (smin > 1e-2); the
other states only have to be finite.
"""
import numpy as np
import pytest

import cases
from oracle import ctrl_batch as cb
from test_ctrl_batch import ARMS, f32_exact, home_states, straight_elbow_states
from test_generic_chains import random_chain

pytestmark = pytest.mark.gpu

EPS32 = float(np.finfo(np.float32).eps)
BIG = 140_000       # more than one grid-stride pass on a 132-SM H100 (1 056 CTAs x 128)
ODD = (1, 31, 33, 129, 135_169)
DISTINCT = 16_384   # distinct states behind the large batches
DTYPES = (np.float64, np.float32)


_MEMO = {}


def _memo(key, fn):
    """a reference computed once per module and shared by the fp64 and fp32 runs"""
    if key not in _MEMO:
        _MEMO[key] = fn()
    return _MEMO[key]


def _report(name, **vals):
    """one line per check with the observed figures (visible with pytest -s)"""
    print(f"[ctrl-fullsize] {name}: " + ", ".join(f"{k}={v:.3e}" if isinstance(v, float) else f"{k}={v}"
                                                  for k, v in vals.items()))


def _cfg(arm, dtype):
    if isinstance(arm, dict):
        from abr_control_b200.arms.base_config import BaseConfig

        return BaseConfig(arm, dtype=dtype)
    import abr_control_b200.arms as arms

    return getattr(arms, arm).Config(dtype=dtype)


def _np(a):
    return np.asarray(a.cpu() if hasattr(a, "cpu") else a, dtype=np.float64)


def _rel(u, ref):
    return np.abs(_np(u) - ref).max(axis=1) / np.maximum(np.abs(ref).max(axis=1), 1e-300)


def _cast(dtype, *arrays):
    return [None if a is None else np.ascontiguousarray(a, dtype=dtype) for a in arrays]


def _check(what, dtype, u, ref, smin=None, keep=None, scale=None, med32=1e-5, p9932=1e-3):
    """rel err = max|du| / max(max|u_ref|, scale) per state.  `smin`: 1 / the amplification of rounding (the smallest
    kept relative singular value, oracle/ctrl_batch.py).  fp64: every state in `keep` (default: smin > 1e-5) within
    1e-9.  fp32: finite everywhere; every state in `keep` within max(1e-4, 1e4 eps32 / smin); the median and p99
    over the well-conditioned ones (smin > 1e-2), where there are at least 100."""
    err = _rel(u, ref) if scale is None else np.abs(_np(u) - ref).max(axis=1) / np.maximum(np.abs(ref).max(axis=1), scale)
    smin = np.ones(len(err)) if smin is None else smin
    assert np.isfinite(_np(u)).all(), f"{what}: non-finite outputs"
    if keep is None:
        keep = smin > 1e-5
    e, well = err[keep], err[keep & (smin > 1e-2)]
    vals = dict(states=len(err), held=int(keep.sum()), max=float(e.max()), well=len(well))
    if len(well) >= 100:
        vals.update(median=float(np.median(well)), p99=float(np.quantile(well, 0.99)))
    _report(f"{what} {np.dtype(dtype).name}", **vals)
    assert keep.sum() >= len(err) // 2, what
    if dtype == np.float64:
        assert e.max() < 1e-9, what
    else:
        if len(well) >= 100:
            assert vals["median"] < med32 and vals["p99"] < p9932, what
        bound = np.maximum(1e-4, 1e4 * EPS32 / smin[keep])
        assert np.all(e <= bound), f"{what}: {(e > bound).sum()} states above max(1e-4, 1e4 eps / smin)"
    return err


def _tiling(n_distinct, B, seed):
    """indices into `n_distinct` states: concatenated independent permutations, cut to B"""
    rng = np.random.default_rng(seed)
    reps = -(-B // n_distinct)
    return np.concatenate([rng.permutation(n_distinct) for _ in range(reps)])[:B]


def _position_independent(what, run, idx, seed):
    """run(idx) on a permutation of the batch gives the same rows bit for bit"""
    perm = np.random.default_rng(seed).permutation(len(idx))
    a = _np(run(idx))
    b = _np(run(idx[perm]))
    same = np.array_equal(a[perm], b)
    _report(f"{what} permuted", states=len(idx), bit_identical=same)
    assert same, what
    return a


def _states(arm, B, seed, home_share=0.1):
    """random states with a share of home and straight-elbow poses, rounded to fp32"""
    n = arm["n_joints"] if isinstance(arm, dict) else cases.ARMS[arm]["n"]
    rng = np.random.default_rng(seed)
    q = f32_exact(rng.uniform(0, 2 * np.pi, (B, n)))
    dq = f32_exact(rng.uniform(-2, 2, (B, n)))
    if not isinstance(arm, dict):
        k = int(B * home_share) // 2
        q[:k] = home_states(arm, k, seed + 1)
        q[k:2 * k] = straight_elbow_states(arm, k, seed + 2)
    return q, dq


# ---------------------------------------------------------------------------------------------- Sliding
@pytest.fixture(scope="module")
def sliding_ref():
    arm, kw = "ur5", dict(kd=40.0, lamb=12.0)
    q, dq = _states(arm, DISTINCT, 1)
    rng = np.random.default_rng(2)
    tg, tv, ta = (f32_exact(rng.uniform(-a, a, (DISTINCT, 3))) for a in (0.6, 0.3, 0.3))
    r = cb.sliding(arm, q, dq, tg, tv, ta, ref_frame="EE", offset=cases.XOFF, **kw)
    _report("sliding reference", states=DISTINCT, smin_lt_1e5=int((r.smin < 1e-5).sum()))
    return dict(arm=arm, kw=kw, q=q, dq=dq, tg=tg, tv=tv, ta=ta, r=r)


@pytest.mark.parametrize("dtype", DTYPES)
def test_sliding_full_batch_and_odd_sizes(sliding_ref, dtype):
    from abr_control_b200.controllers import Sliding

    S = sliding_ref
    ctrl = Sliding(_cfg(S["arm"], dtype), **S["kw"])
    q, dq, tg, tv, ta = _cast(dtype, S["q"], S["dq"], S["tg"], S["tv"], S["ta"])

    def run(idx):
        return ctrl.generate(q[idx], dq[idx], tg[idx], target_velocity=tv[idx], target_acc=ta[idx],
                             offset=cases.XOFF)

    idx = _tiling(DISTINCT, BIG, 3)
    u = _position_independent("sliding", run, idx, 4)
    r = S["r"]
    _check(f"sliding B={BIG}", dtype, u, r.u[idx], r.smin[idx])
    run(idx)
    _check(f"sliding s B={BIG}", dtype, ctrl.s, r.s[idx], r.smin[idx])
    for B in ODD:
        ub = _np(run(idx[:B]))
        assert ub.shape == (B, 6) and np.array_equal(ub, u[:B]), B  # same rows as in the full batch, bit for bit
    _report(f"sliding odd sizes {np.dtype(dtype).name}", sizes=str(ODD), bit_identical_to_full=True)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("arm", ["ur5", "jaco2"])
def test_sliding_every_frame(arm, dtype):
    from abr_control_b200.controllers import Sliding

    B, kw = 1024, dict(kd=40.0, lamb=12.0)
    q, dq = _states(arm, B, 10, home_share=0.25)
    rng = np.random.default_rng(11)
    tg, tv = f32_exact(rng.uniform(-0.6, 0.6, (B, 3))), f32_exact(rng.uniform(-0.3, 0.3, (B, 3)))
    ctrl = Sliding(_cfg(arm, dtype), **kw)
    qc, dqc, tgc, tvc = _cast(dtype, q, dq, tg, tv)
    for frame in cases.frames(6):
        for offset in (None, cases.XOFF):
            r = _memo(("frame", arm, frame, offset is None),
                      lambda: cb.sliding(arm, q, dq, tg, tv, None, ref_frame=frame, offset=offset, **kw))
            u = ctrl.generate(qc, dqc, tgc, target_velocity=tvc, ref_frame=frame, offset=offset)
            _check(f"sliding {arm} {frame} offset={offset is not None}", dtype, u, r.u, r.smin)


@pytest.mark.parametrize("dtype", DTYPES)
def test_sliding_input_forms(dtype):
    """joint mode with rows / None, Cartesian with no target velocity or acceleration, a broadcast (stride-0) target"""
    from abr_control_b200.controllers import Sliding

    arm, B = "jaco2", 4099
    q, dq = _states(arm, B, 20)
    rng = np.random.default_rng(21)
    tq, tvq, taq = (f32_exact(rng.uniform(-a, a, (B, 6))) for a in (2 * np.pi, 1.0, 1.0))
    one = f32_exact(np.array([0.2, -0.3, 0.5]))
    rc = _cfg(arm, dtype)
    qc, dqc, tqc, tvqc, taqc = _cast(dtype, q, dq, tq, tvq, taq)
    jm = Sliding(rc, kd=20.0, lamb=5.0, cartesian=False)
    for tv, ta, label in ((tvq, taq, "rows"), (None, None, "none"), (tvq, None, "tv only")):
        r = cb.sliding(arm, q, dq, tq, tv, ta, kd=20.0, lamb=5.0, cartesian=False)
        kwg = {}
        if tv is not None:
            kwg["target_velocity"] = np.ascontiguousarray(tv, dtype=dtype)
        if ta is not None:
            kwg["target_acc"] = np.ascontiguousarray(ta, dtype=dtype)
        u = jm.generate(qc, dqc, tqc, **kwg)
        _check(f"sliding joint mode {label}", dtype, u, r.u)
        _check(f"sliding joint mode {label} s", dtype, jm.s, r.s)
    cm = Sliding(rc, kd=40.0, lamb=12.0)
    r = cb.sliding(arm, q, dq, one, None, None, kd=40.0, lamb=12.0)
    u = cm.generate(qc, dqc, one.astype(dtype))
    _check("sliding broadcast target", dtype, u, r.u, r.smin)
    _check("sliding broadcast target s", dtype, cm.s, r.s, r.smin)
    u2 = cm.generate(qc, dqc, np.ascontiguousarray(np.broadcast_to(one, (B, 3)), dtype=dtype))
    assert np.array_equal(_np(u), _np(u2))  # the stride-0 row and the same row per state agree bit for bit


# ---------------------------------------------------------------------------------------------- Joint / Floating
@pytest.mark.parametrize("dtype", DTYPES)
def test_joint_full_batch(dtype):
    from abr_control_b200.controllers import Joint

    arm = "ur5"
    q, dq = _states(arm, DISTINCT, 30)
    rng = np.random.default_rng(31)
    # target - q across (-pi, pi), shifted by 2 pi k, k in -3..3: the wrap of q_tilde
    tq = f32_exact(q + rng.uniform(-np.pi, np.pi, q.shape) + 2 * np.pi * rng.integers(-3, 4, q.shape))
    tv = f32_exact(rng.uniform(-1, 1, q.shape))
    idx = _tiling(DISTINCT, BIG, 32)
    qc, dqc, tqc, tvc = _cast(dtype, q, dq, tq, tv)
    for grav in (True, False):
        for with_tv in (True, False):
            kw = dict(kp=25.0, kv=7.0, account_for_gravity=grav)
            r = _memo(("joint", grav, with_tv), lambda: cb.joint(arm, q, dq, tq, tv if with_tv else None, **kw))
            ctrl = Joint(_cfg(arm, dtype), **kw)
            run = lambda i: ctrl.generate(qc[i], dqc[i], tqc[i], tvc[i] if with_tv else None)  # noqa: E731
            u = _position_independent(f"joint g={grav} tv={with_tv}", run, idx, 33)
            _check(f"joint B={BIG} gravity={grav} tv={with_tv}", dtype, u, r.u[idx], keep=r.wrap[idx] > 1e-3,
                   scale=r.scale[idx], p9932=1e-4)
            for B in ODD:
                assert np.array_equal(_np(run(idx[:B])), u[:B]), B
    # a broadcast (stride-0) target
    ctrl = Joint(_cfg(arm, dtype), kp=25.0, kv=7.0)
    r = cb.joint(arm, q, dq, tq[0], None, kp=25.0, kv=7.0)
    _check("joint broadcast target", dtype, ctrl.generate(qc, dqc, tqc[0]), r.u, keep=r.wrap > 1e-3, scale=r.scale)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("arm", ["ur5", "jaco2"])
def test_floating_every_flag(arm, dtype):
    from abr_control_b200.controllers import Floating

    q, dq = _states(arm, DISTINCT, 40, home_share=0.2)
    idx = _tiling(DISTINCT, BIG, 41)
    qc, dqc = _cast(dtype, q, dq)
    for task_space in (False, True):
        for dynamic in (False, True):
            r = _memo(("floating", arm, task_space, dynamic),
                      lambda: cb.floating(arm, q, dq, dynamic=dynamic, task_space=task_space))
            ctrl = Floating(_cfg(arm, dtype), dynamic=dynamic, task_space=task_space)
            u = _position_independent(f"floating {arm} ts={task_space} dyn={dynamic}",
                                      lambda i: ctrl.generate(qc[i], dqc[i]), idx, 42)
            near = r.det_gap < (1e-6 if dtype == np.float64 else 1e-2)
            keep = ~near & ~r.amb
            label = f"floating {arm} task_space={task_space} dynamic={dynamic}"
            if task_space:
                _report(label, pinv_route=int(r.pinv.sum()), pinv_route_held=int((r.pinv & keep).sum()),
                        near_det_switch=int(near.sum()))
                assert (r.pinv & keep).sum() >= 100  # the pinv(rcond=1e-4) route is exercised, not just present
            _check(f"{label} B={BIG}", dtype, u, r.u[idx], np.minimum(r.smin, 1 / r.cond)[idx], keep=keep[idx],
                   p9932=1e-4)
            for B in ODD:
                assert np.array_equal(_np(ctrl.generate(qc[idx[:B]], dqc[idx[:B]])), u[:B]), B


# ---------------------------------------------------------------------------------------------- InverseKinematics
IK_TRAJ, IK_DISTINCT, IK_STEPS, IK_DT = 65_536, 8_192, 24, 0.02


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("method", [1, 2, 3])
def test_ik_full_batch(method, dtype):
    import torch

    from abr_control_b200.controllers.path_planners import InverseKinematics

    arm = "ur5"
    q, _ = _states(arm, IK_DISTINCT, 50 + method, home_share=0.2)
    tg = f32_exact(cases.ik_targets(arm, IK_DISTINCT))
    idx = _tiling(IK_DISTINCT, IK_TRAJ, 52)
    ik = InverseKinematics(_cfg(arm, dtype))
    qd, tgd = (torch.as_tensor(np.ascontiguousarray(a[idx], dtype=dtype), device="cuda") for a in (q, tg))
    pos, vel = ik.generate_path(qd, tgd, n_timesteps=IK_STEPS, dt=IK_DT, method=method)
    n = q.shape[1]
    # (B, T, n) views of one (T, B, n) buffer
    assert tuple(pos.shape) == (IK_TRAJ, IK_STEPS, n) and pos.stride() == (n, IK_TRAJ * n, 1)
    assert vel.stride() == pos.stride()
    pos, vel = _np(pos), _np(vel)
    assert np.isfinite(pos).all() and np.isfinite(vel).all()
    assert np.array_equal(pos[:, 0], q[idx].astype(dtype).astype(np.float64))
    # trajectories are independent: the first 8 192 rows are each distinct state once; a permutation of them agrees
    perm = np.random.default_rng(53).permutation(IK_DISTINCT)
    pt = torch.as_tensor(perm, device="cuda")
    pos2, vel2 = ik.generate_path(qd[:IK_DISTINCT][pt], tgd[:IK_DISTINCT][pt], n_timesteps=IK_STEPS, dt=IK_DT,
                                  method=method)
    same = np.array_equal(_np(vel2), vel[:IK_DISTINCT][perm]) and np.array_equal(_np(pos2), pos[:IK_DISTINCT][perm])
    _report(f"ik m{method} permuted", trajectories=IK_DISTINCT, bit_identical=same)
    assert same
    label = f"ik m{method} {IK_TRAJ}x{IK_STEPS}"
    if dtype == np.float64:
        r = _memo(("ik", method), lambda: cb.ik_path(arm, q, tg, IK_STEPS, IK_DT, method))
        keep = r.smin[idx] > 1e-4  # rounding grows by up to 1 / smin at every step of the path
        e = np.abs(vel - r.vel[idx]).max(axis=(1, 2)) / np.abs(r.vel[idx]).max(axis=(1, 2))
        ep = np.abs(pos - r.pos[idx]).max(axis=(1, 2))
        _report(f"{label} float64", held=int(keep.sum()), vel_max=float(e[keep].max()), pos_max=float(ep[keep].max()))
        assert keep.sum() >= IK_TRAJ // 4 and e[keep].max() < 1e-9 and ep[keep].max() < 1e-9
    else:
        # each step against the reference's step from the state the kernel reached (the fp32 and fp64 paths part
        # near singular poses); a sample of the trajectories, every step
        sub = np.arange(0, IK_TRAJ, 16)
        st = cb.ik_step(arm, pos[sub].reshape(-1, n), np.repeat(tg[idx[sub]], IK_STEPS, axis=0), IK_DT, method)
        _check(label, dtype, vel[sub].reshape(-1, n), st.dq, st.smin, scale=st.scale)


# ---------------------------------------------------------------------------------------------- N < 3 and home poses
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("n", [1, 2])
def test_short_chains(n, dtype):
    """Sliding (Cartesian: 3-wide rows on a chain of fewer than three joints), Joint, Floating and IK"""
    from abr_control_b200.controllers import Floating, Joint, Sliding
    from abr_control_b200.controllers.path_planners import InverseKinematics

    desc = random_chain(n, True, 60 + n)
    B = 4099
    q, dq = _states(desc, B, 61)
    rng = np.random.default_rng(62)
    tg, tv, ta = (f32_exact(rng.uniform(-a, a, (B, 3))) for a in (0.5, 0.3, 0.3))
    rc = _cfg(desc, dtype)
    qc, dqc, tgc, tvc, tac = _cast(dtype, q, dq, tg, tv, ta)
    r = cb.sliding(desc, q, dq, tg, tv, ta, kd=40.0, lamb=12.0)
    ctrl = Sliding(rc, kd=40.0, lamb=12.0)
    _check(f"sliding n={n}", dtype, ctrl.generate(qc, dqc, tgc, target_velocity=tvc, target_acc=tac), r.u, r.smin)
    _check(f"sliding s n={n}", dtype, ctrl.s, r.s, r.smin)
    r = cb.sliding(desc, q, dq, tg[0], None, None, kd=40.0, lamb=12.0)
    _check(f"sliding n={n} broadcast", dtype, ctrl.generate(qc, dqc, tgc[0]), r.u, r.smin)
    tq = f32_exact(rng.uniform(-2 * np.pi, 4 * np.pi, (B, n)))
    r = cb.joint(desc, q, dq, tq, None, kp=12.0, kv=3.0)
    _check(f"joint n={n}", dtype, Joint(rc, kp=12.0, kv=3.0).generate(qc, dqc, tq.astype(dtype)), r.u,
           keep=r.wrap > 1e-3, scale=r.scale)
    for ts in (False, True):
        r = cb.floating(desc, q, dq, dynamic=True, task_space=ts)
        keep = (r.det_gap > (1e-6 if dtype == np.float64 else 1e-2)) & ~r.amb
        _check(f"floating n={n} task_space={ts}", dtype, Floating(rc, dynamic=True, task_space=ts).generate(qc, dqc),
               r.u, np.minimum(r.smin, 1 / r.cond), keep=keep)
    tgi = f32_exact(np.hstack([rng.uniform(-0.5, 0.5, (B, 3)), rng.uniform(-np.pi, np.pi, (B, 3))]))
    for method in (1, 2, 3):
        pos, vel = InverseKinematics(rc).generate_path(qc, tgi.astype(dtype), n_timesteps=8, dt=IK_DT, method=method)
        pos, vel = _np(pos), _np(vel)
        st = cb.ik_step(desc, pos.reshape(-1, n), np.repeat(tgi, 8, axis=0), IK_DT, method)
        _check(f"ik n={n} m{method}", dtype, vel.reshape(-1, n), st.dq, st.smin, scale=st.scale)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("arm", ARMS)
def test_home_poses(arm, dtype):
    """Sliding at every frame's worth of singular poses is in test_sliding_every_frame; here the home pose alone
    (every joint but the base at 0) for Sliding and the first IK steps, where fp32 used to return huge values"""
    from abr_control_b200.controllers import Sliding
    from abr_control_b200.controllers.path_planners import InverseKinematics

    B = 2048
    q = home_states(arm, B, 70)
    n = q.shape[1]
    rng = np.random.default_rng(71)
    dq = f32_exact(rng.uniform(-2, 2, (B, n)))
    tg, tv = f32_exact(rng.uniform(-0.5, 0.5, (B, 3))), f32_exact(rng.uniform(-0.3, 0.3, (B, 3)))
    rc = _cfg(arm, dtype)
    r = cb.sliding(arm, q, dq, tg, tv, None, kd=40.0, lamb=12.0)
    qc, dqc, tgc, tvc = _cast(dtype, q, dq, tg, tv)
    _check(f"sliding home {arm}", dtype, Sliding(rc, kd=40.0, lamb=12.0).generate(qc, dqc, tgc, target_velocity=tvc),
           r.u, r.smin)
    tgi = f32_exact(np.hstack([rng.uniform(-0.5, 0.5, (B, 3)) + [0, 0, 0.3], rng.uniform(-np.pi, np.pi, (B, 3))]))
    for method in (1, 2, 3):
        pos, vel = InverseKinematics(rc).generate_path(qc, tgi.astype(dtype), n_timesteps=4, dt=0.01, method=method)
        pos, vel = _np(pos), _np(vel)
        st = cb.ik_step(arm, pos.reshape(-1, n), np.repeat(tgi, 4, axis=0), 0.01, method)
        _check(f"ik home {arm} m{method}", dtype, vel.reshape(-1, n), st.dq, st.smin, scale=st.scale)


# ---------------------------------------------------------------------------------------------- fp32 rollout
def test_sliding_fp32_rollout_from_home_toward_unreachable_target():
    """Sliding.rollout_path shares sliding_state with generate.  From the twojoint home pose (stretched straight) toward
    a target out of reach along the arm, the position Jacobian has rank one and the error lies in its null space, so
    the controller holds the arm still: the fp64 reference gives |u| ~ 1e-5 at the start (from the fp32 rounding of
    the target off the arm's line).  In fp32 the null direction
    has a residual of a few eps32, which a cut-off of 1e-30 amplified to torques of 1e14-1e20.  The rollout must stay
    finite, start with the reference's u and keep the arm where it is.  (Past the first step the fp64 reference is no
    yardstick: rounding bends the elbow by ~1e-12 rad, a singular value numpy keeps and divides by.)"""
    from abr_control_b200.controllers import Sliding
    from oracle import rbd_oracle as ro

    arm, B, S, dt = "twojoint", 256, 40, 1e-3
    q0 = home_states(arm, B, 80)
    dq0 = np.zeros_like(q0)
    x0 = ro.ChainOracle(arm).Tx("EE", q0)
    target = f32_exact(3.0 * x0 / np.linalg.norm(x0, axis=1, keepdims=True))  # |x| = 3 m, the arm reaches ~0.5 m
    path = np.ascontiguousarray(np.broadcast_to(target, (S, B, 3)))
    qf, dqf, traj, _ = Sliding(_cfg(arm, np.float32), kd=40.0, lamb=12.0).rollout_path(
        q0.astype(np.float32), dq0.astype(np.float32), path.astype(np.float32), dt=dt)
    u32, q32 = _np(traj["u"]), _np(traj["q"])
    assert np.isfinite(u32).all() and np.isfinite(_np(qf)).all() and np.isfinite(_np(dqf)).all()
    r = cb.sliding(arm, q0, dq0, target, kd=40.0, lamb=12.0)
    first = float(np.abs(u32[0] - r.u).max())
    drift = float(np.abs(q32 - q0).max())
    _report("sliding fp32 rollout twojoint home", trajectories=B, steps=S, u_ref0=float(np.abs(r.u).max()),
            u32_0_err=first, max_u32=float(np.abs(u32).max()), max_q_drift=drift)
    assert np.abs(r.u).max() < 1e-3 and first < 1e-3 and np.abs(u32).max() < 1e-3 and drift < 1e-6
