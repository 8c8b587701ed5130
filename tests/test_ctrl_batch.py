"""CPU suite: the batched fp64 references of Joint, Floating, Sliding and InverseKinematics (oracle/ctrl_batch.py)
against the per-state oracles, and the kernels' per-state Sliding and IK code (tests/hostsim, g++) at singular poses
and on chains of fewer than three joints.

Singular poses: the home pose of each arm (every joint but the base at 0), where the arms stand straight and J[:3] or
J loses rank exactly, and straight-elbow poses (the elbow at 0, the other joints random).  There the reference drops a
singular value that is zero up to fp64 rounding; an fp32 evaluation of the same J leaves a residual of a few eps32 in
that direction, which the kernels' pseudo-inverses must drop as well (abrb_math.cuh, pinv_cut2).

Error model: rel err = max|du| / max|u_ref| per state.  Rounding reaches u through the pseudo-inverses amplified by
about 1 / smin (smallest kept relative singular value, oracle/ctrl_batch.py), so a state is held to
max(floor, K eps / smin); states with smin below the fp32 cut-off (1e-6) plus a margin are only required to be finite
in fp32, because there fp64 keeps a direction that fp32 cannot resolve.
"""
import ctypes as C

import numpy as np
import pytest

import cases
from abr_control_b200 import _abi
from oracle import ctrl_batch as cb
from oracle import ik_oracle
from oracle import osc_oracle as oo
from test_generic_chains import random_chain

ARMS = ("twojoint", "threejoint", "ur5", "jaco2")
ELBOW = dict(twojoint=1, threejoint=1, ur5=2, jaco2=2)
EPS = {0: np.finfo(np.float64).eps, 1: np.finfo(np.float32).eps}
AMBIGUOUS32 = 1e-5  # smin below this: fp32 may drop a direction fp64 keeps (cut 1e-6, a decade of margin)


def P(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def f32_exact(a):
    """round to fp32 and back: the inputs an fp32 evaluation sees exactly, so one fp64 reference serves both types"""
    return None if a is None else np.ascontiguousarray(np.asarray(a, dtype=np.float32), dtype=np.float64)


def _desc(arm):
    return _abi.load_arm_json(arm) if isinstance(arm, str) else arm


def home_states(arm, count, seed):
    """every joint but the base at 0, the base angle random"""
    n = _desc(arm)["n_joints"]
    q = np.zeros((count, n))
    q[:, 0] = np.random.default_rng(seed).uniform(0, 2 * np.pi, count)
    return f32_exact(q)


def straight_elbow_states(arm, count, seed):
    n = _desc(arm)["n_joints"]
    q = np.random.default_rng(seed).uniform(0, 2 * np.pi, (count, n))
    q[:, ELBOW[arm]] = 0.0
    return f32_exact(q)


def hs_sliding(hs, arm, q, dq, tg, tv=None, ta=None, f32=0, frame="EE", offset=None, kd=40.0, lamb=12.0,
               cartesian=True):
    cd = _abi.chain_desc_from_dict(_desc(arm))
    n, B = cd.n_joints, len(q)
    fid = hs.hs_frame_id(n, frame.encode())
    assert fid >= 0
    u, s = np.zeros((B, n)), np.zeros((B, n))
    q, dq, tg, tv, ta = (None if a is None else np.ascontiguousarray(a, dtype=np.float64) for a in (q, dq, tg, tv, ta))
    xo = None if offset is None else np.ascontiguousarray(offset, dtype=np.float64)
    assert hs.hs_sliding(C.byref(cd), f32, 0, C.c_double(kd), C.c_double(lamb), int(cartesian), fid, P(xo), P(q), P(dq),
                         P(tg), P(tv), P(ta), C.c_int64(B), P(u), P(s)) == 0
    return u, s


def hs_ik(hs, arm, q, tg, method, steps, dt, f32=0):
    """-> (pos, vel), each (B, steps, n)"""
    cd = _abi.chain_desc_from_dict(_desc(arm))
    n, B = cd.n_joints, len(q)
    pp, vv = np.zeros((steps, B, n)), np.zeros((steps, B, n))
    q, tg = np.ascontiguousarray(q, dtype=np.float64), np.ascontiguousarray(tg, dtype=np.float64)
    assert hs.hs_ik(C.byref(cd), f32, 0, C.c_double(0.2), C.c_double(2 * np.pi), C.c_double(np.pi), method,
                    C.c_double(dt), steps, P(q), P(tg), C.c_int64(B), P(pp), P(vv)) == 0
    return pp.transpose(1, 0, 2), vv.transpose(1, 0, 2)


def rel_err(u, ref):
    return np.abs(u - ref).max(axis=1) / np.maximum(np.abs(ref).max(axis=1), 1e-300)


def check_rel(err, smin, f32, floor, K, what):
    """every state within max(floor, K eps / smin); in fp32 states below AMBIGUOUS32 only finite (checked by the
    caller); -> the number of states held to the bound"""
    held = smin > AMBIGUOUS32 if f32 else smin > 1e-12
    bound = np.maximum(floor, K * EPS[f32] / smin)
    bad = held & ~(err <= bound)
    assert not bad.any(), (f"{what}: {bad.sum()} states out of bound; worst err {err[bad].max():.3e} at smin "
                           f"{smin[bad][np.argmax(err[bad])]:.3e}")
    return int(held.sum())


def sliding_inputs(rng, B, w):
    return (f32_exact(rng.uniform(-0.5, 0.5, (B, w))), f32_exact(rng.uniform(-0.3, 0.3, (B, w))),
            f32_exact(rng.uniform(-0.3, 0.3, (B, w))))


# ---------------------------------------------------------------------------------------------- references vs oracles
@pytest.mark.parametrize("name", list(cases.CTRL_CASES))
def test_joint_floating_batch_vs_oracle(name):
    cs = cases.CTRL_CASES[name]
    arm = cs["arm"]
    q, dq, _, _ = cases.states(arm, 160)
    q = np.vstack([q, home_states(arm, 40, 1), straight_elbow_states(arm, 40, 2)])
    dq = np.vstack([dq, np.random.default_rng(3).uniform(-2, 2, (80, q.shape[1]))])
    tq, tdq = cases.joint_targets(arm, len(q))
    kind, kw = cs["ctrl"]
    ref = oo.run_ctrl_case(cs, q, dq, tq, tdq)
    if kind == "Joint":
        r = cb.joint(arm, q, dq, tq, tdq if cs.get("tv") else None, **kw)
        keep = r.wrap > 1e-9
    else:
        r = cb.floating(arm, q, dq, **kw)
        keep = (r.det_gap > 1e-9) & ~r.amb
        if kw.get("task_space"):
            assert r.pinv.sum() >= 20, r.pinv.sum()  # both routes are pinned
    assert keep.sum() >= len(q) - 2
    assert rel_err(r.u, ref)[keep].max() < 1e-11


@pytest.mark.parametrize("arm,frame,offset,cartesian,extra", [
    ("ur5", "EE", None, True, False), ("ur5", "EE", cases.XOFF, True, True), ("ur5", "link3", cases.XOFF, True, True),
    ("jaco2", "joint1", None, True, True), ("jaco2", "link4", None, True, False), ("threejoint", "EE", None, True, True),
    ("twojoint", "EE", None, True, True), ("ur5", "EE", None, False, True), ("rand1", "EE", None, True, True),
    ("rand2", "EE", cases.XOFF, True, True)])
def test_sliding_batch_vs_oracle(arm, frame, offset, cartesian, extra):
    if arm.startswith("rand"):
        arm = random_chain(int(arm[4:]), True, 11)
    rng = np.random.default_rng(5)
    n = _desc(arm)["n_joints"]
    q = np.vstack([f32_exact(rng.uniform(0, 2 * np.pi, (120, n))), home_states(arm, 40, 6)])
    dq = f32_exact(rng.uniform(-2, 2, (len(q), n)))
    tg, tv, ta = sliding_inputs(rng, len(q), 3 if cartesian else n)
    if not extra:
        tv = ta = None
    kw = dict(kd=40.0, lamb=12.0, cartesian=cartesian)
    case = dict(arm=arm, ctrl=kw, ref_frame=frame, offset=offset)
    ref, ref_s = oo.run_sliding_case(case, q, dq, tg, tv, ta)
    r = cb.sliding(arm, q, dq, tg, tv, ta, ref_frame=frame, offset=offset, **kw)
    keep = r.smin > 1e-6
    assert keep.sum() >= len(q) - 4
    assert rel_err(r.u, ref)[keep].max() < 1e-10
    assert rel_err(r.s, ref_s)[keep].max() < 1e-10


@pytest.mark.parametrize("method", [1, 2, 3])
@pytest.mark.parametrize("arm", ["ur5", "jaco2", "threejoint"])
def test_ik_batch_vs_oracle(arm, method):
    n = _desc(arm)["n_joints"]
    q = np.vstack([cases.states(arm, 24)[0], home_states(arm, 8, 7)])
    tg = cases.ik_targets(arm, len(q))
    cs = dict(arm=arm, path=dict(n_timesteps=12, dt=0.05, method=method))
    ref_p, ref_v = ik_oracle.run_ik_case(cs, q, tg)
    r = cb.ik_path(arm, q, tg, **cs["path"])
    assert r.pos.shape == (len(q), 12, n)
    keep = r.smin > 1e-6
    assert keep.sum() >= len(q) // 2
    vs = np.abs(ref_v).max()
    assert np.abs(r.vel - ref_v)[keep].max() < 1e-10 * vs
    assert np.abs(r.pos - ref_p)[keep].max() < 1e-10


# ---------------------------------------------------------------------------------------------- kernel arithmetic
@pytest.mark.parametrize("f32", [0, 1])
@pytest.mark.parametrize("n", [1, 2, 3, 4, 5, 6, 7])
def test_sliding_random_chains(hostsim, n, f32):
    """Cartesian Sliding on random chains of every joint count; a Cartesian row is 3 wide whatever n is."""
    desc = random_chain(n, n % 2 == 0, 40 + n)
    rng = np.random.default_rng(n)
    B = 200
    q, dq = f32_exact(rng.uniform(0, 2 * np.pi, (B, n))), f32_exact(rng.uniform(-2, 2, (B, n)))
    tg, tv, ta = sliding_inputs(rng, B, 3)
    r = cb.sliding(desc, q, dq, tg, tv, ta, kd=40.0, lamb=12.0)
    u, s = hs_sliding(hostsim, desc, q, dq, tg, tv, ta, f32)
    assert np.isfinite(u).all() and np.isfinite(s).all()
    held = check_rel(rel_err(u, r.u), r.smin, f32, 1e-12 if not f32 else 1e-5, 1e3, f"n={n}")
    check_rel(rel_err(s, r.s), r.smin, f32, 1e-12 if not f32 else 1e-5, 1e3, f"s n={n}")
    assert held >= B - 4


def _singular_poses(arm):
    return np.vstack([home_states(arm, 48, 11), straight_elbow_states(arm, 48, 12)])


@pytest.mark.parametrize("f32", [0, 1])
@pytest.mark.parametrize("arm,frame", [(a, "EE") for a in ARMS] + [(a, fr) for a in ("ur5", "jaco2")
                                                                    for fr in cases.frames(6) if fr != "EE"])
def test_sliding_at_singular_poses(hostsim, arm, frame, f32):
    rng = np.random.default_rng(cases.hash_name(frame))
    q = _singular_poses(arm)
    B, n = q.shape
    dq = f32_exact(rng.uniform(-2, 2, (B, n)))
    tg, tv, ta = sliding_inputs(rng, B, 3)
    for offset in (None, cases.XOFF):
        r = cb.sliding(arm, q, dq, tg, tv, ta, kd=40.0, lamb=12.0, ref_frame=frame, offset=offset)
        u, s = hs_sliding(hostsim, arm, q, dq, tg, tv, ta, f32, frame, offset)
        assert np.isfinite(u).all() and np.isfinite(s).all(), (frame, offset)
        held = check_rel(rel_err(u, r.u), r.smin, f32, 1e-12 if not f32 else 1e-5, 1e3, f"{arm} {frame} {offset}")
        assert held >= B // 2


@pytest.mark.parametrize("f32", [0, 1])
@pytest.mark.parametrize("method", [1, 2, 3])
@pytest.mark.parametrize("arm", ARMS)
def test_ik_at_singular_poses(hostsim, arm, method, f32):
    """The first step from a singular pose against the reference, and every later step against the reference's step
    from the state the kernel reached (the paths of the two precisions part near singular poses)."""
    q = _singular_poses(arm)
    B, n = q.shape
    rng = np.random.default_rng(method)
    tg = f32_exact(np.hstack([rng.uniform(-0.5, 0.5, (B, 3)) + [0, 0, 0.3], rng.uniform(-np.pi, np.pi, (B, 3))]))
    steps, dt = 8, 0.01
    pos, vel = hs_ik(hostsim, arm, q, tg, method, steps, dt, f32)
    assert np.isfinite(pos).all() and np.isfinite(vel).all()
    assert np.array_equal(pos[:, 0], q)
    # the step from each state the kernel visited (fp32: that state in fp32, exactly representable)
    st = cb.ik_step(arm, pos.reshape(-1, n), np.repeat(tg, steps, axis=0), dt, method)
    err = np.abs(vel.reshape(-1, n) - st.dq).max(axis=1) / np.maximum(np.abs(st.dq).max(axis=1), st.scale)
    held = check_rel(err, st.smin, f32, 1e-12 if not f32 else 1e-5, 1e3, f"{arm} method {method}")
    assert held >= len(err) // 2
    if not f32:  # fp64 follows the whole reference path
        r = cb.ik_path(arm, q, tg, steps, dt, method)
        keep = r.smin > 1e-6
        assert np.abs(pos - r.pos)[keep].max() < 1e-10
