"""GPU parity tests proper: the CUDA path, called through the C ABI (via the ctypes-based Python mirror of the
reference's interface), against the reference's golden fixtures and against the oracle on seeded inputs.

Tolerances (SURVEY.md S8d):
  * fp64 kernels vs raw fp64 reference / oracle: rtol 1e-10, atol 1e-12 for Tx, T, R, T_inv, J, dJ, M, g, C;
  * fp32 kernels vs the same: rtol 1e-4, atol 1e-5 (on quantities of O(1)), scaled by the row's magnitude;
  * OSC.generate: fp64 <= 1e-9 * |u|_inf of the fp64-mode reference; fp32 <= 1e-3 * |u|_inf, excluding states whose
    task-space inertia is ill conditioned (cond(J M^-1 J^T) > 1e4, where pinv truncation makes u discontinuous).
"""
import numpy as np
import pytest

import cases

pytestmark = pytest.mark.gpu

GOLD = __import__("os").path.join(__import__("os").path.dirname(__file__), "golden")


def _cfg(arm, **kw):
    import abr_control_b200.arms as arms

    return getattr(arms, arm).Config(**kw)


def _close(a, b, rtol, atol, what):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    assert a.shape == b.shape, (what, a.shape, b.shape)
    bad = np.abs(a - b) > atol + rtol * np.abs(b)
    assert not bad.any(), f"{what}: max abs err {np.abs(a - b).max():.3e} (rtol {rtol}, atol {atol})"


def _quat_close(a, b, tol, what):
    # q and -q are the same rotation and the reference's sign is arbitrary when w == 0 (rotation by pi)
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    e = np.minimum(np.abs(a - b).max(axis=-1), np.abs(a + b).max(axis=-1))
    flip_ok = np.abs(b[..., 0]) < 1e-7
    direct = np.abs(a - b).max(axis=-1)
    assert np.all((direct < tol) | (flip_ok & (e < tol))), f"{what}: {direct.max():.3e}"


@pytest.mark.parametrize("arm", list(cases.ARMS))
@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_rbd_vs_reference_golden(arm, dtype):
    g = np.load(f"{GOLD}/{arm}_rbd.npz")
    rc = _cfg(arm, dtype=dtype)
    q, dq, xoff = g["q"].astype(dtype), g["dq"].astype(dtype), g["xoff"]
    rtol, atol = (1e-10, 1e-12) if dtype == np.float64 else (1e-4, 2e-5)
    n = rc.N_JOINTS
    for fr in cases.frames(n):
        out = rc.eval(q, dq, name=fr, want=("Tx", "R", "T_inv", "J"))
        assert out["J"].dtype == dtype and out["J"].shape == (len(q), 6, n)
        _close(out["Tx"], g[f"Tx_{fr}"], rtol, atol, f"Tx {fr}")
        _close(out["R"], g[f"R_{fr}"], rtol, atol, f"R {fr}")
        _close(out["T_inv"], g[f"Tinv_{fr}"], rtol, atol, f"T_inv {fr}")
        _close(out["J"], g[f"J_{fr}"], rtol, atol, f"J {fr}")
    for fr in ("EE", cases.ARMS[arm]["mid"]):
        out = rc.eval(q, dq, name=fr, want=("T", "dJ", "quat"))
        _close(out["T"], g[f"T_{fr}"], rtol, atol, f"T {fr}")
        _close(out["dJ"], g[f"dJ_{fr}"], rtol * 10, atol * 50, f"dJ {fr}")
        _quat_close(out["quat"], g[f"quat_{fr}"], 1e-9 if dtype == np.float64 else 1e-5, f"quat {fr}")
        outx = rc.eval(q, dq, name=fr, x=xoff, want=("Tx", "J"))
        _close(outx["Tx"], g[f"Txx_{fr}"], rtol, atol, f"Tx(x) {fr}")
        _close(outx["J"], g[f"Jx_{fr}"], rtol, atol, f"J(x) {fr}")
    _close(rc.dJ("EE", q, dq, x=xoff), g["dJx_EE"], rtol * 10, atol * 50, "dJ(x) EE")
    dyn = rc.eval(q, dq, want=("M", "g") + (("C",) if "C" in g else ()))
    scale_g = max(1.0, np.abs(g["g"]).max())
    _close(dyn["M"], g["M"], rtol, atol * max(1.0, np.abs(g["M"]).max()), "M")
    _close(dyn["g"], g["g"], rtol, atol * scale_g * 10, "g")
    if "C" in g:
        _close(dyn["C"], g["C"], rtol * 10, atol * 50 * max(1.0, np.abs(g["C"]).max()), "C")


def test_jaco2_C_vs_oracle():
    """The reference cannot generate Jaco2's C (SURVEY.md S0.7); pin it through the oracle restatement, which is
    itself pinned on UR5/twojoint/threejoint where the reference C exists, and through finite differences of M."""
    from oracle import rbd_oracle

    rc = _cfg("jaco2")
    q, dq, _, _ = cases.states("jaco2", 24)
    C = rc.C(q, dq)
    _close(C, rbd_oracle.ChainOracle("jaco2").C(q, dq), 1e-10, 1e-11, "jaco2 C vs oracle")
    # Christoffel consistency: dM/dt = C + C^T along dq (finite differences of the GPU's own M)
    h = 1e-6
    Mdot = (rc.M(q + h * dq) - rc.M(q - h * dq)) / (2 * h)
    _close(C + np.swapaxes(C, 1, 2), Mdot, 1e-5, 1e-6, "Mdot = C + C^T")


def _build_ctrl(rc, case):
    from abr_control_b200 import controllers

    nulls = [getattr(controllers, k)(rc, **kw) for k, kw in case.get("null", [])] or None
    return controllers.OSC(rc, null_controllers=nulls, **case["osc"])


def _gen(ctrlr, case, q, dq, target, tvel):
    kw = {}
    if case.get("ref_frame"):
        kw["ref_frame"] = case["ref_frame"]
    if case.get("xyz_offset") is not None:
        kw["xyz_offset"] = case["xyz_offset"]
    if case.get("tv"):
        kw["target_velocity"] = tvel
    return ctrlr.generate(q, dq, target, **kw)


def _well_conditioned(case, q):
    """states whose J M^-1 J^T (controlled rows) has cond <= 1e4 (oracle-side diagnostic)."""
    from oracle import rbd_oracle

    ch = rbd_oracle.ChainOracle(case["arm"])
    mask = np.array(case["osc"].get("ctrlr_dof", [1, 1, 1, 0, 0, 0]), dtype=bool)
    x = case.get("xyz_offset")
    J = ch.J(case.get("ref_frame", "EE"), q, x)[:, mask]
    S = J @ np.linalg.inv(ch.M(q)) @ np.swapaxes(J, 1, 2)
    return np.linalg.cond(S) <= 1e4


@pytest.mark.parametrize("name", list(cases.OSC_CASES))
def test_osc_vs_reference_golden(name):
    case = cases.OSC_CASES[name]
    o = np.load(f"{GOLD}/{case['arm']}_osc.npz")
    q, dq, target, tvel = o["q"], o["dq"], o["target"], o["target_velocity"]
    ref = o[f"{name}__u64"]
    scale = np.abs(ref).max(axis=1, keepdims=True)
    ok = _well_conditioned(case, q)
    assert ok.sum() >= len(q) // 2
    # fp64
    rc = _cfg(case["arm"])
    ctrlr = _build_ctrl(rc, case)
    u = _gen(ctrlr, case, q, dq, target, tvel)
    assert u.dtype == np.float64 and u.shape == ref.shape
    err = np.abs(u - ref) / scale
    assert err[ok].max() < 1e-9, f"{name} fp64: {err[ok].max():.3e}"
    assert err.max() < 1e-6, f"{name} fp64 incl. ill-conditioned states: {err.max():.3e}"
    tr = np.abs(ctrlr.training_signal - o[f"{name}__train64"]) / scale
    assert tr[ok].max() < 1e-9
    # fp32 kernel against the fp64-mode reference
    rc32 = _cfg(case["arm"], dtype=np.float32)
    u32 = _gen(_build_ctrl(rc32, case), case, q.astype(np.float32), dq.astype(np.float32),
               target.astype(np.float32), tvel.astype(np.float32))
    assert u32.dtype == np.float32
    e32 = np.abs(u32 - ref) / scale
    assert e32[ok].max() < 1e-3, f"{name} fp32: {e32[ok].max():.3e}"
    # and the reference as shipped (float32-rounded J/M/g) is no closer to its own fp64 mode than we are, x10
    ship = np.abs(o[f"{name}__u32"] - ref) / scale
    assert np.median(e32[ok]) < 10 * max(np.median(ship[ok]), 1e-7)


@pytest.mark.parametrize("name", list(cases.NULL_CASES))
def test_null_controllers_vs_reference_golden(name):
    from abr_control_b200 import controllers

    case = cases.NULL_CASES[name]
    o = np.load(f"{GOLD}/{case['arm']}_osc.npz")
    rc = _cfg(case["arm"])
    kind, kw = case["ctrl"]
    ctrl = getattr(controllers, kind)(rc, **kw)
    u = ctrl.generate(o["q"], o["dq"])
    ref = o[f"{name}__null64"]
    _close(u, ref, 1e-8, 1e-9 * max(1.0, np.abs(ref).max()), name)


@pytest.mark.parametrize("name", list(cases.SLIDING_CASES))
def test_sliding_vs_reference_golden(name):
    import torch

    from abr_control_b200.controllers import Sliding

    cs = cases.SLIDING_CASES[name]
    o = np.load(f"{GOLD}/{cs['arm']}_osc.npz")
    q, dq = o["q"], o["dq"]
    tgt, tv, ta = cases.sliding_inputs(cs)
    ref, ref_s = o[f"{name}__sliding64"], o[f"{name}__s64"]
    kw = {}
    if cs.get("ref_frame"):
        kw["ref_frame"] = cs["ref_frame"]
    if cs.get("offset") is not None:
        kw["offset"] = cs["offset"]
    scale = np.abs(ref).max(axis=1, keepdims=True)
    sscale = np.abs(ref_s).max(axis=1, keepdims=True)
    for dtype, tol in ((np.float64, 1e-9), (np.float32, 5e-3)):
        ctrl = Sliding(_cfg(cs["arm"], dtype=dtype), **cs["ctrl"])
        cast = lambda a: None if a is None else a.astype(dtype)  # noqa: E731
        u = ctrl.generate(cast(q), cast(dq), cast(tgt), target_velocity=0 if tv is None else cast(tv),
                          target_acc=0 if ta is None else cast(ta), **kw)
        assert u.dtype == dtype and u.shape == ref.shape
        assert (np.abs(u - ref) / scale).max() < tol, (name, dtype)
        assert (np.abs(ctrl.s - ref_s) / sscale).max() < tol
    # one state: float64 out like the reference; CUDA tensors in -> CUDA tensors out
    ctrl = Sliding(_cfg(cs["arm"]), **cs["ctrl"])
    one = ctrl.generate(q[0], dq[0], tgt[0], target_velocity=0 if tv is None else tv[0],
                        target_acc=0 if ta is None else ta[0], **kw)
    assert one.shape == ref[0].shape and np.abs(one - ref[0]).max() < 1e-9 * max(1.0, np.abs(ref[0]).max())
    assert np.abs(ctrl.s - ref_s[0]).max() < 1e-9 * max(1.0, np.abs(ref_s[0]).max())
    ud = ctrl.generate(torch.as_tensor(q, device="cuda"), torch.as_tensor(dq, device="cuda"),
                       torch.as_tensor(tgt, device="cuda"), **kw)
    assert ud.is_cuda and ud.shape == ref.shape and ctrl.s.is_cuda


@pytest.mark.parametrize("name", list(cases.IK_CASES))
def test_inverse_kinematics_paths_vs_reference_golden(name):
    import torch

    from abr_control_b200.controllers.path_planners import InverseKinematics

    cs = cases.IK_CASES[name]
    o = np.load(f"{GOLD}/{cs['arm']}_ik.npz")
    position, target = o["position"], o["target"]
    ref_p, ref_v = o[f"{name}__pos64"], o[f"{name}__vel64"]
    vs = np.abs(ref_v).max()
    # fp64: the iteration is contracting, errors do not grow over the horizon; fp32 drifts by rounding per step
    for dtype, tol in ((np.float64, 1e-8), (np.float32, 2e-2)):
        ik = InverseKinematics(_cfg(cs["arm"], dtype=dtype), **cs.get("init", {}))
        pos, vel = ik.generate_path(position.astype(dtype), target.astype(dtype), **cs["path"])
        assert pos.shape == ref_p.shape and pos.dtype == dtype
        assert np.abs(vel - ref_v).max() < tol * vs, (name, dtype)
        assert np.abs(pos - ref_p).max() < tol * max(1.0, vs * ref_p.shape[1])
    ik = InverseKinematics(_cfg(cs["arm"]), **cs.get("init", {}))
    one_p, one_v = ik.generate_path(position[0], target[0], **cs["path"])  # the reference's single-path contract
    assert one_p.shape == ref_p[0].shape and np.abs(one_p - ref_p[0]).max() < 1e-8
    assert np.abs(one_v - ref_v[0]).max() < 1e-8 * vs
    p0, _ = ik.next()
    assert np.array_equal(p0, one_p[0]) and ik.n == 1
    dp, dv = ik.generate_path(torch.as_tensor(position, device="cuda"), torch.as_tensor(target[0], device="cuda"),
                              **cs["path"])  # CUDA tensors, one broadcast target
    assert dp.is_cuda and tuple(dp.shape) == ref_p.shape and bool(torch.isfinite(dv).all())


@pytest.mark.parametrize("name", list(cases.CTRL_CASES))
def test_joint_and_floating_vs_reference_golden(name):
    import torch

    from abr_control_b200 import controllers

    cs = cases.CTRL_CASES[name]
    o = np.load(f"{GOLD}/{cs['arm']}_osc.npz")
    q, dq, tq, tdq = o["q"], o["dq"], o["joint_target"], o["joint_target_velocity"]
    ref = o[f"{name}__ctrl64"]
    kind, kw = cs["ctrl"]
    for dtype, tol in ((np.float64, 1e-9), (np.float32, 2e-3)):
        rc = _cfg(cs["arm"], dtype=dtype)
        ctrl = getattr(controllers, kind)(rc, **kw)
        cast = lambda a: a.astype(dtype)  # noqa: E731
        if kind == "Joint":
            u = ctrl.generate(cast(q), cast(dq), cast(tq), cast(tdq) if cs.get("tv") else None)
            one = ctrl.generate(q[0], dq[0], tq[0], tdq[0] if cs.get("tv") else None)
        else:
            u = ctrl.generate(cast(q), cast(dq))
            one = ctrl.generate(q[0], dq[0])
        assert u.dtype == dtype and u.shape == ref.shape
        scale = np.abs(ref).max(axis=1, keepdims=True) + 1e-12
        assert (np.abs(u - ref) / scale).max() < tol, (name, dtype)
        assert one.shape == ref[0].shape and one.dtype == np.float64
        assert np.abs(one - ref[0]).max() < 1e-9 * max(1.0, np.abs(ref[0]).max())
    # CUDA tensors in -> CUDA tensor out
    rc = _cfg(cs["arm"])
    ctrl = getattr(controllers, kind)(rc, **kw)
    tq_, tdq_ = torch.as_tensor(q, device="cuda"), torch.as_tensor(dq, device="cuda")
    if kind == "Joint":
        ud = ctrl.generate(tq_, tdq_, torch.as_tensor(tq, device="cuda"))
    else:
        ud = ctrl.generate(tq_, tdq_)
    assert ud.is_cuda and ud.shape == ref.shape


def test_single_state_contract():
    """One state in -> the reference's shapes/dtypes out (float32 J/M/g/C/R, float64 Tx/T/T_inv, fresh arrays)."""
    from abr_control_b200.controllers import OSC

    rc = _cfg("ur5")
    g = np.load(f"{GOLD}/ur5_rbd.npz")
    q, dq = g["q"][3], g["dq"][3]
    J = rc.J("EE", q)
    assert J.shape == (6, 6) and J.dtype == np.float32
    assert np.allclose(J, g["J_EE"][3].astype(np.float32), rtol=1e-6, atol=1e-7)
    assert rc.M(list(q)).dtype == np.float32 and rc.g(q).shape == (6,) and rc.C(q, dq).dtype == np.float32
    assert rc.Tx("EE", q).dtype == np.float64 and rc.Tx("EE", q).shape == (3,)
    assert rc.T("EE", q).shape == (4, 4) and rc.T_inv("link3", q).shape == (4, 4) and rc.R("joint2", q).shape == (3, 3)
    with pytest.raises(Exception, match="Invalid transformation name"):
        rc.Tx("link9", q)
    with pytest.raises(Exception, match="Invalid transformation name"):
        rc.J("hand", q)
    ctrlr = OSC(rc, kp=10)
    o = np.load(f"{GOLD}/ur5_osc.npz")
    u = ctrlr.generate(o["q"][0], o["dq"][0], o["target"][0])
    assert u.shape == (6,) and u.dtype == np.float64 and u.flags.writeable
    ref = o["ur5_xyz__u64"][0]
    assert np.abs(u - ref).max() < 1e-9 * np.abs(ref).max()
    u *= -1  # CoppeliaSim.send_forces negates in place (interfaces/coppeliasim.py:204)
    assert ctrlr.training_signal.shape == (6,)
    assert OSC(rc, ki=0.1).integrated_error.shape == (6,)  # osc.py:81-82
    with pytest.raises(Exception, match="Invalid algorithm number"):
        OSC(rc, orientation_algorithm=2)


@pytest.mark.parametrize("B", [0, 1, 31, 32, 33, 127, 129, 1000])
def test_ragged_batches_and_device_tensors(B):
    """Empty, sub-warp and ragged batch sizes; CUDA-tensor path equals host-buffer path bit for bit."""
    import torch

    from abr_control_b200.controllers import OSC, Damping

    rc = _cfg("jaco2")
    q, dq, target, _ = cases.states("jaco2", max(B, 1))
    q, dq, target = q[:B], dq[:B], target[:B]
    ctrlr = OSC(rc, kp=200, ctrlr_dof=[True] * 5 + [False], null_controllers=[Damping(rc, kv=10)])
    u_host = ctrlr.generate(q, dq, target)
    assert u_host.shape == (B, 6)
    tq, tdq, tt = (torch.as_tensor(a, device="cuda") for a in (q, dq, target))
    u_dev = ctrlr.generate(tq, tdq, tt)
    assert u_dev.is_cuda and u_dev.shape == (B, 6)
    assert np.array_equal(u_dev.cpu().numpy(), u_host)
    if B:
        one = ctrlr.generate(q[B - 1], dq[B - 1], target[B - 1])
        assert np.array_equal(one, u_host[B - 1])
        out = rc.eval(tq, tdq, want=("J", "M", "g", "C", "Tx"))
        out_h = rc.eval(q, dq, want=("J", "M", "g", "C", "Tx"))
        for k in out:
            assert np.array_equal(out[k].cpu().numpy(), out_h[k]), k
        # broadcast target row
        ub = ctrlr.generate(q, dq, target[0])
        assert np.array_equal(ub[0], u_host[0])


def test_singular_states_take_the_pinv_branch():
    """Stretched-out planar arms make J M^-1 J^T singular: the reference's pinv(rcond=1e-4) branch (osc.py:143-145)."""
    from oracle import osc_oracle

    for arm, qs in (("twojoint", [[0.3, 0.0], [1.0, np.pi], [2.0, 1e-9]]),
                    ("threejoint", [[0.5, 0.0, 0.0], [1.0, np.pi, 0.0], [0.2, 1e-7, -1e-7]])):
        q = np.array(qs)
        dq = np.full_like(q, 0.3)
        target = np.tile([0.5, 0.4, 0, 0, 0, 0.0], (len(q), 1))
        case = dict(arm=arm, osc=dict(kp=10, ctrlr_dof=[True, True, False, False, False, False]))
        ref, _ = osc_oracle.run_case(case, q, dq, target)
        u = _gen(_build_ctrl(_cfg(arm), case), case, q, dq, target, None)
        assert np.all(np.isfinite(u))
        assert np.abs(u - ref).max() < 1e-7 * np.abs(ref).max(), (arm, u, ref)


def test_large_batch_deferred_pinv_states():
    """Every state of a 4096-state UR5 6-DOF batch that takes the truncating-pinv branch (|det| < 1e-3, ~3.75 % of
    uniformly random states) must match the oracle, fp64 and fp32, and must not depend on the batch it sits in."""
    from oracle import osc_oracle, rbd_oracle

    rng = np.random.default_rng(11)
    B = 4096
    q, dq, target = rng.uniform(0, 2 * np.pi, (B, 6)), rng.uniform(0, 5, (B, 6)), rng.uniform(-1, 1, (B, 6))
    ch = rbd_oracle.ChainOracle("ur5")
    J = ch.J("EE", q)
    S = J @ np.linalg.inv(ch.M(q)) @ np.swapaxes(J, 1, 2)
    slow = np.where(np.abs(np.linalg.det(S)) < 1e-3)[0]
    assert 80 < len(slow) < 300  # ~3.75 % of uniformly random states
    pick = np.concatenate([slow, np.arange(0, B, 97)])
    case = dict(arm="ur5", osc=dict(kp=50, ctrlr_dof=[True] * 6, use_C=True), null=[("Damping", dict(kv=10))])
    ref, _ = osc_oracle.run_case(case, q[pick], dq[pick], target[pick])
    scale = np.abs(ref).max(axis=1, keepdims=True)
    w = np.linalg.eigvalsh(S[pick])
    # states with an eigenvalue within 0.1 % of the pinv cutoff are genuinely ambiguous: exclude them
    clear = np.all(np.abs(w / (1e-4 * w[:, -1:]) - 1) > 1e-3, axis=1)
    for dtype, tol in ((np.float64, 1e-6), (np.float32, 5e-2)):
        rc = _cfg("ur5", dtype=dtype)
        ctrlr = _build_ctrl(rc, case)
        u = ctrlr.generate(q.astype(dtype), dq.astype(dtype), target.astype(dtype))
        err = (np.abs(u[pick] - ref) / scale).max(axis=1)
        assert err[clear].max() < tol, (dtype, err[clear].max())
        assert np.median(err) < (1e-12 if dtype == np.float64 else 1e-5)
        # and identical to evaluating the same rows in a small batch
        # (64 such states in one CTA overflow its queue of 32: half of them take the in-line cooperative route, the other
        # half the deferred one — same arithmetic, different rounding order)
        small = ctrlr.generate(q[slow[:64]].astype(dtype), dq[slow[:64]].astype(dtype), target[slow[:64]].astype(dtype))
        dev = np.abs(small - u[slow[:64]]).max(axis=1) / np.abs(u[slow[:64]]).max(axis=1)
        assert dev.max() < (1e-9 if dtype == np.float64 else 2e-5), (dtype, dev.max())


def test_cooperative_pinv_every_lane_and_ragged_batches():
    """The warp-cooperative truncating pseudo-inverse (abr_control_b200/csrc/abrb_coop.cuh) when EVERY lane of every warp
    needs it (a 3-joint arm asked to control 6 task DOF: J M^-1 J^T is rank deficient for every state, osc.py:91-98),
    i.e. eight passes of four states per warp, with batch sizes that leave ragged last warps / CTAs, fp64 and fp32,
    with a secondary controller (two right-hand sides) — against the oracle."""
    from oracle import osc_oracle

    rng = np.random.default_rng(41)
    for arm, n, dof in (("threejoint", 3, [True] * 6), ("twojoint", 2, [True, True, False, False, False, True]),
                        ("threejoint", 3, [True, True, True, False, False, False])):
        case = dict(arm=arm, osc=dict(kp=20, ctrlr_dof=dof), null=[("Damping", dict(kv=5))])
        for B in (1, 31, 33, 127, 129, 300):
            q, dq = rng.uniform(0.2, 2 * np.pi - 0.2, (B, n)), rng.uniform(-2, 2, (B, n))
            target = rng.uniform(-1, 1, (B, 6))
            ref, _ = osc_oracle.run_case(case, q, dq, target)
            scale = np.abs(ref).max(axis=1, keepdims=True)
            for dtype, tol in ((np.float64, 1e-8), (np.float32, 5e-3)):
                ctrlr = _build_ctrl(_cfg(arm, dtype=dtype), case)
                u = ctrlr.generate(q.astype(dtype), dq.astype(dtype), target.astype(dtype))
                err = (np.abs(u - ref) / scale).max(axis=1)
                assert np.isfinite(u).all() and np.quantile(err, 0.9) < tol and np.median(err) < tol * 0.1, (arm, dof, B, dtype, err.max())
    # one waiting lane per warp at most: UR5 rows picked so that exactly the chosen lanes are singular
    case = dict(arm="ur5", osc=dict(kp=50, ctrlr_dof=[True] * 6, use_C=True))
    q = rng.uniform(0.3, 6.0, (256, 6))
    q[5::32, 2] = 0.0  # elbow stretched: J loses rank
    q[5::32, 4] = 0.0
    dq, target = rng.uniform(-1, 1, (256, 6)), rng.uniform(-1, 1, (256, 6))
    ref, _ = osc_oracle.run_case(case, q, dq, target)
    u = _build_ctrl(_cfg("ur5"), case).generate(q, dq, target)
    err = np.abs(u - ref).max(axis=1) / np.abs(ref).max(axis=1)
    assert err.max() < 1e-6 and np.median(err) < 1e-12


def test_unaligned_row_slices_are_accepted():
    """Row slices of contiguous arrays start at element-aligned (not 16-byte aligned) addresses: q[1:] of an fp32 (B, 6)
    tensor is 24 bytes in.  The kernels only need element alignment (scalar loads and stores)."""
    import torch

    rc = _cfg("ur5", dtype=np.float32)
    ctrlr = _build_ctrl(rc, dict(arm="ur5", osc=dict(kp=10, ctrlr_dof=[True] * 6)))
    rng = np.random.default_rng(2)
    q, dq, tg = (torch.as_tensor(rng.uniform(0, 6, (1001, 6)), device="cuda", dtype=torch.float32) for _ in range(3))
    full = ctrlr.generate(q, dq, tg)
    for lo in (1, 3, 501):
        part = ctrlr.generate(q[lo:], dq[lo:], tg[lo:])
        assert torch.equal(part, full[lo:])
        out = torch.empty_like(q)
        ctrlr.generate_into(q[lo:], dq[lo:], tg[lo:], out[lo:])
        assert torch.equal(out[lo:], full[lo:])
    M = rc.M(q[1:])
    assert torch.equal(M, rc.M(q)[1:])


def test_cuda_graph_capture_and_replay():
    """A launch-bound inner loop captured once and replayed (torch.cuda.CUDAGraph): several OSC and rigid-body launches —
    issued with programmatic stream serialization, tile counters and deferred-state queues included — must give, on every
    replay, bit for bit what the same calls give eagerly; inputs are changed between replays through the captured buffers."""
    import torch

    rc = _cfg("ur5")
    ctrlr = _build_ctrl(rc, dict(arm="ur5", osc=dict(kp=10, ctrlr_dof=[True] * 6, use_C=True)))
    xyz = _build_ctrl(rc, dict(arm="ur5", osc=dict(kp=10)))
    rng = np.random.default_rng(11)
    Bq = 128 * 37 + 5  # ragged, several tiles per persistent CTA would need > 296 tiles: covered by the full-size tests
    mk = lambda: tuple(torch.as_tensor(rng.uniform(0, 6, (Bq, 6)), device="cuda") for _ in range(3))  # noqa: E731
    q, dq, tg = mk()
    outs = [torch.empty((Bq, 6), dtype=torch.float64, device="cuda") for _ in range(3)]
    M = torch.empty((Bq, 6, 6), dtype=torch.float64, device="cuda")
    g = torch.empty((Bq, 6), dtype=torch.float64, device="cuda")

    def work():
        ctrlr.generate_into(q, dq, tg, outs[0])
        rc.eval_into(q, dq, dict(M=M, g=g))
        xyz.generate_into(q, dq, tg, outs[1])
        ctrlr.generate_into(q, dq * 0.5, tg, outs[2])

    work()  # warm-up outside the capture (workspace, tile-counter pool, function attributes)
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(side):
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.graph(graph, stream=side):
            work()
    torch.cuda.synchronize()
    for rep in range(3):
        nq, ndq, ntg = mk()
        q.copy_(nq), dq.copy_(ndq), tg.copy_(ntg)
        for o in outs:
            o.zero_()
        M.zero_(), g.zero_()
        graph.replay()
        torch.cuda.synchronize()
        got = [o.clone() for o in outs] + [M.clone(), g.clone()]
        work()
        torch.cuda.synchronize()
        for a, b in zip(got, outs + [M, g]):
            assert torch.equal(a, b), f"replay {rep}"
        assert float(outs[0].abs().max()) > 0


def test_ki_integrator_sequences():
    """ki != 0 (osc.py:81-82, :262-264): per-state integrated task-space error over a 12-call sequence, fp64 and fp32,
    CUDA tensors and host arrays, against oracle controllers stepped the same way (one per state stream); the
    single-state path keeps the reference's `integrated_error` attribute."""
    import torch

    from oracle import osc_oracle as oo

    case = dict(arm="ur5", osc=dict(kp=30, ki=0.7, ctrlr_dof=[True] * 6, use_C=True), null=[("Damping", dict(kv=10))])
    Bq, T = 40, 12
    for dtype, tol in ((np.float64, 1e-9), (np.float32, 2e-3)):
        for kind in ("torch", "numpy"):
            rng = np.random.default_rng(9)
            refs = []
            for b in range(Bq):
                rco = oo.RobotOracle("ur5", "fp64")
                refs.append(oo.OSC(rco, null_controllers=[oo.Damping(rco, kv=10)], **case["osc"]))
            ctrlr = _build_ctrl(_cfg("ur5", dtype=dtype), case)
            for t in range(T):
                q, dq, tg = rng.uniform(0, 2 * np.pi, (Bq, 6)), rng.uniform(0, 2, (Bq, 6)), rng.uniform(-1, 1, (Bq, 6))
                ref = np.array([refs[b].generate(q[b], dq[b], tg[b]) for b in range(Bq)])
                args = [a.astype(dtype) for a in (q, dq, tg)]
                if kind == "torch":
                    u = ctrlr.generate(*[torch.as_tensor(a, device="cuda") for a in args]).cpu().numpy()
                else:
                    u = ctrlr.generate(*args)
                err = np.abs(u - ref).max(axis=1) / np.abs(ref).max(axis=1)
                assert np.median(err) < tol and np.quantile(err, 0.9) < tol * 50, (dtype, kind, t, err.max())
            (buf,) = ctrlr.integrated_error_batch.values()
            got = buf.cpu().numpy() if kind == "torch" else buf
            assert np.abs(got - np.array([c.err_sum for c in refs])).max() < (1e-10 if dtype == np.float64 else 1e-3)
            ctrlr.reset_integrated_error()
            assert not np.asarray(buf.cpu() if kind == "torch" else buf).any()
    # single state: the reference's attribute
    ctrlr = _build_ctrl(_cfg("ur5"), case)
    rco = oo.RobotOracle("ur5", "fp64")
    ref = oo.OSC(rco, null_controllers=[oo.Damping(rco, kv=10)], **case["osc"])
    rng = np.random.default_rng(1)
    for t in range(5):
        q, dq, tg = rng.uniform(0, 6, 6), rng.uniform(0, 1, 6), rng.uniform(-1, 1, 6)
        u, r = ctrlr.generate(q, dq, tg), ref.generate(q, dq, tg)
        assert np.abs(u - r).max() < 1e-9 * np.abs(r).max()
        assert np.abs(ctrlr.integrated_error - ref.err_sum).max() < 1e-12


def test_config5_obstacle_avoidance_on_a_large_random_batch():
    """BASELINE config 5 (Jaco2 OSC x,y,z + vmax + AvoidObstacles + Damping,
    /root/reference/examples/CoppeliaSim/force_osc_xyz_avoid_obstacle.py:17-28) on 8192 uniformly random states, fp32
    and fp64: EVERY state whose obstacle term is active and a sample of the others against the oracle."""
    from oracle import osc_oracle as oo

    rng = np.random.default_rng(55)
    B = 8192
    q, dq, target = rng.uniform(0, 2 * np.pi, (B, 6)), rng.uniform(0, 5, (B, 6)), rng.uniform(-1, 1, (B, 6))
    obstacle = [0.09596, -0.2661, 0.64204, 0.05]
    case = dict(arm="jaco2", osc=dict(kp=200, vmax=[0.5, 0], ctrlr_dof=[True, True, True, False, False, False]),
                null=[("AvoidObstacles", dict(obstacles=[obstacle], threshold=0.2)), ("Damping", dict(kv=10))])
    rco = oo.RobotOracle("jaco2", "fp64")
    avoid = oo.AvoidObstacles(rco, obstacles=[obstacle], threshold=0.2)
    active = np.array([np.any(avoid.generate(q[i]) != 0) for i in range(B)])
    assert 200 < active.sum() < 6000  # the obstacle sits inside the arm's workspace
    pick = np.concatenate([np.where(active)[0], np.where(~active)[0][::16]])
    ref, _ = oo.run_case(case, q[pick], dq[pick], target[pick])
    scale = np.abs(ref).max(axis=1, keepdims=True)
    for dtype, med, p99 in ((np.float64, 1e-12, 1e-8), (np.float32, 2e-5, 5e-3)):
        ctrlr = _build_ctrl(_cfg("jaco2", dtype=dtype), case)
        u = ctrlr.generate(q.astype(dtype), dq.astype(dtype), target.astype(dtype))
        err = (np.abs(u[pick] - ref) / scale).max(axis=1)
        assert np.isfinite(u).all() and np.median(err) < med and np.quantile(err, 0.99) < p99, (dtype, np.median(err), err.max())


def test_full_size_properties():
    """BASELINE configs at full size, through size-independent properties (the oracle is too slow here):
    config 2 (UR5 {J,M,g,C}, B=65536, fp64) and config 3 (Jaco2 OSC, B=262144, fp32)."""
    import torch

    from abr_control_b200.controllers import OSC, Damping

    rng = np.random.default_rng(7)
    B = 65536
    rc = _cfg("ur5")
    q = torch.as_tensor(rng.uniform(0, 2 * np.pi, (B, 6)), device="cuda")
    dq = torch.as_tensor(rng.uniform(0, 5, (B, 6)), device="cuda")
    out = rc.eval(q, dq, want=("J", "M", "g", "C", "Tx"))
    M, Cm = out["M"], out["C"]
    assert torch.equal(M, M.transpose(1, 2).contiguous())  # built from one triangle
    assert int(torch.linalg.cholesky_ex(M).info.abs().max()) == 0  # positive definite
    assert all(torch.isfinite(v).all() for v in out.values())
    # idempotence / determinism and batch-composition independence: a permuted batch gives permuted rows
    perm = torch.randperm(B, device="cuda")
    out_p = rc.eval(q[perm].contiguous(), dq[perm].contiguous(), want=("J", "M", "g", "C", "Tx"))
    for k in out:
        assert torch.equal(out_p[k], out[k][perm]), k
    # the Jacobian is the derivative of Tx: central differences along a random direction
    d = torch.as_tensor(rng.normal(size=(B, 6)), device="cuda")
    h = 1e-6
    fd = (rc.Tx("EE", q + h * d) - rc.Tx("EE", q - h * d)) / (2 * h)
    jd = torch.einsum("bij,bj->bi", out["J"][:, :3], d)
    assert (fd - jd).abs().max() < 1e-7
    # Christoffel identity: dM/dt - 2C is skew  <=>  dM/dt = C + C^T
    Mdot = (rc.M(q + h * dq) - rc.M(q - h * dq)) / (2 * h)
    assert (Cm + Cm.transpose(1, 2) - Mdot).abs().max() < 5e-5
    # gravity is minus the gradient of the potential energy sum_l m_l g z_l: check via energy differences
    # (skipped for brevity of runtime: covered at small size against the reference golden)

    B3 = 262144
    rc3 = _cfg("jaco2", dtype=np.float32)
    ctrlr = OSC(rc3, kp=200, ctrlr_dof=[True] * 5 + [False], null_controllers=[Damping(rc3, kv=10)])
    q3 = torch.as_tensor(rng.uniform(0, 2 * np.pi, (B3, 6)), device="cuda", dtype=torch.float32)
    dq3 = torch.as_tensor(rng.uniform(0, 5, (B3, 6)), device="cuda", dtype=torch.float32)
    t3 = torch.as_tensor(rng.uniform(-1, 1, (B3, 6)), device="cuda", dtype=torch.float32)
    u = ctrlr.generate(q3, dq3, t3)
    assert u.shape == (B3, 6) and torch.isfinite(u).all()
    perm = torch.randperm(B3, device="cuda")
    assert torch.equal(ctrlr.generate(q3[perm].contiguous(), dq3[perm].contiguous(), t3[perm].contiguous()), u[perm])
    # fp32 against the fp64 kernel on the same inputs
    rc3d = _cfg("jaco2")
    ctrlr_d = OSC(rc3d, kp=200, ctrlr_dof=[True] * 5 + [False], null_controllers=[Damping(rc3d, kv=10)])
    ud = ctrlr_d.generate(q3.double(), dq3.double(), t3.double())
    rel = (u.double() - ud).abs().amax(dim=1) / ud.abs().amax(dim=1)
    assert rel.median() < 1e-5 and torch.quantile(rel[:100000], 0.99) < 1e-3


def test_rollout_matches_stepwise():
    """The fused rollout kernel equals calling generate + the plant update step by step."""
    import torch

    from abr_control_b200.controllers import OSC

    rc = _cfg("ur5")
    ctrlr = OSC(rc, kp=10)
    q, dq, target, _ = cases.states("ur5", 64)
    dq = dq * 0.1
    steps, dt = 16, 1e-3
    qf, dqf, traj = ctrlr.rollout(q, dq, target, steps=steps, dt=dt)
    assert traj["q"].shape == (steps, 64, 6)
    qs, dqs = q.copy(), dq.copy()
    for t in range(steps):
        u = ctrlr.generate(qs, dqs, target)
        d = rc.eval(qs, dqs, want=("M", "g", "C"))
        rhs = u + d["g"] - np.einsum("bij,bj->bi", d["C"], dqs)
        ddq = np.linalg.solve(d["M"], rhs[..., None])[..., 0]
        dqs = dqs + ddq * dt
        qs = qs + dqs * dt
        assert np.abs(traj["u"][t] - u).max() < 1e-7 * max(1.0, np.abs(u).max())
    assert np.abs(qf - qs).max() < 1e-9 and np.abs(dqf - dqs).max() < 1e-7


@pytest.mark.parametrize("name,osc_kw", [("xyz", dict(kp=10)), ("6dof_C_ki", dict(kp=10, ki=0.2, ctrlr_dof=[True] * 6, use_C=True))])
def test_rollout_vs_oracle_stepped_loop(name, osc_kw):
    """BASELINE config 4's kernel against the ORACLE stepped the same way: u from oracle/osc_oracle.py, plant
    ddq = M^-1 (u + g - C dq) from oracle/rbd_oracle.py, semi-implicit Euler as
    /root/reference/abr_control/arms/twojoint/arm_sim.py:131-132 (dq += ddq dt; q += dq dt), 48 trajectories x 32 steps."""
    from oracle import osc_oracle as oo
    from oracle import rbd_oracle

    Bq, steps, dt = 48, 32, 1e-3
    q, dq, target, _ = cases.states("ur5", Bq)
    dq = dq * 0.1
    ctrlr = _build_ctrl(_cfg("ur5"), dict(arm="ur5", osc=osc_kw))
    qf, dqf, traj = ctrlr.rollout(q, dq, target, steps=steps, dt=dt)
    ch = rbd_oracle.ChainOracle("ur5")
    refs = [oo.OSC(oo.RobotOracle("ur5", "fp64"), **osc_kw) for _ in range(Bq)]
    qs, dqs = q.copy(), dq.copy()
    for t in range(steps):
        u = np.array([refs[b].generate(qs[b], dqs[b], target[b]) for b in range(Bq)])
        rhs = u + ch.g(qs) - np.einsum("bij,bj->bi", ch.C(qs, dqs), dqs)
        ddq = np.linalg.solve(ch.M(qs), rhs[..., None])[..., 0]
        dqs = dqs + ddq * dt
        qs = qs + dqs * dt
        # the closed loop amplifies rounding differences slowly: compare each step's u on the oracle's own state history
        assert np.abs(traj["u"][t] - u).max() < 1e-6 * max(1.0, np.abs(u).max()), t
        assert np.abs(traj["q"][t] - qs).max() < 1e-8 and np.abs(traj["dq"][t] - dqs).max() < 1e-6, t
    assert np.abs(qf - qs).max() < 1e-8 and np.abs(dqf - dqs).max() < 1e-6


# ---------------------------------------------------------------------------------------------------------------
# Chains that are not one of the four reference arms: every joint count the library is built for, orthonormal and
# sheared constant frames (SURVEY.md S8f row 4, the generic `_calc_T` contract of base_config.py:729-737), on the
# device through the C ABI — the same cases tests/test_generic_chains.py runs through the host instantiation.
@pytest.mark.parametrize("ortho", [True, False])
@pytest.mark.parametrize("n", [1, 2, 3, 4, 5, 6, 7])
def test_random_chains_rigid_body_quantities_on_the_device(n, ortho):
    from abr_control_b200.arms.base_config import BaseConfig
    from oracle import rbd_oracle as ro
    from test_generic_chains import random_chain

    desc = random_chain(n, ortho, 100 * n + ortho)
    c = ro.ChainOracle(desc)
    rng = np.random.default_rng(n)
    q, dq = rng.uniform(0, 2 * np.pi, (70, n)), rng.uniform(-3, 3, (70, n))
    for dtype, tol in ((np.float64, 1e-11), (np.float32, 3e-4)):
        rc = BaseConfig(desc, dtype=dtype)
        assert rc.N_JOINTS == n
        for fr in ("EE", f"link{n}", f"joint{n - 1}", "link0", f"link{(n + 1) // 2}"):
            o = rc.eval(q.astype(dtype), dq.astype(dtype), name=fr, want=("Tx", "R", "J", "dJ"))
            assert np.abs(o["Tx"] - c.Tx(fr, q)).max() < tol
            assert np.abs(o["R"] - c.R(fr, q)).max() < tol
            assert np.abs(o["J"] - c.J(fr, q)).max() < tol
            assert np.abs(o["dJ"] - c.dJ(fr, q, dq)).max() < tol * 30
        o = rc.eval(q.astype(dtype), dq.astype(dtype), want=("M", "g", "C"))
        for k, ref in (("M", c.M(q)), ("g", c.g(q)), ("C", c.C(q, dq))):
            assert np.abs(o[k] - ref).max() < tol * 10 * max(1.0, np.abs(ref).max()), (k, dtype)


@pytest.mark.parametrize("n,dof,ortho", [(1, [1, 0, 0, 0, 0, 0], True), (3, [1, 1, 1, 0, 0, 0], True),
                                         (4, [1, 1, 1, 0, 1, 0], True), (5, [1, 1, 1, 1, 1, 0], True),
                                         (5, [1, 1, 1, 1, 1, 1], False), (6, [1, 1, 1, 1, 1, 1], False),
                                         (7, [1, 1, 1, 1, 1, 1], True), (7, [1, 1, 1, 0, 0, 0], False)])
def test_random_chains_osc_rollout_and_controllers_on_the_device(n, dof, ortho):
    """OSC (incl. the redundant 7-joint arm and a 5-joint arm asked for 6 task DOF: every state on the cooperative
    pseudo-inverse route), the closed-loop rollout, Joint and Sliding on random chains vs the oracle."""
    import torch

    from abr_control_b200.arms.base_config import BaseConfig
    from abr_control_b200.controllers import OSC, Damping, Joint, Sliding
    from oracle import osc_oracle as oo
    from test_generic_chains import random_chain

    desc = random_chain(n, ortho, 7 * n + sum(dof), shear=2e-3)
    case = dict(arm=desc, osc=dict(kp=25, ko=15, ctrlr_dof=[bool(d) for d in dof], use_C=True), null=[("Damping", dict(kv=4))])
    rng = np.random.default_rng(n + 40)
    B = 70
    q, dq, target = rng.uniform(0, 2 * np.pi, (B, n)), rng.uniform(-2, 2, (B, n)), rng.uniform(-0.6, 0.6, (B, 6))
    ref, _ = oo.run_case(case, q, dq, target)
    scale = np.abs(ref).max(axis=1, keepdims=True)
    rank_deficient = sum(dof) > n
    for dtype, tol in ((np.float64, 1e-8), (np.float32, 2e-3)):
        rc = BaseConfig(desc, dtype=dtype)
        ctrlr = OSC(rc, null_controllers=[Damping(rc, kv=4)], **case["osc"])
        u = ctrlr.generate(q.astype(dtype), dq.astype(dtype), target.astype(dtype))
        err = (np.abs(u - ref) / scale).max(axis=1)
        assert np.median(err) < tol and np.quantile(err, 0.9) < tol * (1e3 if rank_deficient else 30), (dtype, err.max())
    # rollout = stepwise generate + plant with the device's own M, g, C
    rc = BaseConfig(desc)
    ctrlr = OSC(rc, **case["osc"])
    q0, dq0 = q[:33], 0.1 * dq[:33]
    qf, dqf, traj = ctrlr.rollout(q0, dq0, target[:33], steps=6, dt=1e-3)
    qs, dqs = q0.copy(), dq0.copy()
    for t in range(6):
        u = ctrlr.generate(qs, dqs, target[:33])
        d = rc.eval(qs, dqs, want=("M", "g", "C"))
        ddq = np.linalg.solve(d["M"], (u + d["g"] - np.einsum("bij,bj->bi", d["C"], dqs))[..., None])[..., 0]
        dqs = dqs + ddq * 1e-3
        qs = qs + dqs * 1e-3
        assert np.abs(traj["u"][t] - u).max() < 1e-6 * max(1.0, np.abs(u).max())
    assert np.abs(qf - qs).max() < 1e-9
    # Joint and Sliding (joint space) through their kernels
    tq = rng.uniform(0, 2 * np.pi, (B, n))
    uj = Joint(rc, kp=12, kv=3).generate(q, dq, tq)
    refj = np.array([oo.Joint(oo.RobotOracle(desc), kp=12, kv=3).generate(q[i], dq[i], tq[i]) for i in range(B)])
    assert np.abs(uj - refj).max() < 1e-9 * max(1.0, np.abs(refj).max())
    tg3 = rng.uniform(-0.4, 0.4, (B, 3))  # Cartesian rows are 3 wide whatever n is
    us = Sliding(rc, kd=40.0, lamb=12.0).generate(q, dq, tg3)
    refs, _ = oo.run_sliding_case(dict(arm=desc, ctrl=dict(kd=40.0, lamb=12.0)), q, dq, tg3, None, None)
    assert np.max(np.abs(us - refs) / np.abs(refs).max(axis=1, keepdims=True)) < 1e-8


def test_ki_integrator_vs_reference_golden():
    """ki != 0 against the REFERENCE's own call sequences (tests/golden/ur5_osc_ki.npz from
    oracle/ref_harness/run_reference_ki.py): 6 streams x 12 consecutive calls, u and integrated_error after every call,
    fp64 (vs the fp64 reference mode) and fp32 (vs the same, fp32 tolerance)."""
    import torch

    g = np.load(f"{GOLD}/ur5_osc_ki.npz")
    q, dq, target = g["q"], g["dq"], g["target"]
    T, S = q.shape[:2]
    case = dict(arm="ur5", osc=dict(kp=float(g["kp"]), ki=float(g["ki"]), ctrlr_dof=[True] * 6, use_C=True),
                null=[("Damping", dict(kv=10))])
    for dtype, tol, itol in ((np.float64, 1e-9, 1e-11), (np.float32, 2e-3, 1e-4)):
        ctrlr = _build_ctrl(_cfg("ur5", dtype=dtype), case)
        for t in range(T):
            u = ctrlr.generate(*[torch.as_tensor(a[t].astype(dtype), device="cuda") for a in (q, dq, target)]).cpu().numpy()
            ref = g["u64"][t]
            err = np.abs(u - ref).max(axis=1) / np.abs(ref).max(axis=1)
            assert np.median(err) < tol and err.max() < tol * 100, (dtype, t, err)
            (buf,) = ctrlr.integrated_error_batch.values()
            assert np.abs(buf.cpu().numpy() - g["integrated_error64"][t]).max() < itol, (dtype, t)


def test_mjcf_imported_chain_on_the_device(tmp_path):
    """An arm read from an MJCF file (abr_control_b200/arms/mjcf.py; the reference's MujocoConfig reads the same format,
    arms/mujoco_config.py:64-117) evaluated by the kernels against the oracle built from the imported descriptor."""
    from abr_control_b200.arms.mjcf import MjcfConfig, chain_desc_from_mjcf
    from oracle import rbd_oracle as ro
    from test_mjcf import _random_model, _write

    bodies, ee = _random_model(6, 77)
    path = str(tmp_path / "arm.xml")
    _write(path, bodies, ee)
    rc = MjcfConfig(path)
    c = ro.ChainOracle(chain_desc_from_mjcf(path))
    rng = np.random.default_rng(3)
    q, dq = rng.uniform(-np.pi, np.pi, (40, 6)), rng.uniform(-2, 2, (40, 6))
    out = rc.eval(q, dq, want=("Tx", "J", "M", "g", "C"))
    for k, ref in (("Tx", c.Tx("EE", q)), ("J", c.J("EE", q)), ("M", c.M(q)), ("g", c.g(q)), ("C", c.C(q, dq))):
        assert np.abs(out[k] - ref).max() < 1e-10 * max(1.0, np.abs(ref).max()), k
