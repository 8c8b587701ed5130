"""The general OSC kernel and the standalone secondary controllers at full size against a batched fp64 reference.

Every `OSC` call that is not plain task-space control (a secondary controller, a target velocity, ki, a frame other
than EE, an xyz_offset, a row mask, vmax, orientation algorithm 1) runs the general instantiation of the fused kernel
(`osc_kernel<..., PLAIN=false>`).  The small oracle tests reach it on at most a few thousand states, where no CTA takes
a second tile.  This module runs it where the persistent CTAs take several tiles each, their deferred pseudo-inverse
queues are flushed mid-loop with a non-zero null-space term and overflow into the in-line route, with every parity
case, with the two BASELINE workloads bench.py times on it (configs 3 and 5), at the ABRB_MAX_NULL = 4 and
ABRB_MAX_OBSTACLES = 16 limits, with ki over three calls, and the standalone secondary controllers (`null_kernel`)
where their grid-stride loop runs twice.

The reference is `oracle.osc_batch`, a batched NumPy restatement of `oracle.osc_oracle` (ChainOracle for the rigid-body
quantities), pinned to the per-state oracle on every parity case by the CPU tests below.  It is built once per arm and
case on a set of base states; results do not depend on a state's position in the batch, so the batches are tilings of
the base states and their references the same tilings of the reference.  The base states are rounded to fp32 once, so
that the fp64 and the fp32 kernels see the same inputs and the fp32 error measures the kernel, not input rounding.

Error measure and bounds: those of test_gpu_fullsize (`_check_f64`, `_check_f32`), with the states where u is
discontinuous and rounding may pick the side of the jump treated as its ambiguous (fp64) and sign(w) (fp32) states:
an eigenvalue of J M^-1 J^T at the pinv cut-off, |w| of the orientation quaternion at 0 (algorithms 0 and 1), an
obstacle pair's singular value at its rcond = 0.01 cut-off, q at a joint limit, a nearer_lo / nearer_hi tie on a
cross_zero joint, and RestingConfig's wrap at +-pi.  "At" is within 1e-9 in fp64 and within 1e-5 in fp32 (|w| as in
test_gpu_fullsize; the kernel's fp32 q - pi, q - lim and rest - q + pi carry a few ulp of 2 pi, ~1e-6).  The bound
on "well-conditioned" states applies where the rounding of the evaluation reaches u amplified by at most 1e4 (the
cond(J M^-1 J^T) <= 1e4 of test_gpu_fullsize), with the amplification through the secondary terms included: the
null-space projector's, and the obstacle terms' sensitivity to the arm's geometry (`_amplification`).
"""
import os
import re

import numpy as np
import pytest

import bench
import cases
import test_gpu_fullsize as fs
from oracle import osc_batch, osc_oracle
from oracle import rbd_oracle as ro

B0 = 65536            # base states per arm: each reference is built on these
BIG = 4 * B0          # 262 144
TILE = 128            # states per CTA tile (kBlock)
THREADS_PER_SM = 2048  # sm_90: a hard upper bound of 16 resident 128-thread CTAs per SM
REGS_PER_SM = 65536
PTXAS_LOG = os.path.join(fs.ROOT, "abr_control_b200", "csrc", "build", "ptxas_n{}.log")  # written by the build
TOL = {np.float64: 1e-9, np.float32: 1e-5}  # distance to a discontinuity within which rounding may pick the side


def _ctas_per_sm(n):
    """an upper bound on resident osc_kernel CTAs per SM for n joints: the register file over the fewest registers any
    instantiation uses (from the build's `ptxas -v` log, so it follows the code as compiled), and never more than the
    thread limit.  Without the log, the thread limit alone."""
    try:
        with open(PTXAS_LOG.format(n)) as fh:
            log = fh.read()
    except OSError:
        return THREADS_PER_SM // TILE
    regs = [int(m.group(1)) for m in re.finditer(r"Compiling entry function '[^']*osc_kernel[^']*'.*?Used (\d+) registers",
                                                  log, re.S)]
    assert regs, f"no osc_kernel entry in {PTXAS_LOG.format(n)}"
    return min(THREADS_PER_SM // TILE, REGS_PER_SM // (TILE * min(regs)))


# ---------------------------------------------------------------------------------------------- base states
def _base(arm):
    """(q, dq, target, target_velocity) of B0 states, fp32 values held in fp64.  UR5: bench.py's first timed set;
    Jaco2: the first B0 rows of the config 3 / config 5 inputs bench.py times; the planar arms: uniform draws as
    cases.states.  target_velocity ~U(-0.5, 0.5) with a quarter of the rows exactly zero, scattered, so that both
    branches of osc.py:275 occur within one warp."""
    n = cases.ARMS[arm]["n"]
    if arm == "ur5":
        q, dq, tg = bench.synth(B0, 6, 0)
    elif arm == "jaco2":
        q, dq, tg = (a[:B0] for a in bench.synth(BIG, 6, 9000, np.float32))
    else:
        rng = np.random.default_rng(cases.hash_name(arm) + 1)
        q, dq, tg = rng.uniform(0, 2 * np.pi, (B0, n)), rng.uniform(-5, 5, (B0, n)), rng.uniform(-1, 1, (B0, 6))
    rng = np.random.default_rng(cases.hash_name(arm) + 2)
    tv = rng.uniform(-0.5, 0.5, (B0, 6))
    tv[rng.random(B0) < 0.25] = 0.0
    return tuple(np.asarray(a, dtype=np.float32).astype(np.float64) for a in (q, dq, tg, tv))


class _Refs:
    """lazily built references on the base states, kept for the module (the C matrices per arm too)"""

    def __init__(self):
        self.base, self.C, self.ref = {}, {}, {}

    def states(self, arm):
        if arm not in self.base:
            self.base[arm] = _base(arm)
        return self.base[arm]

    def coriolis(self, arm):
        if arm not in self.C:
            q, dq, _, _ = self.states(arm)
            self.C[arm] = osc_batch.coriolis(ro.ChainOracle(arm), q, dq)
        return self.C[arm]

    def osc(self, key, case, tv=None):
        """the reference of `case` on its arm's base states; tv: None, "rows" (the base rows) or a (6,) vector"""
        if key not in self.ref:
            arm = case["arm"]
            q, dq, tg, tvr = self.states(arm)
            C = self.coriolis(arm) if case["osc"].get("use_C") else None
            tv = tvr if isinstance(tv, str) else tv
            r = self.ref[key] = osc_batch.generate(case, q, dq, tg, tv, C=C)
            if any(k == "AvoidObstacles" for k, _ in case.get("null", [])):
                r.gspread = _geometric_spread(lambda d: osc_batch.generate(dict(case, arm=d), q, dq, tg, tv, C=C).u, arm)
        return self.ref[key]


def _sms():
    import torch

    return torch.cuda.get_device_properties(0).multi_processor_count


def _tiling(seed, B):
    """B indices into the base states: independent permutations of them, concatenated and cut to B"""
    rng = np.random.default_rng(seed)
    return np.concatenate([rng.permutation(B0) for _ in range(-(-B // B0))])[:B]


def _size(n, at_least=BIG):
    """a batch with more tiles than twice the resident CTAs, so that every CTA takes several tiles"""
    need = (2 * _sms() * _ctas_per_sm(n) + 1) * TILE
    return max(at_least, -(-need // B0) * B0)


GEOM_REL = 4 * float(np.finfo(np.float32).eps)  # relative perturbation of the arm's constants (_geometric_spread)


def _geometric_spread(fn, arm):
    """the reference's own conditioning in the arm's geometry: the largest relative change of u (scale as _check_null)
    when every constant of the arm description is perturbed by +-GEOM_REL relative, two random draws.  The fp32 kernel
    holds positions with errors of that size.  Obstacle terms are ill conditioned there: a pair torque is about |F| / l
    over the distance l of its closest point from the joint axes acting on it, so an error dx of the positions moves
    it by |tau_pair| dx / l on every joint it acts on (through Mx ~ 1 / l^2), and the pair torques of one state can be
    thousands that cancel to tens (on Jaco2, joint 1's origin lies 9.4e-5 m from joint 0's axis).  Turning a joint
    does not change such a lever arm, so q-perturbations miss it.  fn(desc) evaluates the reference with the arm
    description desc."""
    base = ro.load_desc(arm)
    u0 = fn(base)
    scale = np.maximum(np.abs(u0).max(axis=1), 1e-3 * np.abs(u0).max())
    rng = np.random.default_rng(0)
    out = np.zeros(len(u0))
    for _ in range(2):
        desc = dict(base)
        for k in ("L0", "A", "B", "E"):
            a = np.asarray(base[k], dtype=float)
            desc[k] = (a * (1 + GEOM_REL * rng.choice([-1.0, 1.0], a.shape))).tolist()
        out = np.maximum(out, np.abs(fn(desc) - u0).max(axis=1) / scale)
    return out


def _amplification(r, idx, floor=False):
    """by how much the rounding of the evaluation is amplified onto u, relative to max|u| per state, in units of the
    dtype's epsilon (the role cond(J M^-1 J^T) plays in test_gpu_fullsize):
      cond(S) max(1, max|tau| / max|u|)   the projector I - J^T Jbar^T carries the error of Mx, eps cond(S), onto the
                                          sum tau of the secondary torques, which can exceed u itself;
      gspread / GEOM_REL                  the reference's measured sensitivity to the arm's geometry (obstacle terms,
                                          _geometric_spread).
    floor: max|u| floored at 1e-3 of the batch's largest, as _check_null measures errors."""
    umax = np.abs(r.u[idx]).max(axis=1)
    if floor:
        umax = np.maximum(umax, 1e-3 * np.abs(r.u).max())
    umax = np.where(umax > 0, umax, np.inf)
    get = lambda k, d: getattr(r, k)[idx] if hasattr(r, k) else d  # noqa: E731
    return get("cond", 1.0) * np.maximum(1.0, get("tau", 0.0) / umax) + get("gspread", 0.0) / GEOM_REL


def _view(r, idx, dtype, floor=False):
    """the reference rows `idx` as _check_f64 / _check_f32 read them: the discontinuity flags folded into their
    ambiguous (fp64) and sign(w) (fp32) states, and `cond` the amplification of the rounding (_amplification)"""
    tol = TOL[dtype]
    near = lambda k: getattr(r, k)[idx] < tol if hasattr(r, k) else np.zeros(len(idx), bool)  # noqa: E731
    jump = near("step") | near("tie") | near("wrap")
    trunc = r.trunc[idx] if hasattr(r, "trunc") else np.zeros(len(idx), bool)
    pinv = r.pinv[idx] if hasattr(r, "pinv") else np.zeros(len(idx), bool)
    cond = _amplification(r, idx, floor)
    amb = (r.amb[idx] if hasattr(r, "amb") else np.zeros(len(idx), bool)) | trunc
    w = r.w[idx] if hasattr(r, "w") else np.full(len(idx), np.inf)
    v = type("View", (), {})()
    v.pinv, v.cond = pinv, cond
    if dtype == np.float64:
        v.amb, v.wflip = amb | jump | (w < tol), np.zeros(len(idx), bool)
    else:
        v.amb, v.wflip = amb, jump | (w < 1e-5)
    return v


def _check(name, dtype, u, u_ref, r, idx):
    """_check_f64 / _check_f32 on rows idx of reference r (the view's own rows are 0..len(idx)-1)"""
    v = _view(r, idx, dtype)
    rows = np.arange(len(idx))
    (fs._check_f64 if dtype == np.float64 else fs._check_f32)(name, u, u_ref[idx], v, rows)
    return v


def _dt(dtype):
    return "f64" if dtype == np.float64 else "f32"


def _ctrl(case, dtype):
    from abr_control_b200 import controllers
    import abr_control_b200.arms as arms

    rc = getattr(arms, case["arm"]).Config(dtype=dtype)
    nulls = [getattr(controllers, k)(rc, **kw) for k, kw in case.get("null", [])] or None
    return controllers.OSC(rc, null_controllers=nulls, **case["osc"])


def _gen(ctrlr, case, q, dq, tg, tv=None):
    kw = {}
    if case.get("ref_frame"):
        kw["ref_frame"] = case["ref_frame"]
    if case.get("xyz_offset") is not None:
        kw["xyz_offset"] = case["xyz_offset"]
    if tv is not None:
        kw["target_velocity"] = tv
    return ctrlr.generate(q, dq, tg, **kw)


def _run(name, case, r, idx, tv=None, dtypes=(np.float64, np.float32), train=True):
    """the kernel on base rows idx (tv: None, "rows" or a (6,) vector), checked in both precisions"""
    arm = case["arm"]
    q, dq, tg, tvr = REFS.states(arm)
    for dtype in dtypes:
        args = fs._dev(q[idx], dq[idx], tg[idx], dtype=dtype)
        tvd = None
        if isinstance(tv, str):
            (tvd,) = fs._dev(tvr[idx], dtype=dtype)
        elif tv is not None:
            (tvd,) = fs._dev(np.asarray(tv, dtype=np.float64), dtype=dtype)
        ctrlr = _ctrl(case, dtype)
        u = _gen(ctrlr, case, *args, tv=tvd)
        _check(f"{name} {_dt(dtype)} B={len(idx)} u", dtype, u, r.u, r, idx)
        if train:
            _check(f"{name} {_dt(dtype)} B={len(idx)} training signal", dtype, ctrlr.training_signal, r.tr, r, idx)


REFS = _Refs()  # the references of this module's GPU tests, built on first use

# ---------------------------------------------------------------------------------------------- 1. the reference itself
def _draw(name, n, B=2048):
    rng = np.random.default_rng(cases.hash_name(name) + 5)
    q, dq, tg = rng.uniform(0, 2 * np.pi, (B, n)), rng.uniform(-5, 5, (B, n)), rng.uniform(-1, 1, (B, 6))
    tv = rng.uniform(-0.5, 0.5, (B, 6))
    tv[rng.random(B) < 0.25] = 0.0
    return q, dq, tg, tv


def _pick(rng, r, sparse_kinds, kinds, B, cap=512):
    """every pinv state, every state where a sparse secondary term (obstacles, joint limits) is non-zero, and 200
    others; obstacle terms with a threshold as large as the parity cases' are non-zero on nearly every state, so
    there at most `cap` of those are drawn (the per-state oracle takes ~15 ms per obstacle state)"""
    pick = [np.where(r.pinv)[0] if hasattr(r, "pinv") else np.zeros(0, int)]
    if any(k in sparse_kinds for k in kinds):
        act = np.where(r.active)[0]
        if "AvoidObstacles" in kinds and len(act) > cap:
            act = rng.choice(act, cap, replace=False)
        pick.append(act)
    pick.append(rng.choice(B, 200, replace=False))
    return np.unique(np.concatenate(pick))


def _agree(name, got, want, cond=None):
    """|got - want| per state over max|want| per state <= max(1e-10, 1e-15 cond(J M^-1 J^T)): two fp64 evaluations of
    the same maths in another order differ by ~eps x cond where the task-space inertia is inverted (not truncated)"""
    scale = np.abs(want).max(axis=1)
    err = np.abs(got - want).max(axis=1) / np.where(scale > 0, scale, 1.0)
    bound = np.maximum(1e-10, 1e-15 * (np.ones(len(err)) if cond is None else cond))
    fs._report(name, states=len(err), max=err.max(), max_over_bound=float((err / bound).max()))
    assert np.all(err <= bound), (name, err.max(), int(np.argmax(err / bound)))


@pytest.mark.parametrize("name", list(cases.OSC_CASES))
def test_batch_reference_vs_numpy_oracle(name):
    """osc_batch.generate against osc_oracle.run_case on a 2 048-state draw: u and the training signal on every
    pseudo-inverse state, every state where a joint-limit or obstacle term is non-zero, and 200 others.  A per-state
    target velocity with a quarter of its rows zero for the tv cases (both branches of osc.py:275)."""
    case = cases.OSC_CASES[name]
    q, dq, tg, tv = _draw(name, cases.ARMS[case["arm"]]["n"])
    tv = tv if case.get("tv") else None
    r = osc_batch.generate(case, q, dq, tg, tv)
    kinds = [k for k, _ in case.get("null", [])]
    pick = _pick(np.random.default_rng(1), r, ("AvoidObstacles", "AvoidJointLimits"), kinds, len(q))
    u, tr = osc_oracle.run_case(case, q[pick], dq[pick], tg[pick], None if tv is None else tv[pick])
    _agree(f"batch reference {name} u", r.u[pick], u, r.cond[pick])
    _agree(f"batch reference {name} training signal", r.tr[pick], tr, r.cond[pick])
    if case.get("tv"):
        assert 0 < r.rest.sum() < len(q)


@pytest.mark.parametrize("name", list(cases.NULL_CASES))
def test_batch_null_reference_vs_numpy_oracle(name):
    """osc_batch.null_generate against osc_oracle.run_null_case on a 2 048-state draw (the same choice of states)"""
    case = cases.NULL_CASES[name]
    q, dq, _, _ = _draw(name, cases.ARMS[case["arm"]]["n"])
    kind, kw = case["ctrl"]
    r = osc_batch.null_generate(case["arm"], kind, kw, q, dq)
    pick = _pick(np.random.default_rng(2), r, ("AvoidObstacles", "AvoidJointLimits"), [kind], len(q))
    u = osc_oracle.run_null_case(case, q[pick], dq[pick])
    zero = ~np.any(u != 0, axis=1)
    assert np.array_equal(zero, ~np.any(r.u[pick] != 0, axis=1)), name
    _agree(f"batch null reference {name}", r.u[pick][~zero], u[~zero])


def test_batch_reference_ki_sequence():
    """ki != 0: three calls, each on other states per row, against one stepped osc_oracle.OSC per row (u and the
    integrator rows after every call)"""
    case = dict(cases.OSC_CASES["ur5_6dof_C_damp"])
    case["osc"] = dict(case["osc"], ki=0.2)
    Bq = 64
    rco = osc_oracle.RobotOracle("ur5")
    rows = [osc_oracle.OSC(rco, null_controllers=[osc_oracle.Damping(rco, kv=10)], **case["osc"]) for _ in range(Bq)]
    es = np.zeros((Bq, 6))
    for t in range(3):
        q, dq, tg, _ = _draw(f"ki{t}", 6, Bq)
        r = osc_batch.generate(case, q, dq, tg, err_sum=es)
        es = r.err_sum
        u = np.array([rows[b].generate(q[b], dq[b], tg[b]) for b in range(Bq)])
        _agree(f"batch reference ki call {t} u", r.u, u, r.cond)
        assert np.abs(es - np.array([c.err_sum for c in rows])).max() < 1e-12 * np.abs(es).max()


# ---------------------------------------------------------------------------------------------- 2. every parity case
RAGGED = "ur5_vmax"  # runs at 262 144 - 37 states: a ragged last warp and tile
TV_BROADCAST = np.array([0.3, -0.2, 0.1, 0.25, -0.15, 0.05])  # non-zero (6,) target velocity, shared by every state


def _one_warp_both_branches(rest):
    w = rest[:len(rest) // 32 * 32].reshape(-1, 32)
    return bool((w.any(axis=1) & ~w.all(axis=1)).any())


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(cases.OSC_CASES))
def test_osc_cases_full_size(name):
    """Every parity case on >= 262 144 states (tilings of its arm's base states), fp64 and fp32, u and the training
    signal.  The tv cases take a per-state target velocity with a quarter of the rows zero (both branches of
    osc.py:275 within one warp) and then a broadcast non-zero (6,) one."""
    case = cases.OSC_CASES[name]
    n = cases.ARMS[case["arm"]]["n"]
    B = _size(n) - (37 if name == RAGGED else 0)
    assert -(-B // TILE) > 2 * _sms() * _ctas_per_sm(n)  # every resident CTA takes several tiles
    idx = _tiling(cases.hash_name(name), B)
    tv = "rows" if case.get("tv") else None
    r = REFS.osc(name, case, tv)
    fs._report(f"{name} reference", B=B, pinv=int(r.pinv[idx].sum()), ambiguous=int(r.amb[idx].sum()),
               secondary_active=int(r.active[idx].sum()))
    if tv:
        assert _one_warp_both_branches(r.rest[idx])
    _run(name, case, r, idx, tv)
    if tv:
        rb = REFS.osc(f"{name} broadcast tv", case, TV_BROADCAST)
        assert not rb.rest.any()
        _run(f"{name} broadcast tv", case, rb, idx, TV_BROADCAST)


# ---------------------------------------------------------------------------------------------- 3. configs 3 and 5
@pytest.mark.gpu
def test_bench_configs_3_and_5():
    """BASELINE configs 3 and 5 exactly as bench.py times them: its first input set of 262 144 Jaco2 states
    (`bench.synth(262144, 6, 9000, np.float32)`), its first 131 072 rows for config 5, generate_into, fp32, with the
    controllers of bench.py (the parity cases jaco2_cfg3 and jaco2_cfg5).  Every state against the reference, and
    config 5 separately on every state where the obstacle term is active.  The fp64 kernel on the same inputs too."""
    import torch

    q, dq, tg = (a.astype(np.float64) for a in bench.synth(BIG, 6, 9000, np.float32))
    for name, B in (("jaco2_cfg3", BIG), ("jaco2_cfg5", BIG // 2)):
        case = cases.OSC_CASES[name]
        r = osc_batch.generate(case, q[:B], dq[:B], tg[:B])
        if name == "jaco2_cfg5":
            r.gspread = _geometric_spread(lambda d: osc_batch.generate(dict(case, arm=d), q[:B], dq[:B], tg[:B]).u, "jaco2")
        fs._report(f"bench {name} reference", B=B, pinv=int(r.pinv.sum()), obstacle_active=int((r.pairs > 0).sum())
                   if hasattr(r, "pairs") else 0)
        idx = np.arange(B)
        for dtype in (np.float32, np.float64):
            ctrlr = _ctrl(case, dtype)
            args = fs._dev(q[:B], dq[:B], tg[:B], dtype=dtype)
            u = torch.empty_like(args[0])
            ctrlr.generate_into(*args, u)
            _check(f"bench {name} {_dt(dtype)} u", dtype, u, r.u, r, idx)
            if hasattr(r, "pairs"):
                act = np.where(r.pairs > 0)[0]
                assert len(act) > 0.05 * B  # the obstacle sits inside the arm's workspace
                _check(f"bench {name} {_dt(dtype)} u, obstacle-active states", dtype, u.cpu().numpy()[act], r.u, r, act)


# ---------------------------------------------------------------------------------------------- 4. deferred route
T, F, PI = True, False, float(np.pi)
DEFERRED = dict(arm="ur5", osc=dict(bench.OSC_KW),
                null=[("Damping", dict(kv=10)),
                      ("RestingConfig", dict(kp=30, kv=6, rest_angles=[None, PI / 4, -PI / 2, PI / 4, None, None]))])


@pytest.mark.gpu
def test_secondary_controllers_on_the_deferred_route():
    """bench.py's controller plus Damping(kv=10) and RestingConfig: a non-zero null-space term on every state, so the
    deferred pseudo-inverse records carry a second right-hand side (two = true in coop_flush_cta).  On the 262 144
    tiling (~10 000 pseudo-inverse states: the CTA queues fill and are flushed mid-loop, in one- and two-record
    rounds), fp64 and fp32; then, fp64, a 65 536 batch with every pseudo-inverse state in one contiguous block that
    starts on a tile boundary, so the queues overflow and the rest take the in-line route with two right-hand sides."""
    r = REFS.osc("deferred", DEFERRED)
    idx = _tiling(41, _size(6))
    assert 8000 < r.pinv[idx].sum() < 12000
    fs._report("deferred reference", pinv=int(r.pinv[idx].sum()))
    _run("deferred", DEFERRED, r, idx)
    slow, rest = np.where(r.pinv)[0], np.where(~r.pinv)[0]
    cut = 200 * TILE
    _run("deferred contiguous pinv block", DEFERRED, r, np.concatenate([rest[:cut], slow, rest[cut:]]),
         dtypes=(np.float64,))


# ---------------------------------------------------------------------------------------------- 5. the limits
# 16 obstacles (ABRB_MAX_OBSTACLES) of radius 4 cm inside the arms' workspace
OBSTACLES16 = [[x, y, z, 0.04] for x in (-0.3, -0.1, 0.1, 0.3)
               for (y, z) in ((-0.25, 0.35), (0.25, 0.55), (0.1, 0.25), (-0.1, 0.65))]
LIMITS = {  # four secondary controllers (ABRB_MAX_NULL)
    "ur5": dict(arm="ur5", osc=dict(kp=40, ko=30, ctrlr_dof=[T] * 6), null=[
        ("Damping", dict(kv=5)),
        ("RestingConfig", dict(kp=10, kv=3, rest_angles=[None, PI / 4, -PI / 2, PI / 4, None, None])),
        cases.OSC_CASES["ur5_limits_grad"]["null"][0],
        ("AvoidObstacles", dict(obstacles=OBSTACLES16, threshold=0.15, gain=1.0, maximum=100.0))]),
    "jaco2": dict(arm="jaco2", osc=dict(kp=100, ctrlr_dof=[T, T, T, F, F, F]), null=[
        ("Damping", dict(kv=5)),
        ("RestingConfig", dict(kp=10, kv=3, rest_angles=[None, 2.5, 1.0, None, 3.0, None])),
        ("AvoidJointLimits", dict(cases.NULL_CASES["jaco2_limits_wall"]["ctrl"][1],
                                  max_torque=[2.0, 3.0, 4.0, 1.0, 5.0, 6.0], gradient=[T, F, T, F, F, T])),
        ("AvoidObstacles", dict(obstacles=OBSTACLES16, threshold=0.15, gain=1.0, maximum=100.0))]),
}


@pytest.mark.gpu
@pytest.mark.parametrize("arm", list(LIMITS))
def test_four_secondary_controllers_and_sixteen_obstacles(arm):
    """One controller with ABRB_MAX_NULL = 4 secondary controllers (Damping, RestingConfig, AvoidJointLimits with
    exp(1/(q - lim)) gradients and a cross_zero joint, AvoidObstacles with ABRB_MAX_OBSTACLES = 16 obstacles) on the
    262 144 tiling, fp64 and fp32.  The joint-limit gradient is well conditioned wherever it is not clipped: it is
    only below max_torque where 1/|q - lim| < ln(max_torque), so |da/dq| = a / (q - lim)^2 < 8 / 0.48^2 here; the
    _check bounds hold unchanged."""
    case = LIMITS[arm]
    r = REFS.osc(f"limits {arm}", case)
    idx = _tiling(cases.hash_name(arm) + 43, _size(6))
    pairs = r.pairs[idx]
    fs._report(f"limits {arm} reference", pinv=int(r.pinv[idx].sum()), obstacle_states=int((pairs > 0).sum()),
               max_pairs=int(pairs.max()), limit_slope_max=float(r.slope.max()), truncated_pairs=int(r.trunc[idx].sum()))
    assert (pairs > 0).mean() > 0.2 and pairs.max() >= 8  # several obstacles act on one state
    _run(f"limits {arm}", case, r, idx)


# ---------------------------------------------------------------------------------------------- 6. ki
@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_integrator_three_calls_full_size(dtype):
    """ki = 0.2 on ur5_6dof_C_damp: three generate calls of 262 144 states, each on another permutation of the base
    states, with one integrator row per batch row.  u against the reference and integrated_error_batch against its
    err_sum after every call (fp64 1e-12, fp32 1e-5 relative to the largest row: the rows sum task-space errors of
    O(1), computed in the kernel's precision)."""
    case = dict(cases.OSC_CASES["ur5_6dof_C_damp"])
    case["osc"] = dict(case["osc"], ki=0.2)
    q, dq, tg, _ = REFS.states("ur5")
    C = REFS.coriolis("ur5")
    ctrlr = _ctrl(case, dtype)
    es = np.zeros((BIG, 6))
    for t in range(3):
        idx = _tiling(50 + t, BIG)
        key = f"ki call {t}"
        if key not in REFS.ref:
            REFS.ref[key] = osc_batch.generate(case, q[idx], dq[idx], tg[idx], err_sum=es, C=C[idx])
        r = REFS.ref[key]
        es = r.err_sum
        u = ctrlr.generate(*fs._dev(q[idx], dq[idx], tg[idx], dtype=dtype))
        _check(f"ki {_dt(dtype)} call {t} u", dtype, u, r.u, r, np.arange(BIG))
        (ie,) = ctrlr.integrated_error_batch.values()
        d = np.abs(ie.double().cpu().numpy() - es).max()
        fs._report(f"ki {_dt(dtype)} call {t} integrator", max_abs=d, max_row=float(np.abs(es).max()))
        assert d < (1e-12 if dtype == np.float64 else 1e-5) * np.abs(es).max(), (t, d)


# ---------------------------------------------------------------------------------------------- 7. null_kernel
B_NULL = 140_000  # null_kernel's grid is capped at 8 CTAs per SM: 1 056 x 128 = 135 168 states per round on 132 SMs


def _check_null(name, dtype, u, u_ref, r, idx):
    """per-state error relative to the state's largest torque, floored at 1e-3 of the batch's largest: obstacle and
    joint-limit terms fade out (or step) to exactly zero, and near there the kernel's rounding is absolute, not
    relative.  The bounds of _check_f64 / _check_f32: `well` are the states whose amplification (_amplification, with
    the same floor) is <= 1e4, `clear` those away from a discontinuity."""
    u = np.asarray(u.cpu(), dtype=np.float64)
    assert np.isfinite(u).all(), name
    ref = u_ref[idx]
    scale = np.maximum(np.abs(ref).max(axis=1), 1e-3 * np.abs(ref).max())
    err = np.abs(u - ref).max(axis=1) / scale
    v = _view(r, idx, dtype, floor=True)
    clear = ~(v.amb | v.wflip)
    well = clear & (v.cond <= 1e4)
    if dtype == np.float64:
        fs._report(name, median=float(np.median(err)), max_well=err[well].max(), max_clear=err[clear].max(),
                   not_well=int((~well).sum()))
        assert np.median(err) < 1e-12, (name, np.median(err))
        assert err[well].max() < 1e-9 and err[clear].max() < 1e-6, (name, err[well].max(), err[clear].max())
    else:
        fs._report(name, median=float(np.median(err)), p99_clear=float(np.quantile(err[clear], 0.99)),
                   max_well=err[well].max(), not_well=int((~well).sum()))
        assert np.median(err) < 2e-5, (name, np.median(err))
        assert np.quantile(err[clear], 0.99) < 5e-3 and err[well].max() < 1e-3, (
            name, np.quantile(err[clear], 0.99), err[well].max())


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(cases.NULL_CASES))
def test_null_cases_full_size(name):
    """Every standalone secondary controller on 140 000 states (two rounds of null_kernel's grid-stride loop), fp64
    and fp32, against osc_batch.null_generate on the arm's base states."""
    from abr_control_b200 import controllers
    import abr_control_b200.arms as arms

    case = cases.NULL_CASES[name]
    assert B_NULL > _sms() * 8 * TILE
    kind, kw = case["ctrl"]
    q, dq, _, _ = REFS.states(case["arm"])
    key = f"null {name}"
    if key not in REFS.ref:
        r = REFS.ref[key] = osc_batch.null_generate(case["arm"], kind, kw, q, dq)
        if kind == "AvoidObstacles":
            r.gspread = _geometric_spread(
                lambda d: osc_batch.null_generate(ro.ChainOracle(d), kind, kw, q, dq).u, case["arm"])
    r = REFS.ref[key]
    idx = _tiling(cases.hash_name(name) + 7, B_NULL)
    fs._report(f"null {name} reference", nonzero=int(r.active[idx].sum()))
    for dtype in (np.float64, np.float32):
        ctrl = getattr(controllers, kind)(getattr(arms, case["arm"]).Config(dtype=dtype), **kw)
        u = ctrl.generate(*fs._dev(q[idx], dq[idx], dtype=dtype))
        _check_null(f"null {name} {_dt(dtype)} B={B_NULL}", dtype, u, r.u, r, idx)
