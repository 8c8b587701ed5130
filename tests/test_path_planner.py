"""Batched path planner (``path_planners.PathPlanner``; ``abrb_path_plan``, ``abrb_path_fill_*``).

CPU part: the NumPy oracle (oracle/path_oracle.py) against the reference's own paths (tests/golden/path_planner.npz,
written by oracle/ref_harness/run_reference_path.py); the profiles' tables and ramps; the device's per-row and per-step
code run on the host through tests/hostsim/plannersim.cpp (TEST INFRASTRUCTURE, never loaded by the package) against
the oracle; the C ABI's argument checks; the Python-level rejections.
GPU part: the golden cases through the public API, single and batched, fp64 and fp32; 4 096 random reaches against the
oracle; batched rows against single-path calls; the planner feeding ``OSC.rollout_path``.
"""
import ctypes as C
import json
import os
import subprocess

import numpy as np
import pytest

from abr_control_b200 import _abi, _lib
from abr_control_b200.controllers.path_planners import PathPlanner, position_profiles, velocity_profiles
from abr_control_b200.controllers.path_planners.path_planner import AXES
from oracle import path_oracle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = np.load(os.path.join(ROOT, "tests", "golden", "path_planner.npz"))
META = json.loads(str(GOLD["meta"]))
CASES = list(range(len(META)))


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def rel_err(got, ref):
    """max |got - ref| over each column's largest |ref|"""
    scale = np.maximum(np.abs(ref).max(axis=-2, keepdims=True), 1e-300)
    return float(np.max(np.abs(got - ref) / scale))


def make_profiles(i):
    (pname, pkw), (vname, vkw) = META[i]["pos"], META[i]["vel"]
    pkw = dict(pkw)
    if pname == "FromPoints":
        pkw["x"], pkw["y"] = np.array(pkw["x"]), np.array(pkw["y"]).T
    return getattr(position_profiles, pname)(**pkw), getattr(velocity_profiles, vname)(**vkw)


def case_inputs(i):
    g = {k[len(f"c{i}_"):]: GOLD[k] for k in GOLD.files if k.startswith(f"c{i}_")}
    vm, v0, v1 = (float(v) for v in g["speeds"])
    kw = dict(max_velocity=vm, start_velocity=v0, target_velocity=v1)
    if META[i]["orient"]:
        kw.update(start_orientation=g["so"], target_orientation=g["to"])
    return g, kw


def oracle_case(i, table=None):
    g, kw = case_inputs(i)
    vname, vkw = META[i]["vel"]
    return path_oracle.plan(g["table"] if table is None else table, g["start"], g["target"], kw["max_velocity"],
                            kw["start_velocity"], kw["target_velocity"], vname.lower(), vkw["dt"], vkw["acceleration"],
                            vkw.get("n_sigma", 3), META[i]["axes"], kw.get("start_orientation"),
                            kw.get("target_orientation"))


def params(vname, vkw, n_points, axes):
    p = _abi.PathParams()
    p.vel_kind = getattr(velocity_profiles, vname).KIND
    p.n_points = n_points
    p.dt, p.acceleration, p.n_sigma = vkw["dt"], vkw["acceleration"], vkw.get("n_sigma", 3)
    for k, v in enumerate(AXES[axes]):
        p.axes[k] = v
    return p


# ---------------------------------------------------------------------------------------------- oracle and profiles
@pytest.mark.parametrize("i", CASES)
def test_oracle_equals_reference(i):
    g, _ = case_inputs(i)
    r = oracle_case(i)
    assert r["lengths"][0] == len(g["path"])
    assert not r["near_integer"][0], "golden cases are chosen away from length ties"
    assert rel_err(r["paths"][0], g["path"]) <= 1e-12


@pytest.mark.parametrize("i", CASES)
def test_profiles_sample_the_reference_table(i):
    prof, vel = make_profiles(i)
    planner = PathPlanner(prof, vel, axes=META[i]["axes"])
    assert np.abs(planner.table - GOLD[f"c{i}_table"]).max() <= 1e-15


@pytest.mark.parametrize("kind", ["Gaussian", "Linear"])
def test_velocity_profiles_generate(kind):
    vp = getattr(velocity_profiles, kind)(dt=0.001, acceleration=2.5)
    for va, vb in ((0.0, 1.0), (0.3, 0.9), (0.5, 0.55)):
        ref, _ = path_oracle.ramp(kind.lower(), 0.001, 2.5, 3, va, vb)
        got = vp.generate(va, vb)
        assert got.shape == ref.shape and np.abs(got - ref).max() <= 1e-15


def test_position_profile_endpoint_asserts():
    class Bad(position_profiles.PosProf):
        def step(self, t):
            return np.array([t, t, 2 * t])

    with pytest.raises(AssertionError):
        Bad()
    position_profiles.Ellipse(-0.5, plane="yz")


# ---------------------------------------------------------------------------------------------- host shim
@pytest.fixture(scope="module")
def plannersim(tmp_path_factory):
    src = os.path.join(ROOT, "tests", "hostsim", "plannersim.cpp")
    so = str(tmp_path_factory.mktemp("plannersim") / "_plannersim.so")
    subprocess.run(["g++", "-O1", "-std=c++17", "-shared", "-fPIC", "-x", "c++", src, "-o", so], check=True)
    lib = C.CDLL(so)
    lib.pl_plan_row.restype = C.c_int64
    lib.pl_plan_row.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_double, C.c_double, C.c_double,
                                C.c_void_p]
    lib.pl_fill_row.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_double, C.c_double, C.c_void_p,
                                C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]
    lib.pl_ramp.argtypes = [C.c_void_p, C.c_double, C.c_double, C.c_int, C.c_void_p]
    lib.pl_slerp.argtypes = [C.c_void_p, C.c_void_p, C.c_double, C.c_void_p]
    return lib


def shim_path(lib, p, table, start, target, vm, v0, v1, so=None, to=None):
    rec = _abi.PathRec()
    args = [np.ascontiguousarray(a, dtype=np.float64) for a in (table, start, target)]
    S = lib.pl_plan_row(C.byref(p), *(_p(a) for a in args), vm, v0, v1, C.byref(rec))
    if S < 2:
        return S, None
    o = [None if a is None else np.ascontiguousarray(a, dtype=np.float64) for a in (so, to)]
    out = np.zeros((S, 12 if so is not None else 6))
    assert lib.pl_fill_row(C.byref(p), *(_p(a) for a in args), v0, v1, _p(o[0]), _p(o[1]), C.byref(rec), S,
                           _p(out)) == 0
    return S, out


@pytest.mark.parametrize("i", CASES)
def test_shim_equals_oracle_on_golden_cases(plannersim, i):
    g, kw = case_inputs(i)
    vname, vkw = META[i]["vel"]
    p = params(vname, vkw, len(g["table"]), META[i]["axes"])
    S, rows = shim_path(plannersim, p, g["table"], g["start"], g["target"], kw["max_velocity"], kw["start_velocity"],
                        kw["target_velocity"], kw.get("start_orientation"), kw.get("target_orientation"))
    assert S == len(g["path"])
    assert rel_err(rows, oracle_case(i)["paths"][0]) <= 1e-12
    assert rel_err(rows, g["path"]) <= 1e-12


@pytest.mark.parametrize("axes", sorted(AXES))
def test_shim_random_rows_equal_oracle(plannersim, axes):
    rng = np.random.default_rng(sum(map(ord, axes)))
    prof = [position_profiles.Linear(), position_profiles.SinCurve(axes=["y"], n_sample_points=300),
            position_profiles.Ellipse(-0.6, plane="xz", n_sample_points=200)][rng.integers(3)]
    table = PathPlanner(prof, velocity_profiles.Linear(0.002, 4)).table
    vname = ["Gaussian", "Linear"][rng.integers(2)]
    vkw = dict(dt=0.002, acceleration=float(rng.uniform(2, 6)))
    p = params(vname, vkw, len(table), axes)
    for _ in range(4):
        start, target = rng.uniform(-0.5, 0.5, 3), rng.uniform(-0.5, 0.5, 3)
        vm = float(rng.uniform(0.5, 1.5))
        v0, v1 = float(rng.choice([0.0, 0.2 * vm, vm])), float(rng.choice([0.0, 0.3 * vm]))
        so, to = rng.uniform(-np.pi, np.pi, 3), rng.uniform(-np.pi, np.pi, 3)
        r = path_oracle.plan(table, start, target, vm, v0, v1, vname.lower(), vkw["dt"], vkw["acceleration"], 3, axes,
                             so, to)
        S, rows = shim_path(plannersim, p, table, start, target, vm, v0, v1, so, to)
        if r["near_integer"][0]:
            assert abs(S - r["lengths"][0]) <= 1
            continue
        assert S == r["lengths"][0]
        if S >= 2:
            assert rel_err(rows[:, :9], r["paths"][0][:, :9]) <= 1e-11
            # the angular velocity differentiates the Euler angles, so a wrap at +-pi between neighbours is a jump of
            # 2 pi / dt that both sides must place on the same step
            assert rel_err(rows[:, 9:], r["paths"][0][:, 9:]) <= 1e-9


@pytest.mark.parametrize("axes", sorted(AXES))
def test_shim_orientation_functions_equal_oracle(plannersim, axes):
    rng = np.random.default_rng(7 + sum(map(ord, axes)))
    ax = (C.c_int32 * 4)(*AXES[axes])
    for _ in range(50):
        e0, e1 = rng.uniform(-np.pi, np.pi, 3), rng.uniform(-np.pi, np.pi, 3)
        q0, q1 = np.zeros(4), np.zeros(4)
        plannersim.pl_quat_from_euler(_p(e0), ax, _p(q0))
        plannersim.pl_quat_from_euler(_p(e1), ax, _p(q1))
        assert np.abs(q0 - path_oracle.quat_from_euler(e0, axes)).max() <= 1e-15
        f = float(rng.choice([0.0, 1.0, rng.uniform()]))
        qs, e = np.zeros(4), np.zeros(3)
        plannersim.pl_slerp(_p(q0), _p(q1), f, _p(qs))
        assert np.abs(qs - path_oracle.slerp(q0, q1, np.array([f]))[0]).max() <= 1e-14
        plannersim.pl_euler_from_quat(_p(qs), ax, _p(e))
        assert np.abs(e - path_oracle.euler_from_quat(qs[None], axes)[0]).max() <= 1e-13


@pytest.mark.parametrize("kind", ["Gaussian", "Linear"])
def test_shim_ramps_equal_generate(plannersim, kind):
    vp = getattr(velocity_profiles, kind)(dt=0.001, acceleration=3.0)
    p = params(kind, dict(dt=0.001, acceleration=3.0), 10, "rxyz")
    for va, vb in ((0.0, 1.0), (0.2, 0.7)):
        ref = vp.generate(va, vb)
        got = np.zeros(len(ref))
        plannersim.pl_ramp(C.byref(p), va, vb, len(ref), _p(got))
        assert np.abs(got - ref).max() <= 1e-14


def test_shim_rejects_rows_the_reference_cannot_plan(plannersim):
    table = PathPlanner(position_profiles.Linear(), velocity_profiles.Gaussian(0.001, 1)).table
    p = params("Gaussian", dict(dt=0.001, acceleration=1.0), len(table), "rxyz")
    z = np.zeros(3)
    cases = [(z, z, 1.0, 0.0, 0.0, -1),                            # zero distance
             (z, -np.ones(3), 1.0, 0.0, 0.0, -2),                   # exactly opposite to (1, 1, 1)
             (z, np.ones(3), 0.0, 0.0, 0.0, -3),                    # no velocity to search from
             (z, np.full(3, 1e-3), 1.0, 0.0, 0.0, -4),              # the search shrinks the ramps below two samples
             (z, np.ones(3), 1.0, 0.9995, 0.0, -4),                 # a one-sample ramp
             (z, np.ones(3), 1e9, 0.0, 0.0, -5)]                    # a ramp of 1e12 steps
    for start, target, vm, v0, v1, want in cases:
        S, _ = shim_path(plannersim, p, table, start, target, vm, v0, v1)
        assert S == want, (target, S)
        r = path_oracle.plan(table, start, target, vm, v0, v1, "gaussian", 0.001, 1.0)
        assert r["lengths"][0] == want


# ---------------------------------------------------------------------------------------------- C ABI
def test_path_struct_layouts_match_the_header(tmp_path):
    prog = r"""
#include <stdio.h>
#include <stddef.h>
#include "abrb.h"
int main(void){
  printf("%zu %zu %zu %zu %zu\n", sizeof(abrb_path_params), offsetof(abrb_path_params, dt),
         offsetof(abrb_path_params, axes), sizeof(abrb_path_rec), offsetof(abrb_path_rec, flags));
  return 0; }
"""
    src, exe = tmp_path / "t.c", tmp_path / "t"
    src.write_text(prog)
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    got = [int(v) for v in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split()]
    assert got == [C.sizeof(_abi.PathParams), _abi.PathParams.dt.offset, _abi.PathParams.axes.offset,
                   C.sizeof(_abi.PathRec), _abi.PathRec.flags.offset]


def _has_device():
    return _lib.lib().abrb_device_count() > 0


def test_path_argument_checks():
    L = _lib.lib()
    EINVAL, EUNSUP, ECUDA = _abi.EINVAL, -4, -5
    buf = (C.c_double * 64)()
    ptr = C.cast(buf, C.c_void_p).value
    mis = ptr + 4
    good = params("Gaussian", dict(dt=0.001, acceleration=1.0), 10, "rxyz")

    def plan(p=good, table=ptr, start=ptr, target=ptr, vm=ptr, v0=ptr, v1=ptr, lengths=ptr, rec=ptr, B=1):
        return L.abrb_path_plan(None if p is None else C.byref(p), table, start, target, vm, v0, v1, lengths, rec, B,
                                None)

    def fill(f32=False, p=good, table=ptr, start=ptr, target=ptr, v0=ptr, v1=ptr, so=None, to=None, rec=ptr,
             lengths=ptr, s_max=5, path=ptr, B=1):
        fn = L.abrb_path_fill_f32 if f32 else L.abrb_path_fill_f64
        return fn(None if p is None else C.byref(p), table, start, target, v0, v1, so, to, rec, lengths, s_max, path,
                  B, None)

    def with_(**kw):
        p = params("Gaussian", dict(dt=0.001, acceleration=1.0), 10, "rxyz")
        for k, v in kw.items():
            if k == "axes":
                for j, a in enumerate(v):
                    p.axes[j] = a
            else:
                setattr(p, k, v)
        return p

    for call in (plan, fill):
        assert call(p=None) == EINVAL
        assert call(B=-1) == EINVAL
        assert call(p=with_(vel_kind=2)) == EUNSUP
        assert call(p=with_(n_points=1)) == EINVAL
        assert call(p=with_(n_points=_abi.PATH_MAX_POINTS + 1)) == EUNSUP
        assert b"shared memory" in L.abrb_last_error()
        assert call(p=with_(axes=(3, 0, 0, 0))) == EUNSUP
        assert call(p=with_(axes=(0, 2, 0, 0))) == EUNSUP
        for bad in (dict(dt=0.0), dict(acceleration=-1.0), dict(n_sigma=float("nan")), dict(dt=float("inf"))):
            assert call(p=with_(**bad)) == EINVAL, bad
        assert call(p=with_(vel_kind=1, n_sigma=0.0)) != EINVAL  # n_sigma only matters to the Gaussian
        for arg in ("table", "start", "target", "v0", "v1"):
            assert call(**{arg: None}) == EINVAL, arg
            assert call(**{arg: mis}) == EINVAL, arg
        assert call(B=0) == 0
    for arg in ("vm", "lengths", "rec"):
        assert plan(**{arg: None}) == EINVAL, arg
        assert plan(**{arg: mis}) == EINVAL, arg
    for f32 in (False, True):
        assert fill(f32, s_max=-1) == EINVAL
        assert fill(f32, s_max=(1 << 30) + 1) == EINVAL
        assert fill(f32, so=ptr) == EINVAL and fill(f32, to=ptr) == EINVAL
        assert fill(f32, s_max=0) == 0
        for arg in ("rec", "lengths", "path"):
            assert fill(f32, **{arg: None}) == EINVAL, arg
            assert fill(f32, **{arg: mis + (2 if f32 and arg == "path" else 0)}) == EINVAL, arg
        assert fill(f32, so=mis, to=ptr) == EINVAL
    if not _has_device():
        assert plan() == ECUDA
        assert fill(False) == ECUDA and fill(True, so=ptr, to=ptr) == ECUDA
        assert b"no CUDA device" in L.abrb_last_error()


# ---------------------------------------------------------------------------------------------- Python rejections
def test_python_rejections():
    planner = PathPlanner(position_profiles.Linear(), velocity_profiles.Gaussian(0.001, 1.0))
    with pytest.raises(AssertionError, match="start velocity"):
        planner.generate_path(np.zeros(3), np.ones(3), 1.0, start_velocity=1.5)
    with pytest.raises(AssertionError, match="target velocity .* in row 1"):
        planner.generate_path(np.zeros((2, 3)), np.ones((2, 3)), [1.0, 0.5], target_velocity=[0.2, 0.6])
    with pytest.raises(NotImplementedError, match="target orientation"):
        planner.generate_path(np.zeros(3), np.ones(3), 1.0, start_orientation=np.zeros(3))

    class MyRamp(velocity_profiles.VelProf):
        def generate(self, start_velocity, target_velocity):
            return np.linspace(start_velocity, target_velocity, 10)

    with pytest.raises(TypeError):
        PathPlanner(position_profiles.Linear(), MyRamp(0.001))
    with pytest.raises(ValueError, match="axes"):
        PathPlanner(position_profiles.Linear(), velocity_profiles.Linear(0.001, 1.0), axes="xyz")


# ---------------------------------------------------------------------------------------------- GPU
gpu = pytest.mark.gpu


@gpu
@pytest.mark.parametrize("i", CASES)
def test_gpu_golden_single_path(i):
    g, kw = case_inputs(i)
    planner = PathPlanner(*make_profiles(i), axes=META[i]["axes"])
    path = planner.generate_path(g["start"], g["target"], **kw)
    assert isinstance(path, np.ndarray) and path.dtype == np.float64
    assert path.shape == g["path"].shape and planner.n_timesteps == len(g["path"])
    assert rel_err(path, g["path"]) <= 1e-10
    assert np.array_equal(planner.next(), path[0]) and np.array_equal(planner.next_at_n(10 ** 6), path[-1])
    p32 = planner.generate_path(g["start"].astype(np.float32), g["target"], **kw)
    assert p32.dtype == np.float32 and p32.shape == g["path"].shape
    assert rel_err(p32.astype(np.float64), g["path"]) <= 1e-5


@gpu
def test_gpu_golden_batched_and_padding():
    import torch

    by_planner = {}
    for i in CASES:
        key = json.dumps([META[i]["pos"], META[i]["vel"], META[i]["axes"], META[i]["orient"]])
        by_planner.setdefault(key, []).append(i)
    for idx in by_planner.values():
        i0 = idx[0]
        planner = PathPlanner(*make_profiles(i0), axes=META[i0]["axes"])
        gs = [case_inputs(i) for i in idx]
        start = torch.tensor(np.stack([g["start"] for g, _ in gs]), device="cuda")
        target = torch.tensor(np.stack([g["target"] for g, _ in gs]), device="cuda")
        kw = {k: torch.tensor([kw_[k] for _, kw_ in gs], device="cuda", dtype=torch.float64)
              for k in ("max_velocity", "start_velocity", "target_velocity")}
        if META[i0]["orient"]:
            kw["start_orientation"] = torch.tensor(np.stack([g["so"] for g, _ in gs]), device="cuda")
            kw["target_orientation"] = torch.tensor(np.stack([g["to"] for g, _ in gs]), device="cuda")
        path = planner.generate_path(start, target, **kw)
        assert path.is_cuda and path.shape[0] == len(idx)
        lengths = planner.lengths.cpu().numpy()
        got = path.cpu().numpy()
        for b, (g, _) in enumerate(gs):
            S = len(g["path"])
            assert lengths[b] == S
            assert rel_err(got[b, :S], g["path"]) <= 1e-10
            assert np.array_equal(got[b, S:], np.broadcast_to(got[b, S - 1], got[b, S:].shape))
        p32 = planner.generate_path(start.float(), target, **kw)
        assert p32.dtype == torch.float32 and np.array_equal(planner.lengths.cpu().numpy(), lengths)


def random_reaches(B, seed):
    rng = np.random.default_rng(seed)
    start = rng.uniform(-0.4, 0.4, (B, 3)) + np.array([0.0, 0.4, 0.5])
    target = rng.uniform(-0.4, 0.4, (B, 3)) + np.array([0.0, 0.4, 0.5])
    vm = rng.uniform(0.3, 1.5, B)
    v0 = np.where(rng.uniform(size=B) < 0.2, vm, rng.uniform(0, 0.5, B) * vm)
    v1 = np.where(rng.uniform(size=B) < 0.5, 0.0, rng.uniform(0, 0.5, B) * vm)
    so, to = rng.uniform(-np.pi, np.pi, (B, 3)), rng.uniform(-np.pi, np.pi, (B, 3))
    return start, target, vm, v0, v1, so, to


@gpu
@pytest.mark.parametrize("vel", ["Gaussian", "Linear"])
def test_gpu_random_reaches_against_oracle(vel):
    import torch

    B = 4096
    vp = getattr(velocity_profiles, vel)(dt=0.002, acceleration=3.0)
    planner = PathPlanner(position_profiles.SinCurve(axes=["x", "z"], n_sample_points=400), vp, axes="rxyz")
    # the first 4 096 of a larger draw that the reference can plan (short reaches with a high start velocity cannot be)
    rows = random_reaches(5000, 11 if vel == "Gaussian" else 12)
    r = path_oracle.plan(planner.table, *rows[:5], vel.lower(), 0.002, 3.0, 3, "rxyz", *rows[5:])
    keep = np.nonzero(r["lengths"] >= 2)[0][:B]
    assert len(keep) == B
    start, target, vm, v0, v1, so, to = (a[keep] for a in rows)
    r = dict(lengths=r["lengths"][keep], near_integer=r["near_integer"][keep], paths=[r["paths"][b] for b in keep])
    t = lambda a: torch.tensor(a, device="cuda")  # noqa: E731
    path = planner.generate_path(t(start), t(target), t(vm), start_orientation=t(so), target_orientation=t(to),
                                 start_velocity=t(v0), target_velocity=t(v1)).cpu().numpy()
    lengths = planner.lengths.cpu().numpy()
    flagged = r["near_integer"]
    print(f"{vel}: {int(flagged.sum())} of {B} rows flagged near-integer")
    assert np.array_equal(lengths[~flagged], r["lengths"][~flagged])
    assert np.all(np.abs(lengths[flagged] - r["lengths"][flagged]) <= 1)
    worst_pos, worst_ang = 0.0, 0.0
    for b in np.nonzero(lengths == r["lengths"])[0]:
        ref, got = r["paths"][b], path[b, : lengths[b]]
        worst_pos = max(worst_pos, rel_err(got[:, :9], ref[:, :9]))
        worst_ang = max(worst_ang, rel_err(got[:, 9:], ref[:, 9:]))
    print(f"{vel}: worst relative error {worst_pos:.2e} (x, dx, angles), {worst_ang:.2e} (angular velocity)")
    assert worst_pos <= 1e-10 and worst_ang <= 1e-8


@gpu
def test_gpu_batched_rows_equal_single_calls():
    import torch

    start, target, vm, v0, v1, so, to = random_reaches(64, 5)
    planner = PathPlanner(position_profiles.Ellipse(0.4, n_sample_points=500), velocity_profiles.Gaussian(0.002, 4.0))
    t = lambda a: torch.tensor(a, device="cuda")  # noqa: E731
    batch = planner.generate_path(t(start), t(target), t(vm), start_orientation=t(so), target_orientation=t(to),
                                  start_velocity=t(v0), target_velocity=t(v1)).cpu().numpy()
    lengths = planner.lengths.cpu().numpy()
    for b in range(0, 64, 7):
        single = planner.generate_path(start[b], target[b], vm[b], start_orientation=so[b], target_orientation=to[b],
                                       start_velocity=v0[b], target_velocity=v1[b])
        assert len(single) == lengths[b]
        assert np.array_equal(single, batch[b, : lengths[b]])
        assert np.array_equal(batch[b, lengths[b]:], np.broadcast_to(single[-1], batch[b, lengths[b]:].shape))


@gpu
def test_gpu_degenerate_rows_raise():
    planner = PathPlanner(position_profiles.Linear(), velocity_profiles.Gaussian(0.001, 1.0))
    start = np.zeros((3, 3))
    target = np.array([[0.3, 0.2, 0.1], [0.0, 0.0, 0.0], [0.5, 0.1, 0.2]])
    with pytest.raises(ValueError, match="row 1: start and target coincide"):
        planner.generate_path(start, target, 1.0)
    with pytest.raises(ValueError, match="opposite"):
        planner.generate_path(np.zeros(3), -np.ones(3), 1.0)
    with pytest.raises(ValueError, match="reached 0"):
        planner.generate_path(np.zeros(3), np.ones(3), 0.0)
    with pytest.raises(ValueError, match="fewer than two samples"):
        planner.generate_path(np.zeros(3), np.full(3, 1e-3), 1.0)


@gpu
def test_gpu_planner_feeds_osc_rollout_path():
    import torch

    from abr_control_b200.arms import ur5
    from abr_control_b200.controllers import OSC

    B = 512
    rng = np.random.default_rng(3)
    rc = ur5.Config()
    q0 = rng.uniform(-0.1, 0.1, (B, 6)) + np.array([0.0, -1.2, 1.6, -0.4, 1.57, 0.0])
    x0 = rc.Tx("EE", torch.tensor(q0, device="cuda")).cpu().numpy()
    target = x0 + rng.uniform(-0.08, 0.08, (B, 3))
    so = np.zeros((B, 3))
    to = rng.uniform(-0.3, 0.3, (B, 3))
    planner = PathPlanner(position_profiles.Linear(), velocity_profiles.Gaussian(dt=0.002, acceleration=3.0))
    t = lambda a: torch.tensor(a, device="cuda")  # noqa: E731
    P = planner.generate_path(t(x0), t(target), 0.5, start_orientation=t(so), target_orientation=t(to))
    r = path_oracle.plan(planner.table, x0, target, 0.5, 0.0, 0.0, "gaussian", 0.002, 3.0, 3, "rxyz", so, to)
    assert np.array_equal(planner.lengths.cpu().numpy(), r["lengths"])
    ref = torch.tensor(path_oracle.padded(r["paths"], r["lengths"]), device="cuda")
    osc = OSC(rc, kp=50, ko=50, ctrlr_dof=[True] * 6)
    dq0 = torch.zeros((B, 6), dtype=torch.float64, device="cuda")
    out = []
    for path in (P, ref):
        tm = path.permute(1, 0, 2).contiguous()  # (S, B, 12)
        pos, vel = torch.cat([tm[..., :3], tm[..., 6:9]], -1), torch.cat([tm[..., 3:6], tm[..., 9:12]], -1)
        out.append(osc.rollout_path(torch.tensor(q0, device="cuda"), dq0, pos, dt=0.002, path_velocity=vel,
                                    record=("x",)))
    (qa, _, ta, ca), (qb, _, tb, cb) = out
    assert torch.isfinite(cb).all()
    print(f"pipeline: {B} reaches of {planner.n_timesteps} steps, median cost {cb.median().item():.3e}")
    rel = (torch.abs(ca - cb) / torch.clamp(torch.abs(cb), min=1e-12)).max().item()
    assert rel < 1e-8, rel
    assert torch.abs(qa - qb).max().item() < 1e-8
    assert torch.abs(ta["x"] - tb["x"]).max().item() < 1e-8
