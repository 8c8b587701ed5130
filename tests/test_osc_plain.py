"""CPU suite: the choice between the plain and the general OSC instantiation (osc_plain, abrb_host.hpp), the plain
instantiation against the oracle, and the plain instantiation against the general one on the calls that qualify.
The per-state code is instantiated by g++ through tests/hostsim/plainsim.cpp (TEST INFRASTRUCTURE, never loaded by the
package)."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import cases
from abr_control_b200 import _abi
from oracle import osc_oracle as oo

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def plainsim(tmp_path_factory):
    src = os.path.join(ROOT, "tests", "hostsim", "plainsim.cpp")
    so = str(tmp_path_factory.mktemp("plainsim") / "_plainsim.so")
    subprocess.run(["g++", "-O1", "-std=c++17", "-shared", "-fPIC", "-x", "c++", src, "-o", so], check=True)
    return C.CDLL(so)


def P(a):
    return a.ctypes.data_as(C.c_void_p) if a is not None else None


def plain(ps, n, osc, frame="EE", tv=False, ierr=False, null=()):
    p = _abi.osc_params(n, null=[_abi.null_params(k, n, **kw) for k, kw in null], **osc)
    return ps.ps_osc_plain(C.byref(p), n, ps.hs_frame_id(n, frame.encode()), int(tv), int(ierr)) == 1


def ps_osc(ps, arm, osc, q, dq, target, f32=0, general=0):
    cd = _abi.chain_desc_from_dict(_abi.load_arm_json(arm))
    n, B = cd.n_joints, len(q)
    p = _abi.osc_params(n, **osc)
    u, tr, acc = np.zeros((B, n)), np.zeros((B, n)), np.zeros((B, n))
    rc = ps.ps_osc(C.byref(cd), C.byref(p), f32, general, ps.hs_frame_id(n, b"EE"), None,
                   P(np.ascontiguousarray(q)), P(np.ascontiguousarray(dq)), P(np.ascontiguousarray(target)), None,
                   C.c_int64(B), P(u), P(tr), P(acc), None)
    assert rc == 0
    return u, tr, acc


def test_plain_predicate(plainsim):
    T, F = True, False
    full = dict(kp=10, ctrlr_dof=[T] * 6, use_C=True)
    assert plain(plainsim, 6, full)  # the headline: UR5 6-DOF, use_C
    assert plain(plainsim, 6, dict(kp=10, use_C=True))  # x, y, z (the 3-row kernel)
    assert plain(plainsim, 6, dict(full, vmax=[0.5, 1.0]))  # vmax, the orientation algorithm stay runtime
    assert plain(plainsim, 6, dict(full, orientation_algorithm=1))
    assert plain(plainsim, 3, dict(kp=10, use_C=True))
    assert not plain(plainsim, 6, dict(kp=10))  # use_C off
    assert not plain(plainsim, 6, dict(full, use_g=False))
    assert not plain(plainsim, 6, dict(full, ki=0.5), ierr=True)
    assert not plain(plainsim, 6, full, tv=True)
    assert not plain(plainsim, 6, full, frame="link4")
    assert not plain(plainsim, 6, full, frame="joint5")
    assert not plain(plainsim, 6, full, null=[("Damping", dict(kv=10))])
    for dof in ([T, T, T, T, T, F], [T, F, T, F, F, F], [T, T, F, F, F, F], [F, F, F, T, T, T], [T, T, T, F, T, F]):
        assert not plain(plainsim, 6, dict(full, ctrlr_dof=dof)), dof


PLAIN_CASES = {
    "ur5_6dof_C": ("ur5", dict(kp=50, ctrlr_dof=[True] * 6, use_C=True)),
    "ur5_xyz_C": ("ur5", dict(kp=10, use_C=True)),
    "ur5_6dof_C_vmax_alg1": ("ur5", dict(kp=10, ko=8, kv=4, ctrlr_dof=[True] * 6, vmax=[0.5, 1.0], use_C=True,
                                         orientation_algorithm=1)),
    "jaco2_6dof_C": ("jaco2", dict(kp=60, ctrlr_dof=[True] * 6, use_C=True)),
    "threejoint_xyz_C": ("threejoint", dict(kp=20, use_C=True)),
}


@pytest.mark.parametrize("name", list(PLAIN_CASES))
def test_plain_instantiation_vs_oracle(plainsim, name):
    arm, osc = PLAIN_CASES[name]
    n = _abi.chain_desc_from_dict(_abi.load_arm_json(arm)).n_joints
    assert plain(plainsim, n, osc)
    q, dq, target, _ = cases.states(arm, 32)
    ref, reft = oo.run_case(dict(arm=arm, osc=osc), q, dq, target, None, "fp64")
    u, tr, _ = ps_osc(plainsim, arm, osc, q, dq, target)
    scale = np.abs(ref).max(axis=1, keepdims=True)
    assert np.max(np.abs(u - ref) / scale) < 1e-9
    assert np.max(np.abs(tr - reft) / scale) < 1e-9


@pytest.mark.parametrize("name", list(PLAIN_CASES))
def test_plain_matches_general_bit_for_bit(plainsim, name):
    """The plain instantiation only folds branches a qualifying call does not take, so without FMA contraction (the
    host build) it computes u, the training signal and the rollout's ddq with the same operations as the general one.
    The random states include ones on the truncating pseudo-inverse route."""
    arm, osc = PLAIN_CASES[name]
    n = _abi.chain_desc_from_dict(_abi.load_arm_json(arm)).n_joints
    rng = np.random.default_rng(5)
    B = 256
    q, dq, target = rng.uniform(0, 2 * np.pi, (B, n)), rng.uniform(0, 5, (B, n)), rng.uniform(-1, 1, (B, 6))
    for f32 in (0, 1):
        a = ps_osc(plainsim, arm, osc, q, dq, target, f32=f32)
        b = ps_osc(plainsim, arm, osc, q, dq, target, f32=f32, general=1)
        for x, y in zip(a, b):
            assert np.array_equal(x, y)
