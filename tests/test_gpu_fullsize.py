"""The benchmarked OSC path at full size against an fp64 CPU reference.

bench.py times UR5 6-DOF `OSC.generate` with use_C, fp64, 65 536 states per launch through `generate_into`; that call
runs the plain instantiation of the fused kernel (`osc_kernel<..., PLAIN=true>`, chosen by `osc_plain` in abrb_host.hpp).
This module checks that path where the small oracle tests cannot reach: at the full batch size, where the persistent
CTAs take several tiles each and flush their deferred pseudo-inverse queues mid-loop; in fp32; through the chunked host
pipeline and its two asynchronous slots; in dependent back-to-back launches; and in the plain rollout kernel.

The reference is built once per module from exactly the states bench.py times first (`bench.synth(65536, 6, 0)`):
J, M, g, C, Tx and R from `oracle.rbd_oracle.ChainOracle` (batched NumPy), the OSC arithmetic from the C restatement
`oracle/c/osc_cpu.c`.  `test_reference_builder_vs_numpy_oracle` pins that pair to `osc_oracle.run_case`.  Results do
not depend on a state's position in the batch, so the larger batches are tilings / permutations of the 65 536 states and
their references are the same permutations of the reference.

Error measure: rel err = max|du| / max|u_ref| per state.  Per-state flags of the reference:
  pinv       |det S| < 1e-3, S = J M^-1 J^T: the reference's truncating pseudo-inverse route (osc.py:143-145);
  ambiguous  an eigenvalue of S within 0.1 % of the cut-off 1e-4 * lambda_max: rounding decides whether it is truncated,
             and u jumps with that decision;
  cond       cond(S);
  wflip      |w| < 1e-5 for the orientation-error quaternion (orientation algorithm 0): u contains sign(w), so it jumps
             where w crosses zero, and fp32 rounding of w is about that large.
"""
import ctypes as C
import os
import subprocess
import types

import numpy as np
import pytest

import bench
from oracle import rbd_oracle as ro

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
B0 = bench.B_PER_GPU  # 65 536
BIG = 4 * B0          # 262 144: ~8 tiles per fp64 CTA, enough tiles for 4 fp32 CTAs per SM
TILE = 128            # states per CTA tile (kBlock)


def _report(name, **vals):
    """one line per check with the observed figures (visible with pytest -s)"""
    print(f"[fullsize] {name}: " + ", ".join(f"{k}={v:.3e}" if isinstance(v, float) else f"{k}={v}" for k, v in vals.items()))


# ---------------------------------------------------------------------------------------------- CPU reference
@pytest.fixture(scope="session")
def oracle_c(tmp_path_factory):
    """oracle/c/liboracle_c.so as build() left it, or, when it is missing or older than its source, a fresh compile
    in a temporary directory (the tree is never written)."""
    src = os.path.join(ROOT, "oracle", "c", "osc_cpu.c")
    so = os.path.join(ROOT, "oracle", "c", "liboracle_c.so")
    if not os.path.exists(so) or os.path.getmtime(so) < os.path.getmtime(src):
        so = str(tmp_path_factory.mktemp("oracle_c") / "liboracle_c.so")
        subprocess.run(["gcc", "-O2", "-fPIC", "-shared", "-o", so, src, "-lm"], check=True)
    lib = C.CDLL(so)
    lib.osc_from_quantities_batch.restype = None
    lib.osc_from_quantities_batch.argtypes = [C.c_void_p, C.c_long] + [C.c_void_p] * 12
    return lib


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def reference(lib, q, dq, tg, chunk=4096):
    """ChainOracle + C OSC for bench.OSC_KW on (B, 6) fp64 states -> namespace of J, M, g, C, Tx, R, u, tr and flags"""
    ch = ro.ChainOracle("ur5")
    B = len(q)
    parts = {k: [] for k in ("J", "M", "g", "C", "Tx", "R")}
    for b0 in range(0, B, chunk):  # chunks bound the memory of the second-order chain walk behind C
        qc, dqc = q[b0:b0 + chunk], dq[b0:b0 + chunk]
        parts["J"].append(ch.J("EE", qc))
        parts["M"].append(ch.M(qc))
        parts["g"].append(ch.g(qc))
        parts["C"].append(ch.C(qc, dqc))
        parts["Tx"].append(ch.Tx("EE", qc))
        parts["R"].append(ch.R("EE", qc))
    r = types.SimpleNamespace(**{k: np.ascontiguousarray(np.concatenate(v)) for k, v in parts.items()})
    q, dq, tg = (np.ascontiguousarray(a, dtype=np.float64) for a in (q, dq, tg))
    r.u, r.tr = np.empty((B, 6)), np.empty((B, 6))
    cfg = bench.osc_cfg()
    lib.osc_from_quantities_batch(C.byref(cfg), B, _p(r.J), _p(r.M), _p(r.g), _p(r.C), _p(r.Tx), _p(r.R), _p(q), _p(dq),
                                  _p(tg), None, _p(r.u), _p(r.tr))
    S = r.J @ np.linalg.inv(r.M) @ np.swapaxes(r.J, 1, 2)
    r.pinv = np.abs(np.linalg.det(S)) < 1e-3
    w = np.linalg.eigvalsh(S)
    r.amb = np.any(np.abs(w / (1e-4 * w[:, -1:]) - 1) <= 1e-3, axis=1)
    r.cond = np.linalg.cond(S)
    qw = np.empty(B)
    for i in range(B):
        want = ro.unit_vector(ro.quaternion_from_euler_rxyz(*tg[i, 3:]))
        have = ro.unit_vector(ro.quaternion_from_matrix(r.R[i]))
        qw[i] = ro.quaternion_multiply(want, ro.quaternion_conjugate(have))[0]
    r.wflip = np.abs(qw) < 1e-5
    return r


@pytest.fixture(scope="module")
def ref(oracle_c):
    """the reference of bench.py's first timed buffer set (rank 0, set 0), byte for byte the same inputs"""
    q, dq, tg = bench.synth(B0, 6, 0)
    r = reference(oracle_c, q, dq, tg)
    r.q, r.dq, r.tg = q, dq, tg
    assert 2000 < r.pinv.sum() < 3000  # ~3.8 % of uniformly random UR5 states take the pseudo-inverse route
    _report("reference", pinv=int(r.pinv.sum()), ambiguous=int(r.amb.sum()), wflip=int(r.wflip.sum()),
            cond_gt_1e4=int((r.cond > 1e4).sum()))
    return r


def _tiling(seed, copies=4):
    """indices into the 65 536 reference states: `copies` independent permutations of them, concatenated"""
    rng = np.random.default_rng(seed)
    return np.concatenate([rng.permutation(B0) for _ in range(copies)])


def _rel(u, u_ref):
    u = np.asarray(u.cpu() if hasattr(u, "cpu") else u, dtype=np.float64)
    return np.abs(u - u_ref).max(axis=1) / np.abs(u_ref).max(axis=1)


def _check_f64(name, u, u_ref, r, idx):
    """fp64 bounds: <1e-9 on regular well-conditioned states, <1e-6 on every unambiguous state, median <1e-12"""
    u = np.asarray(u.cpu() if hasattr(u, "cpu") else u)
    assert np.isfinite(u).all(), name
    err = _rel(u, u_ref)
    well = (r.cond[idx] <= 1e4) & ~r.pinv[idx]
    clear = ~r.amb[idx]
    _report(name, max_well=err[well].max(), max_clear=err[clear].max(), median=float(np.median(err)),
            max_pinv_clear=err[r.pinv[idx] & clear].max() if (r.pinv[idx] & clear).any() else 0.0)
    assert err[well].max() < 1e-9, (name, err[well].max())
    assert err[clear].max() < 1e-6, (name, err[clear].max(), int(np.argmax(np.where(clear, err, 0))))
    assert np.median(err) < 1e-12, (name, np.median(err))


def _check_f32(name, u, u_ref, r, idx):
    """fp32 kernel vs the fp64 reference: median <2e-5, p99 <5e-3 on unambiguous states, <1e-3 on regular
    well-conditioned states; states at a sign(w) flip are excluded from the last two (fp32 rounding of w decides)"""
    u = np.asarray(u.cpu() if hasattr(u, "cpu") else u)
    assert np.isfinite(u).all(), name
    err = _rel(u, u_ref)
    steady = ~r.wflip[idx]
    clear = ~r.amb[idx] & steady
    well = (r.cond[idx] <= 1e4) & ~r.pinv[idx] & steady
    _report(name, median=float(np.median(err)), p99_clear=float(np.quantile(err[clear], 0.99)), max_well=err[well].max())
    assert np.median(err) < 2e-5, (name, np.median(err))
    assert np.quantile(err[clear], 0.99) < 5e-3, (name, np.quantile(err[clear], 0.99))
    assert err[well].max() < 1e-3, (name, err[well].max())
    return err


def _dev(*arrays, dtype=None):
    import torch

    return tuple(torch.as_tensor(np.ascontiguousarray(a if dtype is None else a.astype(dtype)), device="cuda")
                 for a in arrays)


def _ctrl(dtype=np.float64, general=None):
    """bench's controller; general="null" adds Damping(kv=0) (a secondary controller whose term is +-0), which moves
    the call onto the general instantiation without changing the arithmetic"""
    from abr_control_b200.arms import ur5
    from abr_control_b200.controllers import OSC, Damping

    rc = ur5.Config(dtype=dtype)
    nulls = [Damping(rc, kv=0)] if general == "null" else None
    return OSC(rc, null_controllers=nulls, **bench.OSC_KW)


# ---------------------------------------------------------------------------------------------- 1. the reference itself
def test_reference_builder_vs_numpy_oracle(oracle_c):
    """ChainOracle + C OSC against the per-state NumPy oracle (osc_oracle.run_case) on every pseudo-inverse state of
    an 8 192-state batch of the bench distribution and 100 others: u and training signal to 1e-10."""
    from oracle import osc_oracle

    q, dq, tg = bench.synth(8192, 6, 1)
    r = reference(oracle_c, q, dq, tg)
    slow = np.where(r.pinv)[0]
    assert 200 < len(slow) < 450
    pick = np.concatenate([slow, np.where(~r.pinv)[0][::80][:100]])
    u, tr = osc_oracle.run_case(dict(arm="ur5", osc=bench.OSC_KW), q[pick], dq[pick], tg[pick])
    eu = _rel(r.u[pick], u)
    et = _rel(r.tr[pick], tr)
    _report("reference builder", states=len(pick), max_u=eu.max(), max_train=et.max())
    assert eu.max() < 1e-10 and et.max() < 1e-10, (eu.max(), et.max())


# ---------------------------------------------------------------------------------------------- 2. headline
@pytest.mark.gpu
def test_headline_generate_into_fp64(ref):
    """bench.py's timed call (generate_into, B = 65 536, fp64) over the whole batch; the training signal via generate."""
    import torch

    sms = torch.cuda.get_device_properties(0).multi_processor_count
    assert -(-B0 // TILE) > 2 * sms  # more tiles than resident fp64 CTAs: the tile counter hands out further tiles
    ctrlr = _ctrl()
    q, dq, tg = _dev(ref.q, ref.dq, ref.tg)
    u = torch.empty_like(q)
    ctrlr.generate_into(q, dq, tg, u)
    torch.cuda.synchronize()
    idx = np.arange(B0)
    _check_f64("headline u", u, ref.u, ref, idx)
    u2 = ctrlr.generate(q, dq, tg)
    _check_f64("headline u (generate)", u2, ref.u, ref, idx)
    _check_f64("headline training signal", ctrlr.training_signal, ref.tr, ref, idx)


@pytest.mark.gpu
def test_headline_vs_reference_generated_c(ref):
    """The headline u against the reference's own generated C (oracle/_ref, built only where the reference is
    available) on all 65 536 states."""
    import torch

    lib = bench.ref_lib()
    if lib is None:
        pytest.skip("oracle/_ref/libabrref_ur5.so was not built")
    u_ref = np.empty((B0, 6))
    lib.ref_ur5_osc_batch(C.byref(bench.osc_cfg()), _p(ref.q), _p(ref.dq), _p(ref.tg), C.c_long(B0), _p(u_ref),
                          C.c_int(max(1, min(8, os.cpu_count() or 1))))
    q, dq, tg = _dev(ref.q, ref.dq, ref.tg)
    u = torch.empty_like(q)
    _ctrl().generate_into(q, dq, tg, u)
    _check_f64("headline vs reference generated C", u, u_ref, ref, np.arange(B0))


# ---------------------------------------------------------------------------------------------- 3. multi-tile
@pytest.mark.gpu
def test_multi_tile_scheduling_fp64(ref):
    """B = 262 144 (four permutations of the set): ~8 tiles per CTA, so the deferred queues are flushed mid-loop as well
    as after the last tile.  Then one 65 536 batch with every pseudo-inverse state in one contiguous block: ~19 tiles
    whose every lane is deferred, so the CTA queue (32 records) overflows and the rest take the in-line route."""
    import torch

    ctrlr = _ctrl()
    idx = _tiling(3)
    q, dq, tg = _dev(ref.q[idx], ref.dq[idx], ref.tg[idx])
    u = torch.empty_like(q)
    ctrlr.generate_into(q, dq, tg, u)
    ctrlr.generate(q, dq, tg)
    _check_f64("262144 tiling u", u, ref.u[idx], ref, idx)
    _check_f64("262144 tiling training signal", ctrlr.training_signal, ref.tr[idx], ref, idx)

    slow, rest = np.where(ref.pinv)[0], np.where(~ref.pinv)[0]
    cut = 200 * TILE  # the block starts on a tile boundary and spans the first and the later tile rounds
    idx = np.concatenate([rest[:cut], slow, rest[cut:]])
    q, dq, tg = _dev(ref.q[idx], ref.dq[idx], ref.tg[idx])
    u = torch.empty_like(q)
    ctrlr.generate_into(q, dq, tg, u)
    _check_f64("contiguous pinv block u", u, ref.u[idx], ref, idx)


# ---------------------------------------------------------------------------------------------- 4. fp32
@pytest.mark.gpu
def test_plain_fp32_full_size(ref):
    """The fp32 plain kernel on B = 262 144 (fp64 states cast to fp32) against the fp64 reference."""
    import torch

    idx = _tiling(4)
    q, dq, tg = _dev(ref.q[idx], ref.dq[idx], ref.tg[idx], dtype=np.float32)
    u = torch.empty_like(q)
    _ctrl(np.float32).generate_into(q, dq, tg, u)
    _check_f32("fp32 262144 u", u, ref.u[idx], ref, idx)


# ---------------------------------------------------------------------------------------------- 5. plain vs general
@pytest.mark.gpu
def test_plain_vs_general_instantiation(ref):
    """The general instantiation on the same maths, reached two ways: a Damping(kv=0) secondary controller (its term is
    +-0) and a broadcast all-zero target velocity (the kernel then takes the reference's tv == 0 branch, osc.py:275)."""
    import torch

    idx = np.arange(B0)
    well = ~ref.pinv & (ref.cond <= 1e4)
    slow = ref.pinv & ~ref.amb
    for dtype in (np.float64, np.float32):
        q, dq, tg = _dev(ref.q, ref.dq, ref.tg, dtype=dtype)
        u_plain = torch.empty_like(q)
        _ctrl(dtype).generate_into(q, dq, tg, u_plain)
        u_null = torch.empty_like(q)
        _ctrl(dtype, "null").generate_into(q, dq, tg, u_null)
        u_tv = torch.empty_like(q)
        _ctrl(dtype).generate_into(q, dq, tg, u_tv, target_velocity=torch.zeros(6, dtype=q.dtype, device="cuda"))
        up = u_plain.double().cpu().numpy()
        for how, ug in (("null", u_null), ("tv", u_tv)):
            ug = ug.double().cpu().numpy()
            d = _rel(ug, up)
            if dtype == np.float64:
                _report(f"plain vs general ({how}) f64", max_well=d[well].max(), max_pinv_clear=d[slow].max())
                assert d[well].max() < 1e-12 and d[slow].max() < 1e-9, (how, d[well].max(), d[slow].max())
            else:
                _check_f32(f"general ({how}) f32 u", ug, ref.u, ref, idx)
                _report(f"plain vs general ({how}) f32", median=float(np.median(d)))
                assert np.median(d) < 1e-6, (how, np.median(d))
        if dtype == np.float32:
            _check_f32("plain f32 65536 u", up, ref.u, ref, idx)


# ---------------------------------------------------------------------------------------------- 6. rigid-body quantities
@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_rigid_body_quantities_full_size(ref, dtype):
    """BASELINE config 2 (UR5 J, M, g, C, Tx) at 65 536 states and at the 262 144 tiling, where the grid-stride loop of
    rbd_kernel runs more than once (the grid is capped at 1 056 CTAs), with the golden tests' tolerances."""
    from abr_control_b200.arms import ur5

    rc = ur5.Config(dtype=dtype)
    rtol, atol = (1e-10, 1e-12) if dtype == np.float64 else (1e-4, 2e-5)
    for idx in (np.arange(B0), _tiling(6)):
        q, dq = _dev(ref.q[idx], ref.dq[idx], dtype=dtype)
        out = rc.eval(q, dq, want=("J", "M", "g", "C", "Tx"))
        for k, r_tol, a_tol in (("J", rtol, atol), ("Tx", rtol, atol),
                                ("M", rtol, atol * max(1.0, np.abs(ref.M).max())),
                                ("g", rtol, atol * 10 * max(1.0, np.abs(ref.g).max())),
                                ("C", rtol * 10, atol * 50 * max(1.0, np.abs(ref.C).max()))):
            got = out[k].double().cpu().numpy()
            want = getattr(ref, k)[idx]
            err = np.abs(got - want)
            _report(f"rbd {k} {np.dtype(dtype).name} B={len(idx)}", max_abs=err.max())
            assert np.all(err <= a_tol + r_tol * np.abs(want)), (k, len(idx), err.max())


# ---------------------------------------------------------------------------------------------- 7. host pipeline
def _same(name, got, want, pinv, tol):
    """host-pipeline result vs the device-tensor result on the same states: bit-identical on regular states; states on
    the pseudo-inverse route may take the in-line instead of the deferred route when the batch is cut differently (same
    arithmetic, other rounding; seen on an H100 with 896-state chunks and ki != 0, 1.6e-16)"""
    got = np.asarray(got, dtype=np.float64)
    want = np.asarray(want.cpu() if hasattr(want, "cpu") else want, dtype=np.float64)
    assert got.shape == want.shape, name
    assert np.array_equal(got[~pinv], want[~pinv]), (name, np.abs(got[~pinv] - want[~pinv]).max())
    d = _rel(got[pinv], want[pinv]) if pinv.any() else np.zeros(1)
    _report(name, pinv_max=d.max(), bit_identical=bool(np.array_equal(got, want)))
    assert d.max() < tol, (name, d.max())


def _pinned(*arrays):
    import torch

    return tuple(torch.as_tensor(np.ascontiguousarray(a)).pin_memory().numpy() for a in arrays)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_host_pipeline_chunks_lanes_and_streams(ref, dtype):
    """generate() on host arrays: the automatic chunk boundaries (49 152 and 196 608 states), 896-state chunks (ragged
    last chunk, many chunks per lane), one to three upload streams, a broadcast target, with and without the training
    signal, pinned and pageable inputs -- each against the device-tensor result on the same states."""
    tol = 1e-9 if dtype == np.float64 else 2e-5
    base = _tiling(7)
    qd, dqd, tgd = _dev(ref.q[base], ref.dq[base], ref.tg[base], dtype=dtype)
    dev_c = _ctrl(dtype)
    u_dev = dev_c.generate(qd, dqd, tgd).cpu().numpy()
    tr_dev = dev_c.training_signal.cpu().numpy()
    u_bc = dev_c.generate(qd, dqd, tgd[0]).cpu().numpy()  # one broadcast target row
    host_arr = lambda a: np.ascontiguousarray(a.astype(dtype))  # noqa: E731

    # every call starts at another offset of the set, so a row left unwritten still holds another state's result
    for k, B in enumerate((49151, 49152, 49153, 196608, 196609, BIG)):
        pos = np.roll(np.arange(BIG), -1000 * k)[:B]
        c = _ctrl(dtype)
        q, dq, tg = _pinned(*(host_arr(a[base][pos]) for a in (ref.q, ref.dq, ref.tg)))
        u = c.generate(q, dq, tg)
        _same(f"host {np.dtype(dtype).name} B={B} u", u, u_dev[pos], ref.pinv[base][pos], tol)
        _same(f"host {np.dtype(dtype).name} B={B} training signal", c.training_signal, tr_dev[pos], ref.pinv[base][pos], tol)

    B = 196609
    variants = (  # (what, execution options, how the call is made)
        ("chunk 896", dict(host_chunk_states=1000), {}),  # 1000 rounds down to whole tiles: 896
        ("1 upload stream", dict(host_upload_streams=1), {}),
        ("2 upload streams", dict(host_upload_streams=2), {}),
        ("3 upload streams", dict(host_upload_streams=3), {}),
        ("chunk 896, 3 streams, broadcast target", dict(host_chunk_states=1000, host_upload_streams=3), dict(bc=True)),
        ("broadcast target", {}, dict(bc=True)),
        ("no training signal", {}, dict(no_tr=True)),
        ("pageable inputs", {}, dict(pageable=True)),
        ("chunk 896, pageable, no training signal", dict(host_chunk_states=1000), dict(pageable=True, no_tr=True)),
    )
    for k, (what, opts, how) in enumerate(variants):
        pos = np.roll(np.arange(BIG), -777 * (k + 1))[:B]
        c = _ctrl(dtype)
        for name, v in opts.items():
            c.set_option(name, v)
        if how.get("no_tr"):
            c.record_training_signal = False
        arrays = [host_arr(a[base][pos]) for a in (ref.q, ref.dq)]
        arrays.append(host_arr(ref.tg[base][0]) if how.get("bc") else host_arr(ref.tg[base][pos]))
        if not how.get("pageable"):
            arrays = list(_pinned(*arrays))
        u = c.generate(*arrays)
        want = u_bc if how.get("bc") else u_dev
        _same(f"host {np.dtype(dtype).name} {what} u", u, want[pos], ref.pinv[base][pos], tol)
        if how.get("no_tr"):
            assert c.training_signal is None
        elif not how.get("bc"):
            _same(f"host {np.dtype(dtype).name} {what} training signal", c.training_signal, tr_dev[pos],
                  ref.pinv[base][pos], tol)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_host_pipeline_integrator_rows(ref, dtype):
    """ki != 0 over three consecutive host calls of 196 609 states (four chunks on two lanes, and 896-state chunks): the
    integrator rows go up and come back per chunk and must equal the device-tensor sequence's integrated_error_batch."""
    from abr_control_b200.arms import ur5
    from abr_control_b200.controllers import OSC

    tol = 1e-9 if dtype == np.float64 else 2e-5
    base = _tiling(8)
    B = 196609
    for chunk in (0, 1000):
        rc = ur5.Config(dtype=dtype)
        kw = dict(bench.OSC_KW, ki=0.2)
        dev_c, host_c = OSC(rc, **kw), OSC(rc, **kw)
        if chunk:
            host_c.set_option("host_chunk_states", chunk)
        for t in range(3):
            pos = np.roll(np.arange(BIG), -5000 * t)[:B]
            arrays = [np.ascontiguousarray(a[base][pos].astype(dtype)) for a in (ref.q, ref.dq, ref.tg)]
            u_dev = dev_c.generate(*_dev(*arrays)).cpu().numpy()
            u = host_c.generate(*_pinned(*arrays))
            _same(f"host ki {np.dtype(dtype).name} chunk={chunk} call {t} u", u, u_dev, ref.pinv[base][pos], tol)
            (ie_dev,) = dev_c.integrated_error_batch.values()
            (ie_host,) = host_c.integrated_error_batch.values()
            assert np.array_equal(ie_host, ie_dev.cpu().numpy()), (chunk, t)
            assert np.abs(ie_host).max() > 0


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_generate_async_slots(ref, dtype):
    """generate_async on slots 0 and 1 alternately, 8 calls over 4 distinct input sets: every wait() returns the u and
    the training signal of its own inputs (no slot or buffer aliasing)."""
    tol = 1e-9 if dtype == np.float64 else 2e-5
    c = _ctrl(dtype)
    sets, want = [], []
    for s in range(4):
        idx = np.random.default_rng(20 + s).permutation(B0)
        arrays = [np.ascontiguousarray(a[idx].astype(dtype)) for a in (ref.q, ref.dq, ref.tg)]
        u = c.generate(*_dev(*arrays)).cpu().numpy()
        want.append((u, c.training_signal.cpu().numpy(), ref.pinv[idx]))
        sets.append(_pinned(*arrays))
    pend = [None, None]

    def finish(p, s):
        u = p.wait()
        u_w, tr_w, pinv = want[s]
        _same(f"async {np.dtype(dtype).name} set {s} u", u, u_w, pinv, tol)
        _same(f"async {np.dtype(dtype).name} set {s} training signal", c.training_signal, tr_w, pinv, tol)

    for i in range(8):
        sl = i & 1
        if pend[sl] is not None:
            finish(*pend[sl])
        pend[sl] = (c.generate_async(*sets[i % 4], slot=sl), i % 4)
    for p in pend:
        finish(*p)


# ---------------------------------------------------------------------------------------------- 8. dependent launches
@pytest.mark.gpu
def test_dependent_back_to_back_launches(ref):
    """Three launches where each reads the previous one's output, with no host synchronisation in between (programmatic
    dependent launch lets each start during its predecessor's tail): u = OSC(q, dq); u2 = OSC(q, u); rbd(q=u2, dq=u).
    Same result as the chain with a synchronize after every launch.  Outputs are filled with NaN first, so a read that
    overtakes the producer shows."""
    import torch

    from abr_control_b200.arms import ur5

    ctrlr, rc = _ctrl(), ur5.Config()
    q, dq, tg = _dev(ref.q, ref.dq, ref.tg)
    A, A2 = torch.empty_like(q), torch.empty_like(q)
    out = dict(J=torch.empty((B0, 6, 6), dtype=q.dtype, device="cuda"), M=torch.empty((B0, 6, 6), dtype=q.dtype, device="cuda"),
               g=torch.empty_like(q), C=torch.empty((B0, 6, 6), dtype=q.dtype, device="cuda"),
               Tx=torch.empty((B0, 3), dtype=q.dtype, device="cuda"))

    def chain(sync):
        for t in [A, A2] + list(out.values()):
            t.fill_(float("nan"))
        torch.cuda.synchronize()
        ctrlr.generate_into(q, dq, tg, A)
        if sync:
            torch.cuda.synchronize()
        ctrlr.generate_into(q, A, tg, A2)
        if sync:
            torch.cuda.synchronize()
        rc.eval_into(A2, A, out)
        torch.cuda.synchronize()
        return {k: v.cpu().numpy() for k, v in dict(out, u=A, u2=A2).items()}

    chain(False)  # warm-up: workspace, tile counters, function attributes
    got, want = chain(False), chain(True)
    slow = ref.pinv
    for k in want:
        assert np.isfinite(got[k]).all() and np.isfinite(want[k]).all(), k
        a, b = got[k].reshape(B0, -1), want[k].reshape(B0, -1)
        # rows of states on the pseudo-inverse route may round differently from run to run (in-line or deferred,
        # depending on which CTA took which tile); everything derived from a regular state is bit-identical
        assert np.array_equal(a[~slow], b[~slow]), k
        d = np.abs(a[slow] - b[slow]).max(axis=1) / np.abs(b[slow]).max(axis=1)
        _report(f"dependent launches {k}", pinv_max=d.max(), bit_identical=bool(np.array_equal(a, b)))
        # u2 = OSC(q, u) is linear and quadratic in u: twice the relative spread of u, with margin
        assert d.max() < (1e-9 if k == "u" else 1e-8), (k, d.max())


# ---------------------------------------------------------------------------------------------- 9. plain rollout
@pytest.mark.gpu
def test_plain_rollout(oracle_c):
    """The plain rollout kernel: 140 000 trajectories x 8 steps (the grid-stride loop runs more than once), against the
    general rollout (Damping(kv=0)) on every trajectory and against a stepped batched reference (ChainOracle + C OSC +
    semi-implicit Euler, as test_rollout_vs_oracle_stepped_loop) on every 64th trajectory."""
    Bt, steps, dt = 140_000, 8, 1e-3
    q, dq, tg = bench.synth(Bt, 6, 9)
    dq = dq * 0.1
    qd, dqd, tgd = _dev(q, dq, tg)
    qf, dqf, traj = _ctrl().rollout(qd, dqd, tgd, steps=steps, dt=dt)
    qg, _, trg = _ctrl(general="null").rollout(qd, dqd, tgd, steps=steps, dt=dt, record=("q",))
    dqg = (traj["q"] - trg["q"]).abs().max().item()
    _report("rollout plain vs general", max_q=dqg)
    assert dqg < 1e-10 and (qf - qg).abs().max().item() < 1e-10
    pick = np.arange(0, Bt, 64)
    tq, tdq, tu = (traj[k][:, pick].cpu().numpy() for k in ("q", "dq", "u"))
    qs, dqs = q[pick].copy(), dq[pick].copy()
    alive = np.ones(len(pick), dtype=bool)
    worst = dict(u=0.0, q=0.0, dq=0.0)
    for t in range(steps):
        r = reference(oracle_c, qs, dqs, tg[pick])
        # once a step of a trajectory is ambiguous (or at a sign(w) flip), u may jump there: the two closed loops part
        alive &= ~(r.amb | r.wflip)
        ddq = np.linalg.solve(r.M, (r.u + r.g - np.einsum("bij,bj->bi", r.C, dqs))[..., None])[..., 0]
        dqs = dqs + ddq * dt
        qs = qs + dqs * dt
        eu = np.abs(tu[t] - r.u).max(axis=1) / np.maximum(1.0, np.abs(r.u).max(axis=1))
        eq, edq = np.abs(tq[t] - qs).max(axis=1), np.abs(tdq[t] - dqs).max(axis=1)
        worst = dict(u=max(worst["u"], eu[alive].max()), q=max(worst["q"], eq[alive].max()), dq=max(worst["dq"], edq[alive].max()))
        assert eu[alive].max() < 1e-6 and eq[alive].max() < 1e-8 and edq[alive].max() < 1e-6, (t, worst)
    _report("rollout vs stepped reference", trajectories=int(alive.sum()), **worst)
    assert alive.sum() > 0.95 * len(pick)
