#!/usr/bin/env python
"""Times the batched path planner: 4 096 UR5-scale reaches with orientation (Gaussian ramps, dt = 1e-3, acceleration 1,
per-path max_velocity in [0.5, 1]), fp64 rows.  Reports the two launches and the lengths' readback separately (CUDA
events, medians over --iters calls), the whole generate_path call, and the NumPy oracle's host time per path.

    python tools/path_planner_bench.py [--batch 4096] [--iters 20]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    import torch

    from abr_control_b200 import _abi, _lib
    from abr_control_b200.controllers.path_planners import PathPlanner, position_profiles, velocity_profiles
    from oracle import path_oracle

    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=4096)
    ap.add_argument("--iters", type=int, default=20)
    a = ap.parse_args()
    B = a.batch
    rng = np.random.default_rng(0)
    start = rng.uniform(-0.3, 0.3, (B, 3)) + np.array([0.0, 0.4, 0.5])
    target = rng.uniform(-0.3, 0.3, (B, 3)) + np.array([0.0, 0.4, 0.5])
    vm = rng.uniform(0.5, 1.0, B)
    so, to = rng.uniform(-np.pi, np.pi, (B, 3)), rng.uniform(-np.pi, np.pi, (B, 3))
    planner = PathPlanner(position_profiles.Linear(), velocity_profiles.Gaussian(dt=1e-3, acceleration=1.0))
    dev = torch.device("cuda", 0)
    t = lambda x: torch.tensor(x, device=dev)  # noqa: E731
    sp, tp, tvm, tso, tto = t(start), t(target), t(vm), t(so), t(to)
    zero = torch.zeros(B, dtype=torch.float64, device=dev)

    # whole public call (includes input conversion and the host synchronisation)
    for _ in range(3):
        planner.generate_path(sp, tp, tvm, start_orientation=tso, target_orientation=tto)
    torch.cuda.synchronize()
    walls = []
    for _ in range(a.iters):
        t0 = time.perf_counter()
        path = planner.generate_path(sp, tp, tvm, start_orientation=tso, target_orientation=tto)
        torch.cuda.synchronize()
        walls.append(time.perf_counter() - t0)
    s_max = planner.n_timesteps
    lengths = planner.lengths.cpu().numpy()

    # the two launches and the readback on their own
    L = _lib.lib()
    p = C.byref(planner.params)
    table = planner._table_on(dev)
    lens = torch.empty(B, dtype=torch.int64, device=dev)
    plan = torch.empty((B, C.sizeof(_abi.PathRec) // 8), dtype=torch.float64, device=dev)
    buf = torch.empty((s_max, B, 12), dtype=torch.float64, device=dev)
    stream = torch.cuda.current_stream(dev).cuda_stream
    ph1, rb, ph2 = [], [], []
    for it in range(a.iters + 3):
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
        ev[0].record()
        _lib.check(L.abrb_path_plan(p, table.data_ptr(), sp.data_ptr(), tp.data_ptr(), tvm.data_ptr(), zero.data_ptr(),
                                    zero.data_ptr(), lens.data_ptr(), plan.data_ptr(), B, stream))
        ev[1].record()
        int(lens.max().item())
        ev[2].record()
        _lib.check(L.abrb_path_fill_f64(p, table.data_ptr(), sp.data_ptr(), tp.data_ptr(), zero.data_ptr(),
                                        zero.data_ptr(), tso.data_ptr(), tto.data_ptr(), plan.data_ptr(),
                                        lens.data_ptr(), s_max, buf.data_ptr(), B, stream))
        ev[3].record()
        torch.cuda.synchronize()
        if it >= 3:
            ph1.append(ev[0].elapsed_time(ev[1]) * 1e3)
            rb.append(ev[1].elapsed_time(ev[2]) * 1e3)
            ph2.append(ev[2].elapsed_time(ev[3]) * 1e3)
    assert torch.equal(buf.permute(1, 0, 2), path)

    n_host = 8
    t0 = time.perf_counter()
    path_oracle.plan(planner.table, start[:n_host], target[:n_host], vm[:n_host], 0.0, 0.0, "gaussian", 1e-3, 1.0, 3,
                     "rxyz", so[:n_host], to[:n_host])
    host_per_path = (time.perf_counter() - t0) / n_host

    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    bytes_out = s_max * B * 12 * 8
    res = dict(batch=B, s_max=s_max, mean_length=float(lengths.mean()), plan_us=float(np.median(ph1)),
               readback_us=float(np.median(rb)), fill_us=float(np.median(ph2)),
               generate_path_us=float(np.median(walls) * 1e6), fill_GBps=bytes_out / (np.median(ph2) * 1e-6) / 1e9,
               oracle_host_ms_per_path=host_per_path * 1e3, gpu=gpu[0] if gpu else "unknown")
    print(json.dumps(res))


if __name__ == "__main__":
    main()
