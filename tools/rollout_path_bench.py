"""Times the path-following rollout against the fixed-target rollout and against the per-step loop a user would write
without it.  UR5, fp64, 4 096 trajectories x 128 steps, dt = 1e-3 (the MPC rollout scale), for two controllers:
OSC(kp=10) (x, y, z; the general kernel) and OSC(kp=10, ctrlr_dof=[True]*6, use_C=True) (the plain kernel).

    (a) rollout to a fixed target, recording q, dq, u
    (b) rollout_path, one shared path, recording q, dq, u, x
    (c) rollout_path, per-trajectory path and path velocity, record=(), cost only
    (d) per step: generate_into, eval_into (M, g, C), torch.linalg.solve, semi-implicit Euler update

Each variant is warmed up, then timed with CUDA events over --reps repeats; the median and the spread are printed.
The card's name, power limit and maximum SM clock are read (nvidia-smi --query-gpu, read only) in the same run.

    python tools/rollout_path_bench.py [--B 4096] [--steps 128] [--reps 7]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})"


def timed(fn, reps):
    import torch

    fn()  # warm-up of this exact shape
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts)), float(min(ts)), float(max(ts))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--B", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=128)
    ap.add_argument("--reps", type=int, default=7)
    args = ap.parse_args()
    import torch

    from abr_control_b200.arms import ur5
    from abr_control_b200.controllers import OSC

    assert torch.cuda.is_available(), "this benchmark needs a CUDA device"
    dev = torch.device("cuda", 0)
    B, S, dt = args.B, args.steps, 1e-3
    rc = ur5.Config()
    rng = np.random.default_rng(0)
    q0 = torch.as_tensor(rng.uniform(0, 2 * np.pi, (B, 6)), device=dev)
    dq0 = torch.as_tensor(rng.uniform(-0.5, 0.5, (B, 6)), device=dev)
    target = torch.as_tensor(rng.uniform(-0.6, 0.6, (B, 6)), device=dev)
    shared = torch.as_tensor(np.linspace(-0.3, 0.3, S)[:, None] * np.ones((1, 6)) + 0.2, device=dev).contiguous()
    per = (target[None] + torch.linspace(0, 0.1, S, device=dev, dtype=torch.float64)[:, None, None]).contiguous()
    per_v = torch.full((S, B, 6), 0.1, device=dev, dtype=torch.float64)
    print(f"card: {card()}", flush=True)
    results = {}
    for label, kw in (("general_xyz_kp10", dict(kp=10)), ("plain_6dof_C", dict(kp=10, ctrlr_dof=[True] * 6, use_C=True))):
        c = OSC(rc, **kw)
        u = torch.empty_like(q0)
        M = torch.empty((B, 6, 6), dtype=q0.dtype, device=dev)
        g, Cm = torch.empty_like(q0), torch.empty((B, 6, 6), dtype=q0.dtype, device=dev)

        def loop():
            q, dq = q0.clone(), dq0.clone()
            for _ in range(S):
                c.generate_into(q, dq, target, u)
                rc.eval_into(q, dq, {"M": M, "g": g, "C": Cm})
                ddq = torch.linalg.solve(M, (u + g - torch.bmm(Cm, dq[..., None])[..., 0])[..., None])[..., 0]
                dq += ddq * dt
                q += dq * dt
            return q

        runs = {
            "a_rollout_fixed_qdqu": lambda: c.rollout(q0, dq0, target, steps=S, dt=dt, record=("q", "dq", "u")),
            "b_path_shared_qdqux": lambda: c.rollout_path(q0, dq0, shared, dt=dt, record=("q", "dq", "u", "x")),
            "c_path_per_traj_pv_cost": lambda: c.rollout_path(q0, dq0, per, dt=dt, path_velocity=per_v, record=()),
            "d_user_loop": loop,
        }
        for name, fn in runs.items():
            med, lo, hi = timed(fn, args.reps)
            results[f"{label}/{name}"] = dict(ms_median=med, ms_min=lo, ms_max=hi, us_per_step=med / S * 1e3)
            print(f"{label:18s} {name:26s} {med:9.3f} ms  (min {lo:.3f}, max {hi:.3f})  {med / S * 1e3:8.2f} us/step",
                  flush=True)
        # (a) and (b) with a constant path describe the same closed loop: say so next to the timing
        qa, _, ta = c.rollout(q0, dq0, target, steps=S, dt=dt)
        qb, _, tb, _ = c.rollout_path(q0, dq0, target[None].expand(S, B, 6).contiguous(), dt=dt)
        results[f"{label}/fixed_vs_constant_path_max_abs_u"] = float((ta["u"] - tb["u"]).abs().max())
    print(json.dumps(dict(card=card(), B=B, steps=S, results=results)))


if __name__ == "__main__":
    main()
