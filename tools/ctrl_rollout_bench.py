"""Times the closed-loop Joint and Sliding rollouts against the loop a user writes without them.  UR5, fp64, dt = 1e-3,
4 096 trajectories x 128 steps, per-trajectory paths: Joint(kp=300, kv=20) along a path planned by
InverseKinematics.generate_path, Sliding(kd=3, lamb=10) along a 5 cm straight line from the end effector.  The
starts are kept away from singularities of J[:3] (condition number below 12).

    (a) rollout_path, record=() (cost only)
    (b) rollout_path with q, dq, u and x recorded
    (c) per step through the public API: generate, forward_dynamics, semi-implicit Euler (what rollout_path replaces)
    (d) simulate of the same torques (the plant alone, for scale)

Each variant is warmed up, then timed with CUDA events over --reps repeats; the median and the spread are printed.
The card's name, power limit and maximum SM clock are read (nvidia-smi --query-gpu, read only) in the same run.

    python tools/ctrl_rollout_bench.py [--B 4096] [--steps 128] [--reps 7]
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from rollout_path_bench import card, timed  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--B", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=128)
    ap.add_argument("--reps", type=int, default=7)
    args = ap.parse_args()
    import numpy as np
    import torch

    from abr_control_b200.arms import ur5
    from abr_control_b200.controllers import Joint, Sliding
    from abr_control_b200.controllers.path_planners.inverse_kinematics import InverseKinematics

    assert torch.cuda.is_available(), "this benchmark needs a CUDA device"
    dev = torch.device("cuda", 0)
    B, S, dt = args.B, args.steps, 1e-3
    rc = ur5.Config()
    rng = np.random.default_rng(0)
    pool = torch.as_tensor(rng.uniform(0, 2 * np.pi, (4 * B, 6)), device=dev)
    q0 = pool[torch.linalg.cond(rc.eval(pool, want=("J",))["J"][:, :3]) < 12][:B].contiguous()
    assert len(q0) == B
    dq0 = torch.as_tensor(rng.uniform(-0.3, 0.3, (B, 6)), device=dev)
    x0 = rc.Tx("EE", q0)
    targets = torch.cat([x0 + torch.as_tensor(rng.uniform(-0.1, 0.1, (B, 3)), device=dev),
                         torch.as_tensor(rng.uniform(-np.pi, np.pi, (B, 3)), device=dev)], 1).contiguous()
    jpath = InverseKinematics(rc).generate_path(q0, targets, n_timesteps=S, dt=0.01)[0].permute(1, 0, 2)
    end = torch.as_tensor(rng.normal(size=(B, 3)), device=dev)
    end = 0.05 * end / end.norm(dim=1, keepdim=True)
    ramp = torch.linspace(0, 1, S, device=dev, dtype=torch.float64)[:, None, None]
    xpath = (x0[None] + ramp * end[None]).contiguous()
    print(f"card: {card()}", flush=True)
    ctrls = {"joint": (Joint(rc, kp=300, kv=20), jpath), "sliding": (Sliding(rc, kd=3.0, lamb=10.0), xpath)}

    def loop(c, path):
        q, dq = q0.clone(), dq0.clone()
        for t in range(S):
            u = c.generate(q, dq, path[t])
            dq = dq + rc.forward_dynamics(q, dq, u) * dt
            q = q + dq * dt
        return q

    results = {}
    for which, (c, path) in ctrls.items():
        u = c.rollout_path(q0, dq0, path, dt=dt, record=("u",))[2]["u"]
        runs = {
            f"{which}_a_rollout_path_cost_only": lambda: c.rollout_path(q0, dq0, path, dt=dt, record=()),
            f"{which}_b_rollout_path_full_records": lambda: c.rollout_path(q0, dq0, path, dt=dt),
            f"{which}_c_user_loop_generate_forward_dynamics_euler": lambda: loop(c, path),
            f"{which}_d_simulate_same_torques": lambda: rc.simulate(q0, dq0, u, dt=dt, record=()),
        }
        for name, fn in runs.items():
            med, lo, hi = timed(fn, args.reps)
            results[name] = dict(ms_median=med, ms_min=lo, ms_max=hi, us_per_step=med / S * 1e3)
            print(f"{name:52s} {med:9.3f} ms  (min {lo:.3f}, max {hi:.3f})  {med / S * 1e3:9.2f} us/step", flush=True)
        # (a) and (c) compute the same closed loop: say how far apart they end
        qa = c.rollout_path(q0, dq0, path, dt=dt, record=())[0]
        results[f"{which}_rollout_vs_user_loop_max_abs_q"] = float((qa - loop(c, path)).abs().max())
    print(json.dumps(dict(card=card(), B=B, steps=S, results=results)))


if __name__ == "__main__":
    main()
