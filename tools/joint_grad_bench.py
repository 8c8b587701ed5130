"""Times the gradient of the Joint closed loop.  UR5, fp64, dt = 1e-3, kp = 300, kv = 20.

    (a) Joint.rollout_path, 4 096 trajectories x 128 steps, per-trajectory path and path velocity, record=() (cost
        only, no grad)
    (b) the same call with the path, the path velocity, q0, dq0 and a 0-d kp requiring grad (the forward pass of a
        gradient step: records q and dq inside)
    (c) the backward pass of (b): cost.sum().backward() through abrb_joint_rollout_path_vjp_*

Each variant is warmed up, then timed with CUDA events over --reps repeats; the median and the spread are printed.
The card's name, power limit and maximum SM clock are read (nvidia-smi --query-gpu, read only) in the same run.
tools/plant_grad_bench.py times the open-loop plant's gradient the same way.

    python tools/joint_grad_bench.py [--B 4096] [--steps 128] [--reps 7]
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

    from abr_control_b200 import controllers
    from abr_control_b200.arms import ur5

    assert torch.cuda.is_available(), "this benchmark needs a CUDA device"
    dev = torch.device("cuda", 0)
    B, S, dt = args.B, args.steps, 1e-3
    rc = ur5.Config()
    rng = np.random.default_rng(0)
    q0 = torch.as_tensor(rng.uniform(-2, 2, (B, 6)), device=dev)
    dq0 = torch.as_tensor(rng.uniform(-0.5, 0.5, (B, 6)), device=dev)
    path = (q0[None] + torch.as_tensor(np.cumsum(rng.normal(scale=0.01, size=(S, B, 6)), 0), device=dev)).contiguous()
    pv = torch.as_tensor(rng.normal(scale=0.5, size=(S, B, 6)), device=dev)
    print(f"card: {card()}", flush=True)
    plain = controllers.Joint(rc, kp=300.0, kv=20.0)
    kp = torch.tensor(300.0, dtype=torch.float64, device=dev, requires_grad=True)
    grad = controllers.Joint(rc, kp=kp, kv=20.0)
    pg, vg, qg, dqg = (t.clone().requires_grad_() for t in (path, pv, q0, dq0))

    def fwd_grad():
        return grad.rollout_path(qg, dqg, pg, dt=dt, path_velocity=vg, record=())[3]

    cost = fwd_grad()

    def bwd():
        pg.grad = vg.grad = qg.grad = dqg.grad = kp.grad = None
        torch.autograd.backward(cost.sum(), retain_graph=True)

    runs = {
        "a_rollout_path_cost_only": lambda: plain.rollout_path(q0, dq0, path, dt=dt, path_velocity=pv, record=()),
        "b_rollout_path_forward_under_grad": fwd_grad,
        "c_rollout_path_backward": bwd,
    }
    results = {}
    for name, fn in runs.items():
        med, lo, hi = timed(fn, args.reps)
        results[name] = dict(ms_median=med, ms_min=lo, ms_max=hi, us_per_step=med / S * 1e3)
        print(f"{name:38s} {med:9.3f} ms  (min {lo:.3f}, max {hi:.3f})  {med / S * 1e3:9.2f} us/step", flush=True)
    print(json.dumps(dict(card=card(), B=B, steps=S, results=results)))


if __name__ == "__main__":
    main()
