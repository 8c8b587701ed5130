"""Times the derivatives of the plant.  UR5, fp64, dt = 1e-3.

    (a) simulate, 4 096 trajectories x 128 steps, per-trajectory torques and path, record=() (cost only, no grad)
    (b) the same call with u, q0, dq0 requiring grad (the forward pass of a gradient step: records q and dq inside)
    (c) the backward pass of (b): cost.sum().backward() through abrb_plant_rollout_vjp_*
    (d) forward_dynamics_derivatives at 65 536 states, against (e) forward_dynamics at the same states

Each variant is warmed up, then timed with CUDA events over --reps repeats; the median and the spread are printed.
The card's name, power limit and maximum SM clock are read (nvidia-smi --query-gpu, read only) in the same run.

    python tools/plant_grad_bench.py [--B 4096] [--steps 128] [--states 65536] [--reps 7]
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
    ap.add_argument("--states", type=int, default=65536)
    ap.add_argument("--reps", type=int, default=7)
    args = ap.parse_args()
    import numpy as np
    import torch

    from abr_control_b200.arms import ur5

    assert torch.cuda.is_available(), "this benchmark needs a CUDA device"
    dev = torch.device("cuda", 0)
    B, S, dt = args.B, args.steps, 1e-3
    rc = ur5.Config()
    rng = np.random.default_rng(0)
    q0 = torch.as_tensor(rng.uniform(0, 2 * np.pi, (B, 6)), device=dev)
    dq0 = torch.as_tensor(rng.uniform(-0.5, 0.5, (B, 6)), device=dev)
    u = torch.as_tensor(rng.normal(size=(S, B, 6)), device=dev) - rc.eval(q0, want=("g",))["g"][None]
    u = u.contiguous()
    target = torch.as_tensor(rng.uniform(-0.6, 0.6, (B, 6)), device=dev)
    path = (target[None] + torch.linspace(0, 0.1, S, device=dev, dtype=torch.float64)[:, None, None]).contiguous()
    print(f"card: {card()}", flush=True)
    ug, qg, dqg = (t.clone().requires_grad_() for t in (u, q0, dq0))

    def fwd_grad():
        return rc.simulate(qg, dqg, ug, dt=dt, path=path, record=())[3]

    cost = fwd_grad()

    def bwd():
        ug.grad = qg.grad = dqg.grad = None
        torch.autograd.backward(cost.sum(), retain_graph=True)

    Bs = args.states
    qs = torch.as_tensor(rng.uniform(0, 2 * np.pi, (Bs, 6)), device=dev)
    dqs = torch.as_tensor(rng.uniform(-0.5, 0.5, (Bs, 6)), device=dev)
    us = torch.as_tensor(rng.normal(size=(Bs, 6)), device=dev)
    runs = {
        "a_simulate_cost_only": (S, lambda: rc.simulate(q0, dq0, u, dt=dt, path=path, record=())),
        "b_simulate_forward_under_grad": (S, fwd_grad),
        "c_simulate_backward": (S, bwd),
        "d_forward_dynamics_derivatives_65536": (1, lambda: rc.forward_dynamics_derivatives(qs, dqs, us)),
        "e_forward_dynamics_65536": (1, lambda: rc.forward_dynamics(qs, dqs, us)),
    }
    results = {}
    for name, (per, fn) in runs.items():
        med, lo, hi = timed(fn, args.reps)
        results[name] = dict(ms_median=med, ms_min=lo, ms_max=hi, us_per_step=med / per * 1e3)
        print(f"{name:38s} {med:9.3f} ms  (min {lo:.3f}, max {hi:.3f})  {med / per * 1e3:9.2f} us/{'step' if per > 1 else 'call'}",
              flush=True)
    print(json.dumps(dict(card=card(), B=B, steps=S, states=Bs, results=results)))


if __name__ == "__main__":
    main()
