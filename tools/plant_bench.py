"""Times the plant on its own against the loops a user writes without it.  UR5, fp64, dt = 1e-3.

    (a) simulate, 4 096 trajectories x 128 steps, per-trajectory torques and path, record=() (cost only)
    (b) the same with full records (q, dq, u, x)
    (c) per step: eval_into (M, g, C), torch.linalg.solve, semi-implicit Euler update (what simulate replaces)
    (d) OSC(kp=10).rollout_path at the same size, per-trajectory path, cost only (the closed loop, for scale)
    (e) forward_dynamics at 65 536 states, against (f) eval_into (M, g, C) + torch.linalg.solve

Each variant is warmed up, then timed with CUDA events over --reps repeats; the median and the spread are printed.
The card's name, power limit and maximum SM clock are read (nvidia-smi --query-gpu, read only) in the same run.

    python tools/plant_bench.py [--B 4096] [--steps 128] [--states 65536] [--reps 7]
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
    from abr_control_b200.controllers import OSC

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
    M = torch.empty((B, 6, 6), dtype=q0.dtype, device=dev)
    g, Cm = torch.empty_like(q0), torch.empty((B, 6, 6), dtype=q0.dtype, device=dev)

    def loop():
        q, dq = q0.clone(), dq0.clone()
        for t in range(S):
            rc.eval_into(q, dq, {"M": M, "g": g, "C": Cm})
            ddq = torch.linalg.solve(M, (u[t] + g - torch.bmm(Cm, dq[..., None])[..., 0])[..., None])[..., 0]
            dq += ddq * dt
            q += dq * dt
        return q

    c = OSC(rc, kp=10)
    Bs = args.states
    qs = torch.as_tensor(rng.uniform(0, 2 * np.pi, (Bs, 6)), device=dev)
    dqs = torch.as_tensor(rng.uniform(-0.5, 0.5, (Bs, 6)), device=dev)
    us = torch.as_tensor(rng.normal(size=(Bs, 6)), device=dev)
    Ms, gs, Cs = (torch.empty((Bs, 6, 6), dtype=qs.dtype, device=dev), torch.empty_like(qs),
                  torch.empty((Bs, 6, 6), dtype=qs.dtype, device=dev))

    def fd_loop():
        rc.eval_into(qs, dqs, {"M": Ms, "g": gs, "C": Cs})
        return torch.linalg.solve(Ms, (us + gs - torch.bmm(Cs, dqs[..., None])[..., 0])[..., None])[..., 0]

    runs = {
        "a_simulate_cost_only": (S, lambda: rc.simulate(q0, dq0, u, dt=dt, path=path, record=())),
        "b_simulate_full_records": (S, lambda: rc.simulate(q0, dq0, u, dt=dt, path=path)),
        "c_user_loop_eval_solve_euler": (S, loop),
        "d_osc_rollout_path_cost_only": (S, lambda: c.rollout_path(q0, dq0, path, dt=dt, record=())),
        "e_forward_dynamics_65536": (1, lambda: rc.forward_dynamics(qs, dqs, us)),
        "f_eval_into_solve_65536": (1, fd_loop),
    }
    results = {}
    for name, (per, fn) in runs.items():
        med, lo, hi = timed(fn, args.reps)
        results[name] = dict(ms_median=med, ms_min=lo, ms_max=hi, us_per_step=med / per * 1e3)
        print(f"{name:30s} {med:9.3f} ms  (min {lo:.3f}, max {hi:.3f})  {med / per * 1e3:9.2f} us/{'step' if per > 1 else 'call'}",
              flush=True)
    # (a) and (c) compute the same plant: say how far apart they end
    qa = rc.simulate(q0, dq0, u, dt=dt, record=())[0]
    results["simulate_vs_user_loop_max_abs_q"] = float((qa - loop()).abs().max())
    results["forward_dynamics_vs_solve_max_abs"] = float((rc.forward_dynamics(qs, dqs, us) - fd_loop()).abs().max())
    print(json.dumps(dict(card=card(), B=B, steps=S, states=Bs, results=results)))


if __name__ == "__main__":
    main()
