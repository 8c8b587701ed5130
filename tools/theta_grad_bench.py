"""Time the link-inertia gradient of ``simulate`` on the GPU: UR5, fp64, 4 096 trajectories x 128 steps, with a path,
an effort weight and compensate_gravity.

    (a) simulate forward + cost.sum().backward() with q0, dq0 and u requiring grad (the plant's adjoint only)
    (b) the same with theta requiring grad too: (b) - (a) is the share of abrb_plant_rollout_theta_vjp_*
    (c) the composed route for the same theta gradient, given the torque cotangents of (a): forward_dynamics at every
        recorded state, inverse_dynamics_regressor of Y(q, dq, ddq) and Y(q, 0, 0) in chunks, contracted by
        torch.matmul

CUDA events around each, medians over the timed repetitions; the card's name and power limit are printed with them.
"""
import argparse
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import abr_control_b200.arms as arms  # noqa: E402


def timed(fn, reps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    out = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        out.append(a.elapsed_time(b))
    return float(np.median(out))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--B", type=int, default=4096)
    ap.add_argument("--S", type=int, default=128)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--chunk", type=int, default=65536)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("theta_grad_bench needs a CUDA device")
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()
    print(f"device: {smi[0] if smi else torch.cuda.get_device_name(0)}")
    rc = arms.ur5.Config()
    B, S, n, dt, ew = a.B, a.S, 6, 1e-3, 1e-4
    g = torch.Generator(device="cuda").manual_seed(0)
    q = torch.rand((B, n), device="cuda", generator=g, dtype=torch.float64) * 2 * np.pi
    dq = torch.rand((B, n), device="cuda", generator=g, dtype=torch.float64) - 0.5
    x0 = rc.Tx("EE", q)
    path = torch.cat([x0, torch.zeros_like(x0)], 1)[None].expand(S, B, 6).contiguous()
    u = torch.randn((S, B, n), device="cuda", generator=g, dtype=torch.float64)
    th0 = torch.as_tensor(rc.inertial_parameters(), device="cuda")
    kw = dict(dt=dt, path=path, effort_weight=ew, compensate_gravity=True, record=("q", "dq", "u"))
    state = {}

    def run(with_theta):
        q0, dq0, uu = q.clone().requires_grad_(), dq.clone().requires_grad_(), u.clone().requires_grad_()
        th = th0.clone().requires_grad_() if with_theta else None
        _, _, tr, cost = rc.simulate(q0, dq0, uu, theta=th, **kw)
        cost.sum().backward()
        state.update(tr=tr, gu=uu.grad, gth=None if th is None else th.grad)

    def composed():
        tr, gu = state["tr"], state["gu"]
        with torch.no_grad():
            qp = torch.cat([q[None], tr["q"][:-1]]).reshape(-1, n)
            dqp = torch.cat([dq[None], tr["dq"][:-1]]).reshape(-1, n)
            tau = tr["u"].reshape(-1, n)
            gur = gu.reshape(-1, n)
            w = gur - 2 * ew * tau
            ddq = rc.forward_dynamics(qp, dqp, tau)
            out = torch.zeros(6 * n, dtype=torch.float64, device="cuda")
            for i in range(0, len(qp), a.chunk):
                s = slice(i, i + a.chunk)
                zero = torch.zeros_like(qp[s])
                Y = rc.inverse_dynamics_regressor(qp[s], dqp[s], ddq[s])
                Y0 = rc.inverse_dynamics_regressor(qp[s], zero, zero)
                out -= torch.matmul(w[s][:, None, :], Y)[:, 0].sum(0)
                out += torch.matmul(gur[s][:, None, :], Y0)[:, 0].sum(0)
            state["ref"] = out

    ta = timed(lambda: run(False), a.reps, a.warmup)
    tb = timed(lambda: run(True), a.reps, a.warmup)
    gth = state["gth"]
    tc = timed(composed, a.reps, a.warmup)
    rel = float((gth - state["ref"]).abs().max() / state["ref"].abs().max())
    print(f"UR5 fp64, {B} trajectories x {S} steps, path, effort weight {ew}, compensate_gravity")
    print(f"(a) simulate forward + backward, q0/dq0/u:        {ta:8.2f} ms")
    print(f"(b) the same with theta requiring grad:           {tb:8.2f} ms   theta share {tb - ta:7.2f} ms")
    print(f"(c) composed route (forward_dynamics, regressor):  {tc:8.2f} ms   (given the torque cotangents of (a))")
    print(f"(b) theta gradient vs (c): {rel:.2e} relative")


if __name__ == "__main__":
    main()
