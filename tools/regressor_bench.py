"""Times the inverse-dynamics regressor and the identification built on it.  UR5, fp64.

    (a) inverse_dynamics_regressor at --states states (3n values in, 6n^2 out per state), and its share of the HBM bound
        (bytes moved over the H100 SXM data-sheet 3.35 TB/s; a bound, not a rate anyone reaches)
    (b) the same regressor through 6n calls of with_link_inertia(e_p).inverse_dynamics (what a user writes without it)
    (c) identify_link_inertia end to end on --B x --steps samples (two passes of the regressor over the samples, the fp64
        normal equations and the host solve), from the nominal model on samples of a perturbed one

(a) and (b) are timed with CUDA events over --iters calls per window, (c) one call per window; --reps windows each, the
median and the spread are printed.  The card's name, power limit and maximum SM clock are read (nvidia-smi
--query-gpu, read only) in the same run.

    python tools/regressor_bench.py [--states 65536] [--B 4096] [--steps 128] [--iters 20] [--reps 7]
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from rollout_path_bench import card, timed  # noqa: E402

HBM_BYTES_PER_S = 3.35e12  # H100 SXM data sheet


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--states", type=int, default=65536)
    ap.add_argument("--B", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=128)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--reps", type=int, default=7)
    args = ap.parse_args()
    import numpy as np
    import torch

    from abr_control_b200.arms import ur5

    assert torch.cuda.is_available(), "this benchmark needs a CUDA device"
    dev = torch.device("cuda", 0)
    print(f"card: {card()}", flush=True)
    rc = ur5.Config()
    n, Bs = 6, args.states
    rng = np.random.default_rng(0)
    q, dq, ddq = (torch.as_tensor(rng.uniform(lo, hi, (Bs, n)), device=dev)
                  for lo, hi in ((0, 2 * np.pi), (-5, 5), (-10, 10)))
    units = [rc.with_link_inertia(np.eye(6 * n)[p]) for p in range(6 * n)]
    Yb = torch.empty((Bs, n, 6 * n), dtype=q.dtype, device=dev)

    def baseline():
        for p, m in enumerate(units):
            Yb[:, :, p] = m.inverse_dynamics(q, dq, ddq)

    # samples of a perturbed UR5 (u from its inverse dynamics at random states) for the end-to-end fit
    K = args.B * args.steps
    th = rc.inertial_parameters().reshape(n, 6)
    th[:, :3] *= rng.uniform(0.5, 1.5, (n, 1))
    th[:, 3:] *= rng.uniform(0.5, 1.5, (n, 3))
    true = rc.with_link_inertia(th.reshape(-1))
    sq, sdq, sddq = (torch.as_tensor(rng.uniform(lo, hi, (K, n)), device=dev)
                     for lo, hi in ((0, 2 * np.pi), (-3, 3), (-20, 20)))
    su = true.inverse_dynamics(sq, sdq, sddq)

    it = args.iters
    runs = {
        "a_regressor": (it, lambda: [rc.inverse_dynamics_regressor(q, dq, ddq) for _ in range(it)]),
        "b_6n_inverse_dynamics_launches": (it, lambda: [baseline() for _ in range(it)]),
        "c_identify_link_inertia": (1, lambda: rc.identify_link_inertia(sq, sdq, sddq, su)),
    }
    results = {}
    for name, (per, fn) in runs.items():
        med, lo, hi = timed(fn, args.reps)
        results[name] = dict(ms_median=med / per, ms_min=lo / per, ms_max=hi / per)
        print(f"{name:32s} {med / per * 1e3:10.1f} us/call  (min {lo / per * 1e3:.1f}, max {hi / per * 1e3:.1f})",
              flush=True)
    moved = Bs * (3 * n + 6 * n * n) * 8
    bound_ms = moved / HBM_BYTES_PER_S * 1e3
    results["a_regressor"].update(bytes=moved, hbm_bound_ms=bound_ms,
                                  share_of_hbm_bound=bound_ms / results["a_regressor"]["ms_median"])
    Y = rc.inverse_dynamics_regressor(q, dq, ddq)
    baseline()
    results["regressor_vs_baseline_max_abs"] = float((Y - Yb).abs().max())
    theta, info = rc.identify_link_inertia(sq, sdq, sddq, su)
    results["identify"] = dict(samples=K, rank=info["rank"], rms_before=info["rms_before"], rms_after=info["rms_after"],
                               max_abs_basis_error=float(np.abs(info["basis"].T @ (theta - th.reshape(-1))).max()))
    print(f"regressor: {moved / 1e6:.1f} MB, HBM bound {bound_ms * 1e3:.1f} us, "
          f"{results['a_regressor']['share_of_hbm_bound']:.2f} of it", flush=True)
    print(json.dumps(dict(card=card(), states=Bs, samples=K, results=results)))


if __name__ == "__main__":
    main()
