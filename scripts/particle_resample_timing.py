"""Cost and gradient variance of the Gaussian-resampled particle rollouts (DESIGN.md section 26).

Metric-like dynamics (n = 300 points, E = 10 state dimensions, U = 2, D = 12, RBF policy with 50 centres, H = 40) for P
in {1024, 16384} particles.  Each round times, with CUDA events around eager calls after a warm-up, the median over
``--reps`` calls of the forward and of the forward + pathwise gradient, without and with resampling, alternated in one
process.  Then the gradient's spread over ``--seeds`` draws of (x0, eps, xi) at P = 1024, for the plain pathwise
estimator and the resampled one, at H = 40 and at ``--long`` steps: the summed per-parameter variance and its ratio to
the squared norm of the mean gradient.  Prints the card's name, power limit and SM clock limit, then one JSON line per
measurement.
Usage: python scripts/particle_resample_timing.py [--reps 5] [--rounds 2] [--seeds 16] [--long 100]"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from pilco_b200 import engine                            # noqa: E402
from particle_angles_timing import median_ms, problem   # noqa: E402


def _inputs(P, H, E, seed):
    rng = np.random.RandomState(seed)
    return 0.1 * rng.randn(P, E) + 0.5, rng.randn(P, H, E), rng.randn(P, H, E)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--seeds", type=int, default=16)
    ap.add_argument("--long", type=int, default=100)
    args = ap.parse_args()
    H, E = 40, 10
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()
    print(json.dumps({"device": torch.cuda.get_device_name(0), "nvidia_smi": card[:1]}))
    dyn, spec, terms = problem(0)
    for rnd in range(args.rounds):
        for P in (1024, 16384):
            x0, eps, xi = _inputs(P, H, E, P)
            row = {"round": rnd, "D": dyn.D, "P": P, "H": H}
            for tag, rs in (("", False), ("resampled_", True)):
                plan = engine.ParticlePlan(dyn, spec, terms, P, H, resample=rs)
                plan.set_inputs(x0, eps, xi=xi if rs else None)
                row[tag + "forward_ms"] = median_ms(plan.launch, args.reps)
                del plan
                plan = engine.ParticlePlan(dyn, spec, terms, P, H, grad=True, resample=rs)
                plan.set_inputs(x0, eps, xi=xi if rs else None)
                row[tag + "grad_ms"] = median_ms(plan.launch_grad, args.reps)
                del plan
                torch.cuda.empty_cache()
            print(json.dumps(row), flush=True)
    P = 1024
    for Hv in (H, args.long):
        row = {"variance": True, "P": P, "H": Hv, "seeds": args.seeds}
        for tag, rs in (("", False), ("resampled_", True)):
            plan = engine.ParticlePlan(dyn, spec, terms, P, Hv, grad=True, resample=rs)
            gs = []
            for k in range(args.seeds):
                x0, eps, xi = _inputs(P, Hv, E, 1000 + k)
                plan.set_inputs(x0, eps, xi=xi if rs else None)
                g = plan.launch_grad()
                gs.append(torch.cat([g[key].reshape(-1) for key in ("X", "Y", "ell")]).cpu().numpy())
            gs = np.stack(gs)
            var, mean = float(gs.var(0, ddof=1).sum()), gs.mean(0)
            row[tag + "grad_var"] = var
            row[tag + "var_over_mean2"] = var / max(float(mean @ mean), 1e-300)
            row[tag + "finite"] = bool(np.isfinite(gs).all())
            del plan
            torch.cuda.empty_cache()
        print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
