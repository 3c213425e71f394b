"""Cost of measurement noise at the policy's input in the particle rollouts (DESIGN.md section 23).

Metric-like dynamics (n = 300 points, E = 10 state dimensions, U = 2, RBF policy with 50 centres, H = 40, no angles)
for P in {1024, 16384} particles.  Each round times, with CUDA events around eager calls after a warm-up, the median
over ``--reps`` calls of four calls without noise and with v = 0.01 in every dimension, alternated in one process:
the step-wise forward, its pathwise gradient, the score-function gradient and the consistent sampler's forward +
gradient.  Prints the card's name, power limit and SM clock limit, then one JSON line per (round, P) in milliseconds
per rollout.  Usage: python scripts/particle_noise_timing.py [--reps 5] [--rounds 2]"""
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=2)
    args = ap.parse_args()
    H, E = 40, 10
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()
    print(json.dumps({"device": torch.cuda.get_device_name(0), "nvidia_smi": card[:1]}))
    dyn, spec, terms = problem(0)
    v = 0.01 * np.ones(E)
    for rnd in range(args.rounds):
        for P in (1024, 16384):
            rng = np.random.RandomState(P)
            x0, eps, nu = 0.1 * rng.randn(P, E) + 0.5, rng.randn(P, H, E), rng.randn(P, H, E)
            row = {"round": rnd, "D": dyn.D, "P": P, "H": H}
            for tag, nz in (("", None), ("noisy_", v)):
                kw = dict(measurement_noise=nz)
                inputs = (x0, eps, None if nz is None else nu)
                plans = [("forward", engine.ParticlePlan(dyn, spec, terms, P, H, **kw), "launch"),
                         ("pathwise", engine.ParticlePlan(dyn, spec, terms, P, H, grad=True, **kw), "launch_grad"),
                         ("score", engine.ParticlePlan(dyn, spec, terms, P, H, grad=True, estimator="score", **kw),
                          "launch_grad")]
                for what, plan, call in plans:
                    plan.set_inputs(*inputs)
                    row[tag + what + "_ms"] = median_ms(getattr(plan, call), args.reps)
                del plans, plan
                torch.cuda.empty_cache()
                plan = engine.ConsistentGradPlan(dyn, spec, terms, P, H, **kw)
                plan.set_inputs(*inputs)
                row[tag + "consistent_ms"] = median_ms(plan.launch_grad, args.reps)
                del plan
                torch.cuda.empty_cache()
            print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
