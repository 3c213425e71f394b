"""Cost of PILCO's exploration objective in the particle rollouts (DESIGN.md section 24).

Metric-like dynamics (n = 300 points, E = 10 state dimensions, U = 2, RBF policy with 50 centres, H = 40, no angles)
for P in {1024, 16384} particles.  Each round times, with CUDA events around eager calls after a warm-up, the median
over ``--reps`` calls of the pathwise gradient and the consistent sampler's forward + gradient without exploration,
at b = 0 (the moments only) and at b = 0.5, alternated in one process.  Prints the card's name, power limit and SM clock
limit, then one JSON line per (round, P) in milliseconds per rollout.
Usage: python scripts/particle_explore_timing.py [--reps 5] [--rounds 2]"""
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
    for rnd in range(args.rounds):
        for P in (1024, 16384):
            rng = np.random.RandomState(P)
            x0, eps = 0.1 * rng.randn(P, E) + 0.5, rng.randn(P, H, E)
            row = {"round": rnd, "D": dyn.D, "P": P, "H": H}
            for tag, b in (("", None), ("b0_", 0.0), ("explore_", 0.5)):
                plan = engine.ParticlePlan(dyn, spec, terms, P, H, grad=True, exploration=b)
                plan.set_inputs(x0, eps)
                row[tag + "pathwise_ms"] = median_ms(plan.launch_grad, args.reps)
                del plan
                torch.cuda.empty_cache()
                plan = engine.ConsistentGradPlan(dyn, spec, terms, P, H, exploration=b)
                plan.set_inputs(x0, eps)
                row[tag + "consistent_ms"] = median_ms(plan.launch_grad, args.reps)
                del plan
                torch.cuda.empty_cache()
            print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
