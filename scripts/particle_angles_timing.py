"""Cost of angular state dimensions in the particle rollouts (DESIGN.md section 20).

Metric-like dynamics (n = 300 points, E = 10 state dimensions, U = 2, RBF policy with 50 centres, H = 40) with A = 0
angles (the entry points without angles; the dynamics GP has D = 12 inputs) and A = 1 (pilco_particles_angles_*;
D = 13).  For P in {1024, 16384} particles it times, with CUDA events around eager calls after a warm-up, the median
over ``--reps`` calls of one rollout: the step-wise forward, its pathwise gradient, the consistent sampler's gradient
(forward included) and the score-function gradient.  Prints the card's name and power limit, then one JSON line per
(A, P) in milliseconds per rollout.  Usage: python scripts/particle_angles_timing.py [--reps 5]"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from pilco_b200 import engine, _lib        # noqa: E402


def problem(A, N=300, E=10, U=2, bf=50, seed=0):
    Dh = E + A
    D = Dh + U
    rng = np.random.RandomState(seed)
    X = rng.rand(N, D)
    Y = 0.05 * (np.sin(X) @ rng.rand(D, E))
    dyn = engine.gp_factorize(X, Y, 1.0 + rng.rand(E, D), 0.05 * (1.0 + rng.rand(E)), 1e-3 * np.ones(E))
    Xc, Yc, lc = 0.5 * rng.randn(bf, Dh) + 0.5, 0.1 * rng.randn(bf, U), 1.0 + 0.1 * rng.randn(U, Dh)
    pgp = engine.gp_factorize(Xc, Yc, lc, np.ones(U), 1e-4 * np.ones(U), need_iK=False, mode=1)
    spec = dict(kind=_lib.POLICY_RBF, Ds=Dh, U=U, squash=True, max_action=np.ones(U), gp=pgp)
    terms = [dict(kind=_lib.REWARD_EXP, coef=1.0, W=np.eye(E), t=np.zeros(E))]
    return dyn, spec, terms


def median_ms(fn, reps):
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    H, E = 40, 10
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()
    print(json.dumps({"device": torch.cuda.get_device_name(0), "nvidia_smi": card[:1]}))
    for A in (0, 1):
        dyn, spec, terms = problem(A)
        angles = [0] if A else None
        for P in (1024, 16384):
            rng = np.random.RandomState(P)
            x0, eps = 0.1 * rng.randn(P, E) + 0.5, rng.randn(P, H, E)
            row = {"A": A, "D": dyn.D, "P": P, "H": H}
            plans = [("forward", engine.ParticlePlan(dyn, spec, terms, P, H, angles=angles), "launch"),
                     ("pathwise", engine.ParticlePlan(dyn, spec, terms, P, H, grad=True, angles=angles), "launch_grad"),
                     ("score", engine.ParticlePlan(dyn, spec, terms, P, H, grad=True, estimator="score",
                                                   angles=angles), "launch_grad")]
            for what, plan, call in plans:
                plan.set_inputs(x0, eps)
                row[what + "_ms"] = median_ms(getattr(plan, call), args.reps)
            del plans, plan
            torch.cuda.empty_cache()
            plan = engine.ConsistentGradPlan(dyn, spec, terms, P, H, angles=angles)
            plan.set_inputs(x0, eps)
            row["consistent_ms"] = median_ms(plan.launch_grad, args.reps)
            del plan
            torch.cuda.empty_cache()
            print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
