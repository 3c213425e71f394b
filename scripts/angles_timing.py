"""Per-step cost of angular state dimensions in the moment-matching rollout (DESIGN.md section 19).

At the metric shape (N = 300 dynamics points, Ds = 10 state dimensions, U = 2, RBF policy with 50 centres, H = 40,
R = 32 restarts) it times one captured CUDA graph of the forward cascade, and of the taped forward + reverse sweep,
for A = 0 angles (the entry points without angles) and A = 1, 2 (pilco_rollout_angles_*: the policy sees Dh = Ds + A
inputs, the dynamics GP D = Dh + U).  Prints one JSON line per A with the median over ``--reps`` replays of
microseconds per rollout step (per restart-step: divide by R).  Usage: python scripts/angles_timing.py [--reps 20]"""
import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from pilco_b200 import engine, _lib        # noqa: E402


def problem(A, N=300, Ds=10, U=2, bf=50, R=32, seed=0):
    Dh = Ds + A
    D = Dh + U
    rng = np.random.RandomState(seed)
    X = rng.rand(N, D)
    Y = 0.05 * (np.sin(X) @ rng.rand(D, Ds))
    dyn = engine.gp_factorize(X, Y, 1.0 + rng.rand(Ds, D), 0.05 * (1.0 + rng.rand(Ds)), 1e-3 * np.ones(Ds))
    Xc, Yc = 0.5 * rng.randn(R, bf, Dh) + 0.5, 0.1 * rng.randn(R, bf, U)
    lc = 1.0 + 0.1 * rng.randn(R, U, Dh)
    pgp = engine.gp_factorize(Xc, Yc, lc, np.ones((R, U)), 1e-4 * np.ones((R, U)), need_iK=False, mode=1)
    spec = dict(kind=_lib.POLICY_RBF, Ds=Dh, U=U, squash=True, max_action=np.ones(U), gp=pgp)
    terms = [dict(kind=_lib.REWARD_EXP, coef=1.0, W=np.eye(Ds), t=np.zeros(Ds))]
    return dyn, spec, terms, X[0, :Ds].copy(), 0.1 * np.eye(Ds)


def time_graph(plan, backward, reps):
    g = plan.capture(backward=backward)
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        g.replay()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b) * 1e3)
    return float(np.median(ts))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    H, R = 40, 32
    for A in (0, 1, 2):
        dyn, spec, terms, m0, S0 = problem(A, R=R)
        angles = list(range(A)) if A else None
        row = {"A": A, "H": H, "R": R, "device": torch.cuda.get_device_name(0)}
        for what, backward in (("forward", False), ("forward_backward", True)):
            plan = engine.RolloutPlan(dyn, spec, terms, m0, S0, H, R=R, grad=backward, angles=angles)
            us = time_graph(plan, backward, args.reps)
            row[what + "_us_per_step"] = us / H
        print(json.dumps(row))


if __name__ == "__main__":
    main()
