"""Cost of measurement noise at the policy's input (pilco_rollout_noisy_*, DESIGN.md section 22) at the metric shape.

N = 300 dynamics points, E = 10 state dimensions, U = 2 (D = 12), RBF policies with 50 centres, H = 40, R = 32 restarts,
taped.  One captured CUDA graph of the forward cascade, and one of the forward + reverse sweep, without noise (the
entry points a rollout without it has always used) and with v = 0.01 on every state dimension (the noisy state and
trig kernels in place of the plain ones), alternated ``--rounds`` times in this process; each entry is the median over
``--reps`` replays in milliseconds per rollout.  Prints the card's name, power limit and SM clock limit, then one JSON
line per round.
Usage: python scripts/obs_noise_timing.py [--reps 30] [--rounds 3]"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from pilco_b200 import engine, _lib        # noqa: E402


def problem(N=300, Ds=10, U=2, bf=50, R=32, seed=0):
    D = Ds + U
    rng = np.random.RandomState(seed)
    X = rng.rand(N, D)
    Y = 0.05 * (np.sin(X) @ rng.rand(D, Ds))
    dyn = engine.gp_factorize(X, Y, 1.0 + rng.rand(Ds, D), 0.05 * (1.0 + rng.rand(Ds)), 1e-3 * np.ones(Ds))
    Xc, Yc = 0.5 * rng.randn(R, bf, Ds) + 0.5, 0.1 * rng.randn(R, bf, U)
    lc = 1.0 + 0.1 * rng.randn(R, U, Ds)
    pgp = engine.gp_factorize(Xc, Yc, lc, np.ones((R, U)), 1e-4 * np.ones((R, U)), need_iK=False, mode=1)
    spec = dict(kind=_lib.POLICY_RBF, Ds=Ds, U=U, squash=True, max_action=np.ones(U), gp=pgp)
    terms = [dict(kind=_lib.REWARD_EXP, coef=1.0, W=np.eye(Ds), t=np.zeros(Ds))]
    return dyn, spec, terms, X[0, :Ds].copy(), 0.1 * np.eye(Ds)


def time_graph(g, reps):
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        g.replay()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts))


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except (OSError, IndexError, subprocess.TimeoutExpired):
        out = torch.cuda.get_device_name(0) + ", power limit unknown"
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    H, R = 40, 32
    print(json.dumps({"card": card(), "N": 300, "E": 10, "D": 12, "bf": 50, "H": H, "R": R, "taped": True}))
    dyn, spec, terms, m0, S0 = problem(R=R)
    graphs = {}
    noise = {"off": None, "on": 0.01 * np.ones(m0.shape[0])}
    for nz in ("off", "on"):
        for what, backward in (("forward", False), ("forward_backward", True)):
            plan = engine.RolloutPlan(dyn, spec, terms, m0, S0, H, R=R, grad=True, measurement_noise=noise[nz])
            graphs[(nz, what)] = (plan, plan.capture(backward=backward))
    torch.cuda.synchronize()
    for rnd in range(args.rounds):
        row = {"round": rnd}
        for what in ("forward", "forward_backward"):
            for nz in ("off", "on"):                   # alternated: without noise, then with it
                row["%s_ms_noise_%s" % (what, nz)] = time_graph(graphs[(nz, what)][1], args.reps)
        print(json.dumps(row))


if __name__ == "__main__":
    main()
