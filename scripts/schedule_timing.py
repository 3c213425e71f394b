"""Cost of the time-varying linear policy (pilco_rollout_scheduled_*, DESIGN.md section 27) at the metric shape, and the
wall time of one receding-horizon step (PILCO.plan).

N = 300 dynamics points, E = 10 state dimensions, U = 2 (D = 12), H = 40, R = 32 restarts, taped.  One captured CUDA
graph of the forward cascade, and one of the forward + reverse sweep, for the stationary linear policy (the noisy call
every linear rollout uses) and for a schedule of H per-step (W_t, b_t), alternated ``--rounds`` times in this process;
each entry is the median over ``--reps`` replays, as rollout-steps/s (R H over the replay's time).  Then ``plan()`` of an
open-loop TimeVaryingLinearController at R = 8 restarts, 10 L-BFGS-B iterations, median wall time over ``--plans``
calls.  Prints the card's name, power limit and SM clock limit, then one JSON line per round.
Usage: python scripts/schedule_timing.py [--reps 30] [--rounds 3] [--plans 5]"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from pilco_b200 import engine, _lib, controllers, rewards        # noqa: E402
from pilco_b200.models.pilco import PILCO                        # noqa: E402
from obs_noise_timing import time_graph, card                   # noqa: E402


def problem(N=300, Ds=10, U=2, H=40, R=32, seed=0):
    D = Ds + U
    rng = np.random.RandomState(seed)
    X = rng.rand(N, D)
    Y = 0.05 * (np.sin(X) @ rng.rand(D, Ds))
    dyn = engine.gp_factorize(X, Y, 1.0 + rng.rand(Ds, D), 0.05 * (1.0 + rng.rand(Ds)), 1e-3 * np.ones(Ds))
    W, b = 0.1 * rng.randn(R, U, Ds), 0.1 * rng.randn(R, U)
    stationary = dict(kind=_lib.POLICY_LINEAR, Ds=Ds, U=U, squash=True, max_action=np.ones(U), W=W, b=b)
    scheduled = dict(stationary, W=W[:, None] + 0.01 * rng.randn(R, H, U, Ds), b=b[:, None] + 0.01 * rng.randn(R, H, U))
    terms = [dict(kind=_lib.REWARD_EXP, coef=1.0, W=np.eye(Ds), t=np.zeros(Ds))]
    return dyn, stationary, scheduled, terms, X, Y


def plan_time(X, Y, H, plans, restarts=8, maxiter=10):
    Ds, U = Y.shape[1], X.shape[1] - Y.shape[1]
    np.random.seed(0)
    c = controllers.TimeVaryingLinearController(Ds, U, H, feedback=False)
    pilco = PILCO((X, Y), controller=c, horizon=H, reward=rewards.ExponentialReward(Ds), m_init=X[:1, :Ds],
                  S_init=0.01 * np.eye(Ds))
    x = X[0, :Ds]
    pilco.plan(x, maxiter=maxiter, restarts=restarts)             # warm-up: factorisation, graph capture
    ts = []
    for _ in range(plans):
        t0 = time.perf_counter()
        pilco.plan(x, maxiter=maxiter, restarts=restarts)
        ts.append(time.perf_counter() - t0)
    return float(np.median(ts))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--plans", type=int, default=5)
    args = ap.parse_args()
    H, R = 40, 32
    print(json.dumps({"card": card(), "N": 300, "E": 10, "D": 12, "H": H, "R": R, "taped": True}))
    dyn, stationary, scheduled, terms, X, Y = problem(H=H, R=R)
    m0, S0 = X[0, :10].copy(), 0.1 * np.eye(10)
    graphs = {}
    for arm, spec in (("stationary", stationary), ("scheduled", scheduled)):
        for what, backward in (("forward", False), ("forward_backward", True)):
            plan = engine.RolloutPlan(dyn, spec, terms, m0, S0, H, R=R, grad=True, schedule=arm == "scheduled")
            graphs[(arm, what)] = (plan, plan.capture(backward=backward))
    torch.cuda.synchronize()
    for rnd in range(args.rounds):
        row = {"round": rnd}
        for what in ("forward", "forward_backward"):
            for arm in ("stationary", "scheduled"):          # alternated
                ms = time_graph(graphs[(arm, what)][1], args.reps)
                row["%s_steps_per_s_%s" % (what, arm)] = round(R * H / (ms * 1e-3))
        print(json.dumps(row))
    print(json.dumps({"plan_R": 8, "plan_H": 20, "maxiter": 10,
                      "plan_wall_s_median": plan_time(X[:200], Y[:200], 20, args.plans)}))


if __name__ == "__main__":
    main()
