"""Cost of the tanh MLP policy in the particle rollouts (pilco_particles_mlp_*, DESIGN.md section 29) beside the RBF
and linear policies.

N = 300 dynamics points, E = 10 state dimensions, U = 2 (D = 12), H = 40, step-wise sampler.  At P = 1024 and 16384
particles: one captured CUDA graph of the forward rollout (R = 1) and one of the forward + pathwise gradient (R = 8
restarts), for the 2 x 64 MLP, an RBF policy of 50 basis functions and a linear policy, alternated ``--rounds`` times
in this process; each entry is the median ms over ``--reps`` replays.  Prints the card's name, power limit and SM
clock limit, then one JSON line per round.
Usage: python scripts/particle_mlp_timing.py [--reps 20] [--rounds 3]"""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from pilco_b200 import engine, _lib                              # noqa: E402
from obs_noise_timing import time_graph, card                   # noqa: E402

ARMS = ("mlp", "rbf", "linear")


def problem(N=300, Ds=10, U=2, R=8, bf=50, hidden=(64, 64), seed=0):
    """the dynamics, {arm: (forward spec at R = 1, gradient spec at R restarts)}, terms, a start state"""
    D = Ds + U
    rng = np.random.RandomState(seed)
    X = rng.rand(N, D)
    Y = 0.05 * (np.sin(X) @ rng.rand(D, Ds))
    dyn = engine.gp_factorize(X, Y, 1.0 + rng.rand(Ds, D), 0.05 * (1.0 + rng.rand(Ds)), 1e-3 * np.ones(Ds))
    base = dict(Ds=Ds, U=U, squash=True, max_action=np.ones(U))
    W, b = 0.1 * rng.randn(R, U, Ds), 0.1 * rng.randn(R, U)
    lin = dict(base, kind=_lib.POLICY_LINEAR, W=W, b=b)
    n = engine.mlp_theta_size(Ds, U, hidden)
    theta = 0.1 * rng.randn(R, n)
    mlp = dict(base, kind=_lib.POLICY_MLP, hidden=hidden, theta=theta)
    Xc, Yc, lc = rng.rand(R, bf, Ds), 0.1 * rng.randn(R, bf, U), 1.0 + rng.rand(R, U, Ds)
    rbf = lambda s: engine.gp_factorize(Xc[s], Yc[s], lc[s], np.ones(np.shape(lc[s])[:-1]),
                                        1e-4 * np.ones(np.shape(lc[s])[:-1]), need_iK=False, mode=1)
    specs = {"linear": (dict(lin, W=W[0], b=b[0]), lin), "mlp": (dict(mlp, theta=theta[0]), mlp),
             "rbf": (dict(base, kind=_lib.POLICY_RBF, gp=rbf(0)), dict(base, kind=_lib.POLICY_RBF, gp=rbf(slice(None))))}
    terms = [dict(kind=_lib.REWARD_EXP, coef=1.0, W=np.eye(Ds), t=np.zeros(Ds))]
    return dyn, specs, terms, X[0, :Ds]


def captured(dyn, spec, terms, x0, eps, R, grad):
    """the plan and a CUDA graph of its launch (grad: launch_grad at R restarts; else launch at R = 1)"""
    P, H = eps.shape[:2]
    plan = engine.ParticlePlan(dyn, spec, terms, P, H, grad=grad, R=R if grad else 1)
    plan.set_inputs(x0, eps)
    run = plan.launch_grad if grad else plan.launch
    run()                                                   # eager warm-up: kernel attributes, predict set-up
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        run()
    return plan, g


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    H, R, E = 40, 8, 10
    print(json.dumps({"card": card(), "N": 300, "E": E, "D": 12, "H": H, "R_grad": R, "sampler": "step-wise",
                      "mlp": "2 x 64 tanh", "rbf_bf": 50}))
    dyn, specs, terms, m0 = problem(R=R)
    graphs = {}
    for P in (1024, 16384):
        rng = np.random.RandomState(P)
        x0, eps = m0[None] + 0.1 * rng.randn(P, E), rng.randn(P, H, E)
        for arm in ARMS:
            for what, grad in (("forward", False), ("forward_grad", True)):
                graphs[(P, arm, what)] = captured(dyn, specs[arm][grad], terms, x0, eps, R, grad)
    torch.cuda.synchronize()
    for rnd in range(args.rounds):
        row = {"round": rnd}
        for P in (1024, 16384):
            for what in ("forward", "forward_grad"):
                for arm in ARMS:                             # alternated
                    row["P%d_%s_ms_%s" % (P, what, arm)] = round(time_graph(graphs[(P, arm, what)][1], args.reps), 4)
        print(json.dumps(row))


if __name__ == "__main__":
    main()
