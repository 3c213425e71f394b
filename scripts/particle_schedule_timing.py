"""Cost of the time-varying linear policy in the particle rollouts (pilco_particles_scheduled_*, DESIGN.md section 28),
and the wall time of one receding-horizon step planned on particles (PILCO.plan(num_samples=...)).

N = 300 dynamics points, E = 10 state dimensions, U = 2 (D = 12), H = 40, step-wise sampler.  At P = 1024 and 16384
particles: one captured CUDA graph of the forward rollout (R = 1) and one of the forward + pathwise gradient (R = 8
restarts), each for the stationary linear policy and for the constant schedule W_t = W, b_t = b (the same rollout
through the scheduled calls), alternated ``--rounds`` times in this process; each entry is the median ms over ``--reps``
replays.  Then ``plan(num_samples=256, restarts=8, maxiter=10)`` of an open-loop TimeVaryingLinearController (H = 10)
on the pendulum of examples/pendulum_numpy.py, median wall time over ``--plans`` calls, beside the moment-matching
``plan`` of the same controller.  Prints the card's name, power limit and SM clock limit, then one JSON line per round.
Usage: python scripts/particle_schedule_timing.py [--reps 20] [--rounds 3] [--plans 5]"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "examples"))
from pilco_b200 import engine, _lib, controllers, rewards        # noqa: E402
from pilco_b200.models.pilco import PILCO                        # noqa: E402
from obs_noise_timing import time_graph, card                   # noqa: E402
from pendulum_numpy import PendulumEnv, rollout                  # noqa: E402


def problem(N=300, Ds=10, U=2, H=40, R=8, seed=0):
    D = Ds + U
    rng = np.random.RandomState(seed)
    X = rng.rand(N, D)
    Y = 0.05 * (np.sin(X) @ rng.rand(D, Ds))
    dyn = engine.gp_factorize(X, Y, 1.0 + rng.rand(Ds, D), 0.05 * (1.0 + rng.rand(Ds)), 1e-3 * np.ones(Ds))
    W, b = 0.1 * rng.randn(R, U, Ds), 0.1 * rng.randn(R, U)
    stationary = dict(kind=_lib.POLICY_LINEAR, Ds=Ds, U=U, squash=True, max_action=np.ones(U), W=W, b=b)
    scheduled = dict(stationary, W=np.repeat(W[:, None], H, 1), b=np.repeat(b[:, None], H, 1))
    terms = [dict(kind=_lib.REWARD_EXP, coef=1.0, W=np.eye(Ds), t=np.zeros(Ds))]
    return dyn, stationary, scheduled, terms, X[0, :Ds]


def captured(dyn, spec, terms, x0, eps, R, grad, schedule):
    """the plan and a CUDA graph of its launch (grad: launch_grad at R restarts; else launch at R = 1)"""
    one = lambda s: dict(s, W=s["W"][0], b=s["b"][0])
    P, H = eps.shape[:2]
    plan = engine.ParticlePlan(dyn, spec if grad else one(spec), terms, P, H, grad=grad, R=R if grad else 1,
                               schedule=schedule)
    plan.set_inputs(x0, eps)
    run = plan.launch_grad if grad else plan.launch
    run()                                                   # eager warm-up: kernel attributes, predict set-up
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        run()
    return plan, g


def pendulum_pilco(H=10, seed=0):
    np.random.seed(seed)
    env = PendulumEnv(seed=seed)
    X, Y = [], []
    for _ in range(3):
        X_, Y_ = rollout(env, lambda x: env.sample_action(), 25)
        X.append(X_); Y.append(Y_)
    c = controllers.TimeVaryingLinearController(2, 1, H, max_action=env.max_torque, feedback=False)
    pilco = PILCO((np.vstack(X), np.vstack(Y)), controller=c, horizon=H,
                  reward=rewards.ExponentialReward(2, W=np.diag([1.0, 0.1]), t=np.array([np.pi / 3, 0.0])),
                  m_init=np.zeros((1, 2)), S_init=np.diag([0.01, 0.01]))
    pilco.optimize_models(restarts=1)
    return pilco, env.reset()


def plan_time(pilco, x, plans, **kw):
    pilco.plan(x, maxiter=10, restarts=8, seed=0, **kw)          # warm-up: plans, factorisation
    ts = []
    for k in range(plans):
        t0 = time.perf_counter()
        pilco.plan(x, maxiter=10, restarts=8, seed=k + 1, **kw)
        ts.append(time.perf_counter() - t0)
    return float(np.median(ts))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--plans", type=int, default=5)
    args = ap.parse_args()
    H, R, E = 40, 8, 10
    print(json.dumps({"card": card(), "N": 300, "E": E, "D": 12, "H": H, "R_grad": R, "sampler": "step-wise"}))
    dyn, stationary, scheduled, terms, m0 = problem(H=H, R=R)
    graphs = {}
    for P in (1024, 16384):
        rng = np.random.RandomState(P)
        x0, eps = m0[None] + 0.1 * rng.randn(P, E), rng.randn(P, H, E)
        for arm, spec in (("stationary", stationary), ("scheduled", scheduled)):
            for what, grad in (("forward", False), ("forward_grad", True)):
                graphs[(P, arm, what)] = captured(dyn, spec, terms, x0, eps, R, grad, arm == "scheduled")
    torch.cuda.synchronize()
    for rnd in range(args.rounds):
        row = {"round": rnd}
        for P in (1024, 16384):
            for what in ("forward", "forward_grad"):
                for arm in ("stationary", "scheduled"):      # alternated
                    row["P%d_%s_ms_%s" % (P, what, arm)] = round(time_graph(graphs[(P, arm, what)][1], args.reps), 4)
        print(json.dumps(row))
    graphs.clear()
    torch.cuda.empty_cache()
    pilco, x = pendulum_pilco()
    print(json.dumps({"plan_H": 10, "plan_R": 8, "maxiter": 10, "num_samples": 256,
                      "plan_wall_s_median_sampled": plan_time(pilco, x, args.plans, num_samples=256),
                      "plan_wall_s_median_moment_matching": plan_time(pilco, x, args.plans)}))


if __name__ == "__main__":
    main()
