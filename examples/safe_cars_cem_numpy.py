"""Gym-free SafePILCO on the two-car crossing of examples/safe_cars_numpy.py, with a stationary linear policy trained
on the sampled return by the cross-entropy method (DESIGN.md section 33): the same SafePILCO reward, an additive
LinearReward for progress and a multiplicative RiskOfCollision for both cars inside the junction, but
``optimize_policy_sampled(optimizer="cem")`` in place of the moment-matching ``optimize_policy``.  The risk term is a
box indicator with no pathwise gradient, so the gradient-based sampled optimisers refuse it; CEM needs only the
candidates' values.  Each iteration trains the dynamics GPs, searches ``population`` candidate policies over
``num_samples`` particles for ``maxiter`` iterations on the device (one CUDA graph), runs the policy on the cars and
adds the episode to the data.  Usage:
    python examples/safe_cars_cem_numpy.py [--iters 3] [--maxiter 10] [--population 400] [--num-samples 256]"""
import argparse
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from pilco.controllers import LinearController                                 # noqa: E402
from pilco.rewards import LinearReward                                         # noqa: E402
from safe_pilco_extension.rewards_safe import RiskOfCollision                  # noqa: E402
from safe_pilco_extension.safe_pilco import SafePILCO                          # noqa: E402
from safe_cars_numpy import TwoCars, rollout                                   # noqa: E402


def run(N=3, T=25, J=4, maxiter=10, population=400, elites=40, num_samples=256, mu=-300.0, verbose=True, seed=0):
    """-> the in-sample value of the policy CEM chose at each of the N iterations"""
    np.random.seed(seed)
    env = TwoCars(seed=seed)
    rand = lambda x: env.sample_action()
    probe = np.vstack([rollout(env, rand, T)[0] for _ in range(3)])
    mean, std = probe[:, :4].mean(0), probe[:, :4].std(0)
    trans = lambda x: (x - mean) / std
    X, Y, _ = rollout(env, rand, T, trans)
    for _ in range(1, J):
        X_, Y_, _ = rollout(env, rand, T, trans)
        X, Y = np.vstack((X, X_)), np.vstack((Y, Y_))
    state_dim, control_dim = 4, 1
    controller = LinearController(state_dim, control_dim, max_action=0.2)
    progress = LinearReward(state_dim, np.array([std[0], 0.0, 0.0, 0.0]))        # raw position of car 1
    b1, b2 = 1.0 / std[0], 1.0 / std[2]                                       # junction: |p| < 1 in raw units
    risk = RiskOfCollision(2, [-b1 - mean[0] / std[0], -b2 - mean[2] / std[2]], [b1 - mean[0] / std[0], b2 - mean[2] / std[2]])
    pilco = SafePILCO((X, Y), controller=controller, mu=mu, reward_add=progress, reward_mult=risk, horizon=T,
                      m_init=X[0:1, :state_dim], S_init=0.1 * np.eye(state_dim))
    for model in pilco.mgpr.models:
        model.likelihood.variance.assign(0.001)
        model.likelihood.variance.trainable = False
    values = []
    for it in range(N):
        pilco.optimize_models(maxiter=100)
        v = pilco.optimize_policy_sampled(optimizer="cem", maxiter=maxiter, population=population, elites=elites,
                                          num_samples=num_samples, seed=it)
        values.append(v)
        X_, Y_, raw = rollout(env, lambda x: pilco.compute_action(x[None, :])[0, :], T, trans)
        collided = bool(np.any((np.abs(raw[:, 0]) < 1.0) & (np.abs(raw[:, 2]) < 1.0)))
        if verbose:
            trace = pilco.cem_search.trace.cpu().numpy()
            print("iteration %d: in-sample value %.3f (top value per CEM iteration %s), final position %.2f, "
                  "collided=%s" % (it, v, np.round(trace[:, 0], 3), raw[-1, 0], collided))
        X, Y = np.vstack((X, X_)), np.vstack((Y, Y_))
        pilco.mgpr.set_data((X, Y))
    return values


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=3)
    ap.add_argument("--maxiter", type=int, default=10, help="CEM iterations per policy search")
    ap.add_argument("--population", type=int, default=400)
    ap.add_argument("--num-samples", type=int, default=256, help="particles of the sampled return")
    a = ap.parse_args()
    run(N=a.iters, maxiter=a.maxiter, population=a.population, num_samples=a.num_samples)
