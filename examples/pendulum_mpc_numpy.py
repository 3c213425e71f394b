"""Gym-free probabilistic MPC (Kamthe & Deisenroth, AISTATS 2018) on the damped torque-limited pendulum of
examples/pendulum_numpy.py: a few episodes of random torques train the dynamics GPs (optimize_models), then at every
control step ``PILCO.plan`` optimises a torque sequence (TimeVaryingLinearController(feedback=False)) over the horizon
through the moment-matching cascade from the measured state, applies its first action and keeps the rest as the next
step's warm start.  No global policy is learnt.  ``--num-samples S`` plans on the mean return of S particle rollouts
of the learnt dynamics instead of the moment-matching cascade (``PILCO.plan(num_samples=S)``).  Usage:
    python examples/pendulum_mpc_numpy.py [--episodes 2] [--angles] [--num-samples 256]"""
import argparse
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from pilco.models import PILCO                                   # noqa: E402
from pilco.controllers import TimeVaryingLinearController        # noqa: E402
from pilco.rewards import ExponentialReward                      # noqa: E402
from pendulum_numpy import PendulumEnv, rollout                  # noqa: E402

TARGET = np.array([np.pi / 3, 0.0])                              # swing to 60 degrees and hold


def task_reward(x):
    return float(np.exp(-0.5 * ((x[0] - TARGET[0]) ** 2 + 0.1 * x[1] ** 2)))


def run(episodes=2, T=25, horizon=10, random_episodes=3, restarts=2, maxiter=10, angles=False, verbose=True, seed=0,
        num_samples=None):
    """-> (the returns of the random episodes, the returns of the MPC episodes): sum over the T steps of
    exp(-((theta - pi/3)^2 + 0.1 omega^2) / 2) at the states reached.  ``num_samples``: plan on that many particles
    (seeded per control step), or None for the moment-matching plan"""
    np.random.seed(seed)
    env = PendulumEnv(seed=seed)
    X, Y, random_returns = [], [], []
    for _ in range(random_episodes):
        X_, Y_ = rollout(env, lambda x: env.sample_action(), T)
        X.append(X_); Y.append(Y_)
        random_returns.append(sum(task_reward(x) for x in X_[:, :2] + Y_))
    X, Y = np.vstack(X), np.vstack(Y)
    state_dim, control_dim = 2, 1
    controller = TimeVaryingLinearController(state_dim + (1 if angles else 0), control_dim, horizon,
                                             max_action=env.max_torque, feedback=False)
    reward = ExponentialReward(state_dim, W=np.diag([1.0, 0.1]), t=TARGET)
    pilco = PILCO((X, Y), controller=controller, horizon=horizon, reward=reward, m_init=np.zeros((1, state_dim)),
                  S_init=np.diag([0.01, 0.01]), angle_dims=[0] if angles else None)
    pilco.optimize_models(restarts=1)
    mpc_returns = []
    for ep in range(episodes):
        x, ret, Xe, Ye = env.reset(), 0.0, [], []
        for k in range(T):
            sampled = {} if num_samples is None else dict(num_samples=num_samples, seed=seed + 1000 * ep + k)
            u = np.asarray(pilco.plan(x, maxiter=maxiter, restarts=restarts, **sampled)).reshape(control_dim)
            x_new = env.step(u[0])
            Xe.append(np.hstack((x, u))); Ye.append(x_new - x)
            ret += task_reward(x_new)
            x = x_new
        mpc_returns.append(ret)
        if verbose:
            print("MPC episode %d: return %.3f (random episodes: %s)" % (ep, ret, np.round(random_returns, 3)))
        X, Y = np.vstack((X, np.stack(Xe))), np.vstack((Y, np.stack(Ye)))
        pilco.set_data((X, Y))
        pilco.optimize_models(restarts=1)
    return random_returns, mpc_returns


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--episodes", type=int, default=2)
    ap.add_argument("--angles", action="store_true", help="treat theta as an angle (sin / cos features)")
    ap.add_argument("--num-samples", type=int, default=None, help="plan on the mean return of this many particles")
    a = ap.parse_args()
    run(episodes=a.episodes, angles=a.angles, num_samples=a.num_samples)
