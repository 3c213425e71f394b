"""Pendulum swing-up to theta = pi with the angle as a periodic input (PILCO's trigonometric augmentation).

The state stays the raw (theta, theta'); ``PILCO(..., angle_dims=[0])`` hands the policy and the dynamics GPs
phi(x) = [theta', sin theta, cos theta], so a policy that sees theta = pi + 2 pi sees the point it has learnt.  The
target "pendulum up" is a reward on the joint [phi(x), u]: exp(-1/2 |(sin theta, cos theta) - (0, -1)|^2_W), which is
the same for every theta = pi + 2 pi k.  Usage:  python examples/pendulum_angles_numpy.py [--iters 3]"""
import argparse
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from pilco.models import PILCO                                  # noqa: E402
from pilco.controllers import RbfController                     # noqa: E402
from pilco.rewards import ExponentialStateActionReward          # noqa: E402
from pendulum_numpy import PendulumEnv, rollout                 # noqa: E402


def swing_up_reward(U=1):
    """periodic target on [theta', sin theta, cos theta, u]: (0, 0, -1), the action free"""
    Dh = 3
    W = np.diag([0.05, 1.0, 1.0, 0.0])
    t = np.array([0.0, 0.0, -1.0, 0.0])
    return ExponentialStateActionReward(Dh, U, W=W, t=t)


def make_pilco(T=25, bf=10, seed=0, episodes=3):
    """random-action episodes -> (env, PILCO with angle_dims=[0], raw X = [x, u], raw Y = delta x)"""
    np.random.seed(seed)
    env = PendulumEnv(max_torque=3.0, seed=seed)
    X, Y = rollout(env, lambda x: env.sample_action(), T)
    for _ in range(episodes - 1):
        X_, Y_ = rollout(env, lambda x: env.sample_action(), T)
        X, Y = np.vstack((X, X_)), np.vstack((Y, Y_))
    controller = RbfController(3, 1, bf, max_action=env.max_torque)      # sees phi(x) = [theta', sin, cos]: Dh = 3
    pilco = PILCO((X, Y), controller=controller, horizon=T, reward=swing_up_reward(),
                  m_init=np.zeros((1, 2)), S_init=np.diag([0.01, 0.01]), angle_dims=[0])
    return env, pilco, X, Y


def run(iters=3, T=25, restarts=4, maxiter=20, bf=10, verbose=True, seed=0):
    env, pilco, X, Y = make_pilco(T, bf, seed)
    history = []
    for it in range(iters):
        pilco.optimize_models(restarts=1)
        pilco.optimize_policy(maxiter=maxiter, restarts=restarts)
        predicted = float(np.asarray(pilco.compute_reward()).item())
        X_, Y_ = rollout(env, lambda x: pilco.compute_action(x[None, :])[0, :], T)
        th, om = X_[:, 0] + Y_[:, 0], X_[:, 1] + Y_[:, 1]
        achieved = float(np.exp(-0.5 * (np.sin(th) ** 2 + (np.cos(th) + 1.0) ** 2 + 0.05 * om ** 2)).sum())
        history.append((predicted, achieved))
        if verbose:
            print("iteration %d: predicted reward %.3f, achieved reward %.3f, N=%d" % (it, predicted, achieved, len(X)))
        X, Y = np.vstack((X, X_)), np.vstack((Y, Y_))
        pilco.set_data((X, Y))                     # raw data: PILCO applies phi (angle deltas are unwrapped)
    return history


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=3)
    a = ap.parse_args()
    run(iters=a.iters)
