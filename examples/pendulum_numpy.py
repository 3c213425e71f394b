"""Gym-free end-to-end PILCO loop on a damped torque-limited pendulum simulated in numpy.

Same outer structure as the reference's example scripts (examples/inverted_pendulum.py:15-39,
examples/utils.py:7-36): collect (x,u)->dx data with random actions, then iterate
  optimize_models -> optimize_policy (batched restarts on the device) -> rollout with the learnt policy ->
  append data -> set_data.
The environment is a stand-in for gym/mujoco (not installable offline); everything from ``pilco`` is the
H100-native engine.  Usage:  python examples/pendulum_numpy.py [--iters 3]"""
import argparse
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from pilco.models import PILCO                      # noqa: E402
from pilco.controllers import RbfController         # noqa: E402
from pilco.rewards import ExponentialReward         # noqa: E402


class PendulumEnv:
    """theta'' = -g/l sin(theta) - b theta' + u/(m l^2); state x = (theta, theta'); theta = 0 hangs down."""

    def __init__(self, dt=0.1, max_torque=2.0, seed=0):
        self.dt, self.max_torque = dt, max_torque
        self.rng = np.random.RandomState(seed)
        self.x = None

    def reset(self):
        self.x = np.array([0.1 * self.rng.randn(), 0.1 * self.rng.randn()])
        return self.x.copy()

    def step(self, u):
        u = float(np.clip(u, -self.max_torque, self.max_torque))
        th, om = self.x
        for _ in range(5):                                   # semi-implicit Euler sub-steps
            om += self.dt / 5 * (-9.81 * np.sin(th) - 0.2 * om + u)
            th += self.dt / 5 * om
        self.x = np.array([th, om])
        return self.x.copy()

    def sample_action(self):
        return self.rng.uniform(-self.max_torque, self.max_torque, size=1)


def rollout(env, policy, timesteps):
    """(x,u) -> dx pairs of one episode (examples/utils.py:7-29)."""
    X, Y = [], []
    x = env.reset()
    for _ in range(timesteps):
        u = policy(x)
        x_new = env.step(u[0])
        X.append(np.hstack((x, u)))
        Y.append(x_new - x)
        x = x_new
    return np.stack(X), np.stack(Y)


def run(iters=3, T=25, restarts=4, maxiter=20, bf=10, verbose=True, seed=0, action_cost=0.0):
    np.random.seed(seed)
    env = PendulumEnv(seed=seed)
    X, Y = rollout(env, lambda x: env.sample_action(), T)
    for _ in range(2):
        X_, Y_ = rollout(env, lambda x: env.sample_action(), T)
        X, Y = np.vstack((X, X_)), np.vstack((Y, Y_))
    state_dim, control_dim = 2, 1
    controller = RbfController(state_dim, control_dim, bf, max_action=env.max_torque)
    reward = ExponentialReward(state_dim, W=np.diag([1.0, 0.1]), t=np.array([np.pi / 3, 0.0]))   # swing to 60 degrees
    if action_cost:       # a torque cost action_cost (1 - exp(-u^2 / 2)) beside the swing-up reward (a reward on [x, u])
        from pilco.rewards import CombinedRewards, action_cost as effort
        reward = CombinedRewards(state_dim, [reward, effort(state_dim, control_dim, [[1.0]])], coefs=[1.0, action_cost])
    pilco = PILCO((X, Y), controller=controller, horizon=T, reward=reward,
                  m_init=np.zeros((1, state_dim)), S_init=np.diag([0.01, 0.01]))
    history = []
    for it in range(iters):
        pilco.optimize_models(restarts=1)
        pilco.optimize_policy(maxiter=maxiter, restarts=restarts)
        predicted = float(np.asarray(pilco.compute_reward()).item())
        X_, Y_ = rollout(env, lambda x: pilco.compute_action(x[None, :])[0, :], T)
        achieved = float(np.exp(-0.5 * ((X_[:, 0] + Y_[:, 0] - np.pi / 3) ** 2 + 0.1 * (X_[:, 1] + Y_[:, 1]) ** 2)).sum())
        history.append((predicted, achieved))
        if verbose:
            print("iteration %d: predicted reward %.3f, achieved reward %.3f, N=%d" % (it, predicted, achieved, len(X)))
        X, Y = np.vstack((X, X_)), np.vstack((Y, Y_))
        pilco.mgpr.set_data((X, Y))
    return history


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=3)
    ap.add_argument("--action-cost", type=float, default=0.0, help="weight of a saturating torque cost (0: none)")
    a = ap.parse_args()
    run(iters=a.iters, action_cost=a.action_cost)
