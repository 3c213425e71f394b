"""Gym-free trajectory-sampling MPC with the cross-entropy method (PETS, Chua et al. 2018) on the damped torque-limited
pendulum of examples/pendulum_numpy.py, swinging it to 60 degrees: a few episodes of random torques train the dynamics
GPs (optimize_models) on the angle's sin / cos features (``angle_dims=[0]``), then at every control step
``PILCO.plan(x, num_samples=20, optimizer="cem", maxiter=5, seed=t)`` searches open-loop torque sequences
(TimeVaryingLinearController(feedback=False)) on the mean return of 20 particle rollouts of the learnt dynamics, every
CEM iteration on the device, applies the first torque and keeps the rest of the best sequence as the next step's warm
start.  Usage:
    python examples/pendulum_cem_numpy.py [--episodes 2] [--steps 25] [--population 400] [--elites 40]"""
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


def run(episodes=2, T=25, horizon=10, random_episodes=3, random_steps=25, population=400, elites=40, iters=5,
        num_samples=20, verbose=True, seed=0):
    """-> (the returns of the random episodes, the returns of the MPC episodes): sum over the T steps of
    exp(-((theta - pi/3)^2 + 0.1 omega^2) / 2) at the states reached; the random episodes take ``random_steps``"""
    np.random.seed(seed)
    env = PendulumEnv(seed=seed)
    X, Y, random_returns = [], [], []
    for _ in range(random_episodes):
        X_, Y_ = rollout(env, lambda x: env.sample_action(), random_steps)
        X.append(X_); Y.append(Y_)
        random_returns.append(sum(task_reward(x) for x in X_[:, :2] + Y_))
    X, Y = np.vstack(X), np.vstack(Y)
    state_dim, control_dim = 2, 1
    controller = TimeVaryingLinearController(state_dim + 1, control_dim, horizon, max_action=env.max_torque,
                                             feedback=False)
    reward = ExponentialReward(state_dim, W=np.diag([1.0, 0.1]), t=TARGET)
    pilco = PILCO((X, Y), controller=controller, horizon=horizon, reward=reward, m_init=np.zeros((1, state_dim)),
                  S_init=np.diag([0.01, 0.01]), angle_dims=[0])
    pilco.optimize_models(restarts=1)
    mpc_returns = []
    for ep in range(episodes):
        x, ret, Xe, Ye = env.reset(), 0.0, [], []
        for t in range(T):
            u = np.asarray(pilco.plan(x, num_samples=num_samples, optimizer="cem", maxiter=iters, seed=t,
                                      population=population, elites=elites)).reshape(control_dim)
            x_new = env.step(u[0])
            Xe.append(np.hstack((x, u))); Ye.append(x_new - x)
            ret += task_reward(x_new)
            x = x_new
        mpc_returns.append(ret)
        if verbose:
            print("CEM-MPC episode %d: return %.3f over %d steps, last plan's in-sample value %.3f (random episodes: %s)"
                  % (ep, ret, T, float(pilco.cem_plan.best_value[0]), np.round(random_returns, 3)))
        X, Y = np.vstack((X, np.stack(Xe))), np.vstack((Y, np.stack(Ye)))
        pilco.set_data((X, Y))
        pilco.optimize_models(restarts=1)
    return random_returns, mpc_returns


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--episodes", type=int, default=2)
    ap.add_argument("--steps", type=int, default=25, help="control steps per episode")
    ap.add_argument("--population", type=int, default=400)
    ap.add_argument("--elites", type=int, default=40)
    a = ap.parse_args()
    run(episodes=a.episodes, T=a.steps, population=a.population, elites=a.elites)
