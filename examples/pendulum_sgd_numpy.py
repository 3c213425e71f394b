"""Gym-free policy search with Adam on fresh particles (Deep PILCO's training loop; DESIGN.md section 32) on the damped
torque-limited pendulum of examples/pendulum_numpy.py, swinging it to 60 degrees: a few episodes of random torques
train the dynamics GPs (optimize_models), then each episode trains a tanh MLP policy (MlpController, 2 x 32) by
``PILCO.optimize_policy_sampled(optimizer="adam")``: every Adam step draws ``num_samples`` new particle rollouts of the
learnt dynamics on the device, and the whole run is one CUDA graph replayed ``maxiter`` times.  The policy then runs
on the pendulum, and its episode joins the data.  Usage:
    python examples/pendulum_sgd_numpy.py [--episodes 3] [--steps 30] [--maxiter 300] [--num-samples 256]"""
import argparse
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from pilco.models import PILCO                                   # noqa: E402
from pilco.controllers import MlpController                      # noqa: E402
from pilco.rewards import ExponentialReward                      # noqa: E402
from pendulum_numpy import PendulumEnv, rollout                  # noqa: E402

TARGET = np.array([np.pi / 3, 0.0])                              # swing to 60 degrees and hold


def task_reward(x):
    return float(np.exp(-0.5 * ((x[0] - TARGET[0]) ** 2 + 0.1 * x[1] ** 2)))


def run(episodes=3, T=30, horizon=30, random_episodes=3, maxiter=300, num_samples=256, restarts=2,
        learning_rate=1e-2, verbose=True, seed=0):
    """-> (the returns of the random episodes, the returns of the policy's episodes): sum over the T steps of
    exp(-((theta - pi/3)^2 + 0.1 omega^2) / 2) at the states reached"""
    np.random.seed(seed)
    env = PendulumEnv(seed=seed)
    X, Y, random_returns = [], [], []
    for _ in range(random_episodes):
        X_, Y_ = rollout(env, lambda x: env.sample_action(), T)
        X.append(X_); Y.append(Y_)
        random_returns.append(sum(task_reward(x) for x in X_[:, :2] + Y_))
    X, Y = np.vstack(X), np.vstack(Y)
    state_dim, control_dim = 2, 1
    controller = MlpController(state_dim, control_dim, hidden=(32, 32), max_action=env.max_torque)
    reward = ExponentialReward(state_dim, W=np.diag([1.0, 0.1]), t=TARGET)
    pilco = PILCO((X, Y), controller=controller, horizon=horizon, reward=reward, m_init=np.zeros((1, state_dim)),
                  S_init=np.diag([0.01, 0.01]))
    returns = []
    for ep in range(episodes):
        pilco.optimize_models(restarts=1)
        held_out = pilco.optimize_policy_sampled(optimizer="adam", maxiter=maxiter, restarts=restarts,
                                                 num_samples=num_samples, learning_rate=learning_rate, seed=ep)
        X_, Y_ = rollout(env, lambda x: np.asarray(pilco.compute_action(x[None])).reshape(control_dim), T)
        ret = sum(task_reward(x) for x in X_[:, :2] + Y_)
        returns.append(ret)
        if verbose:
            last = np.asarray(pilco.adam_trace.value[-1])
            print("Adam episode %d: return %.3f over %d steps; held-out value %.3f, last step's in-sample values %s "
                  "(random episodes: %s)" % (ep, ret, T, held_out, np.round(last, 3), np.round(random_returns, 3)))
        X, Y = np.vstack((X, X_)), np.vstack((Y, Y_))
        pilco.set_data((X, Y))
    return random_returns, returns


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--episodes", type=int, default=3)
    ap.add_argument("--steps", type=int, default=30, help="control steps per episode (and the horizon)")
    ap.add_argument("--maxiter", type=int, default=300, help="Adam steps per episode")
    ap.add_argument("--num-samples", type=int, default=256, help="particles drawn afresh at every Adam step")
    a = ap.parse_args()
    run(episodes=a.episodes, T=a.steps, horizon=a.steps, maxiter=a.maxiter, num_samples=a.num_samples)
