"""Gym-free safe-PILCO loop on a two-car crossing: the controlled car must make progress along its lane without
being inside the junction while the other car is (the scenario of the reference's examples/safe_cars_run.py with
its pure-numpy linear environment; gym itself is not installable offline).

Outer structure of examples/safe_cars_run.py:43-139: random rollouts -> state normalisation -> SafePILCO with an
additive LinearReward (progress) and a multiplicative RiskOfCollision (both cars inside the junction box) ->
per iteration: optimize_models, optimize_policy, predicted per-step risks along the planned trajectory
(``pilco.predict`` for every prefix + ``RiskOfCollision.compute_reward``), act with ``compute_action`` only when the
predicted overall risk is below the threshold, adapt ``mu``.  Everything imported from ``pilco`` /
``safe_pilco_extension`` is the H100-native engine.  Usage:  python examples/safe_cars_numpy.py [--iters 3]"""
import argparse
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from pilco.controllers import RbfController                                    # noqa: E402
from pilco.rewards import LinearReward                                         # noqa: E402
from safe_pilco_extension.rewards_safe import RiskOfCollision                  # noqa: E402
from safe_pilco_extension.safe_pilco import SafePILCO                          # noqa: E402


class TwoCars:
    """State (p1, v1, p2, v2): positions/velocities of two cars approaching a junction at p = 0 on crossing
    lanes.  The action is the force on car 1 (unit mass, slight viscous friction); car 2 coasts.  Explicit Euler
    with a 0.5 s step, i.e. a linear time-invariant system x' = x + A x + B u."""

    def __init__(self, dt=0.5, friction=1e-3, max_force=0.4, seed=0):
        self.dt, self.max_force = dt, max_force
        self.A = np.zeros((4, 4))
        self.A[0, 1] = dt
        self.A[1, 1] = -friction * dt
        self.A[2, 3] = dt
        self.B = np.array([0.0, dt, 0.0, 0.0])
        self.x0 = np.array([-6.0, 1.0, -5.0, 1.0])
        self.rng = np.random.RandomState(seed)
        self.x = None

    def reset(self):
        self.x = self.x0 + 0.03 * self.rng.randn(4)
        return self.x.copy()

    def step(self, u):
        u = float(np.clip(u, -self.max_force, self.max_force))
        self.x = self.x + self.A @ self.x + self.B * u
        return self.x.copy()

    def sample_action(self):
        return self.rng.uniform(-self.max_force, self.max_force, size=1)


def rollout(env, policy, timesteps, trans=lambda x: x):
    """(x,u) -> dx pairs of one episode in (optionally normalised) coordinates (examples/utils.py:7-29)."""
    X, Y, raw = [], [], []
    x = trans(env.reset())
    for _ in range(timesteps):
        u = policy(x)
        raw_new = env.step(u[0])
        x_new = trans(raw_new)
        X.append(np.hstack((x, u)))
        Y.append(x_new - x)
        raw.append(raw_new)
        x = x_new
    return np.stack(X), np.stack(Y), np.stack(raw)


def run(iters=3, T=25, J=4, restarts=2, maxiter=20, bf=20, th=0.10, mu=-300.0, verbose=True, seed=0):
    np.random.seed(seed)
    env = TwoCars(seed=seed)
    rand = lambda x: env.sample_action()
    probe = np.vstack([rollout(env, rand, T)[0] for _ in range(3)])
    mean, std = probe[:, :4].mean(0), probe[:, :4].std(0)
    trans = lambda x: (x - mean) / std                                        # safe_cars_run.py:20-41
    X, Y, _ = rollout(env, rand, T, trans)
    for _ in range(1, J):
        X_, Y_, _ = rollout(env, rand, T, trans)
        X, Y = np.vstack((X, X_)), np.vstack((Y, Y_))
    state_dim, control_dim = 4, 1
    m_init = X[0:1, :state_dim]
    S_init = 0.1 * np.eye(state_dim)
    controller = RbfController(state_dim, control_dim, bf, max_action=0.2)
    progress = LinearReward(state_dim, np.array([std[0], 0.0, 0.0, 0.0]))        # raw position of car 1
    b1, b2 = 1.0 / std[0], 1.0 / std[2]                                       # junction: |p| < 1 in raw units
    risk = RiskOfCollision(2, [-b1 - mean[0] / std[0], -b2 - mean[2] / std[2]], [b1 - mean[0] / std[0], b2 - mean[2] / std[2]])
    pilco = SafePILCO((X, Y), controller=controller, mu=mu, reward_add=progress, reward_mult=risk, horizon=T,
                      m_init=m_init, S_init=S_init)
    for model in pilco.mgpr.models:
        model.likelihood.variance.assign(0.001)
        model.likelihood.variance.trainable = False
    history = []
    for it in range(iters):
        pilco.optimize_models(maxiter=100)
        pilco.optimize_policy(maxiter=maxiter, restarts=restarts)
        risks = np.zeros(T)
        for h in range(T):                                                    # safe_cars_run.py:107-112
            m_h, S_h, _ = pilco.predict(m_init, S_init, h)
            risks[h] = float(np.asarray(risk.compute_reward(m_h, S_h)[0]))
        overall = 1.0 - np.prod(1.0 - risks)
        objective = float(np.asarray(pilco.compute_reward()).item())
        X_, Y_, raw = rollout(env, lambda x: pilco.compute_action(x[None, :])[0, :], T, trans)
        collided = bool(np.any((np.abs(raw[:, 0]) < 1.0) & (np.abs(raw[:, 2]) < 1.0)))
        history.append(dict(overall_risk=float(overall), objective=objective, collided=collided,
                            progress=float(raw[-1, 0]), mu=float(pilco.mu.numpy())))
        if verbose:
            print("iteration %d: predicted overall risk %.4f, objective %.2f, final position %.2f, collided=%s, mu=%.1f"
                  % (it, overall, objective, raw[-1, 0], collided, float(pilco.mu.numpy())))
        X, Y = np.vstack((X, X_)), np.vstack((Y, Y_))
        pilco.mgpr.set_data((X, Y))
        if overall < th / 4:
            pilco.mu.assign(0.75 * pilco.mu.numpy())                          # safe_cars_run.py:126-127
        elif overall >= th:
            pilco.mu.assign(1.5 * pilco.mu.numpy())                           # safe_cars_run.py:137
    return history


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=3)
    a = ap.parse_args()
    run(iters=a.iters)
