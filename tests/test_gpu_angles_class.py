"""GPU tests of PILCO(angle_dims=...): predict against H propagates, compute_action against the RBF mean at phi(x)
and its periodicity, the captured predict graph against an eager rollout, policy_gradient against central
differences of predict, and optimize_policy raising the moment-matching reward on the swing-up example."""
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "examples"))


@pytest.fixture(scope="module")
def swing():
    import pendulum_angles_numpy as ex
    env, pilco, X, Y = ex.make_pilco(T=15, bf=8, seed=1)
    pilco.optimize_models(restarts=1)
    return pilco


def test_predict_equals_repeated_propagate(swing):
    p = swing
    m, S = np.array([[0.3, -0.2]]), np.diag([0.02, 0.03])
    Mn, Sn, _ = p.predict(m, S, 6)
    mt, St = m, S
    for _ in range(6):
        mt, St = p.propagate(mt, St)
    assert np.max(np.abs(np.asarray(Mn) - np.asarray(mt))) <= 1e-10 * max(1.0, np.max(np.abs(Mn)))
    assert np.max(np.abs(np.asarray(Sn) - np.asarray(St))) <= 1e-10 * np.max(np.abs(Sn))


def test_predict_graph_equals_eager_rollout(swing):
    p = swing
    m, S = np.array([[0.1, 0.4]]), np.diag([0.01, 0.02])
    Mn, Sn, rew = p.predict(m, S, 8)
    plan = p.rollout_plan(m, S, 8)
    tm, tS, r = plan.forward()
    torch.cuda.synchronize()
    assert np.array_equal(np.asarray(Mn)[0], tm[0, -1].cpu().numpy())
    assert np.array_equal(np.asarray(Sn), tS[0, -1].cpu().numpy())
    assert float(np.asarray(rew).item()) == float(r[0])


def test_compute_action_is_rbf_mean_at_phi(swing):
    from oracle import torch_port as tp
    from pilco_b200 import engine
    p = swing
    c = p.controller
    X, Y, th = c.split_flat(c.get_flat()[None])
    ell = c.models[0].kernel.lengthscales.transform.forward(th)
    T = lambda a: torch.tensor(np.asarray(a), dtype=torch.float64)
    for x in (np.array([0.4, -1.0]), np.array([3.0, 0.5]), np.array([-2.5, 2.0])):
        phi = engine.trig_feature_map(x[None], [0])
        M, _, _ = tp.rbf_action(T(X[0]), T(Y[0]), T(ell[0]), T(phi), torch.zeros((3, 3), dtype=torch.float64),
                                T(np.atleast_1d(c.max_action))[None])
        u = np.asarray(p.compute_action(x[None]))
        assert np.max(np.abs(u - M.numpy())) < 1e-9 * max(1.0, np.max(np.abs(u)))
        u2 = np.asarray(p.compute_action((x + np.array([2 * np.pi, 0.0]))[None]))
        assert np.max(np.abs(u2 - u)) < 1e-12 * max(1.0, np.max(np.abs(u)))


def test_policy_gradient_matches_central_differences(swing):
    p = swing
    c = p.controller
    flat0 = np.array(c.get_flat(), copy=True)
    val, grad = p.policy_gradient()
    # policy_gradient runs the taped tile pass, predict the plain one: their sums run in different orders
    assert abs(val - float(np.asarray(p.compute_reward()).item())) < 1e-9 * max(1.0, abs(val))
    # compute_reward replays the plain tile pass, whose table exponential leaves a noise floor near 1e-10 on the
    # reward (the same without angles): a step of 1e-4 keeps the difference quotient above it, at a truncation
    # error of about 1e-3 of the gradient's scale
    h = 1e-4
    try:
        for i in (0, 1, 5, len(flat0) // 2, len(flat0) - 1):
            vals = []
            for sgn in (1, -1):
                f = flat0.copy()
                f[i] += sgn * h
                c.set_flat(f)
                vals.append(float(np.asarray(p.compute_reward()).item()))
            fd = (vals[0] - vals[1]) / (2 * h)
            assert abs(fd - grad[i]) < 2e-3 * np.max(np.abs(grad)), (i, fd, grad[i])
    finally:
        c.set_flat(flat0)


def test_optimize_policy_raises_the_reward():
    import pendulum_angles_numpy as ex
    env, p, X, Y = ex.make_pilco(T=15, bf=8, seed=2)
    p.optimize_models(restarts=1)
    r0 = float(np.asarray(p.compute_reward()).item())
    p.optimize_policy(maxiter=15, restarts=8)
    r1 = float(np.asarray(p.compute_reward()).item())
    assert r1 > r0
