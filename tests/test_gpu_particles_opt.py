"""Policy optimisation on the sampled return (pilco_particles_rollout_batch_grad through engine.ParticlePlan(R=...),
policy_opt.ParticleEvaluator and PILCO.optimize_policy_sampled): every restart of a batched call bitwise equal to the
unbatched call with that restart's policy, bitwise reproducibility and CUDA-graph replay, the evaluator against
sample_policy_gradient and a directional central difference, and the optimiser end to end."""
from functools import partial

import numpy as np
import pytest
import torch

from pilco_b200 import engine, _lib, policy_opt
from particle_cases import _batch_case, _draw, _pilco, _pilco_data

pytestmark = pytest.mark.gpu


def _grad_run(gp, spec, terms, x0, eps, mu, R=1):
    plan = engine.ParticlePlan(gp, spec, terms, x0.shape[0], eps.shape[1], mult_mu=mu, grad=True, R=R)
    plan.set_inputs(x0, eps)
    g = {k: v.clone() for k, v in plan.launch_grad().items()}
    return plan, g, [t.clone() for t in plan.outputs()]


@pytest.mark.parametrize("kind,R", [("rbf", 1), ("rbf", 3), ("rbf", 5), ("linear", 3), ("linear", 5), ("fitc", 3)])
def test_batched_restarts_bitwise_equal_unbatched(kind, R):
    gp, spec, singles, terms, m0, S0, H, P, mu = _batch_case(kind, R)
    assert P % 128 and H >= 3
    x0, eps = _draw(m0, S0, P, H, seed=34)
    plan, g, out = _grad_run(gp, spec, terms, x0, eps, mu, R=R)
    assert g["value"].shape == (R,) and out[0].shape == (R, P, H + 1, spec["Ds"])
    for r in range(R):
        _, g1, out1 = _grad_run(gp, singles[r], terms, x0, eps, mu)
        for what, a, b in zip(("traj", "act", "step_reward", "step_risk", "ret"), out, out1):
            assert torch.equal(a[r], b), (r, what)
        for k in g1:
            assert torch.equal(g[k][r], g1[k].reshape(g[k][r].shape)), (r, k)
    assert len(set(float(v) for v in g["value"])) == R           # the restarts are different policies


def test_shared_policy_array_with_zero_stride():
    gp, spec, singles, terms, m0, S0, H, P, mu = _batch_case("linear", 3)
    x0, eps = _draw(m0, S0, P, H, seed=35)
    plan = engine.ParticlePlan(gp, spec, terms, P, H, mult_mu=mu, grad=True, R=3)
    plan.set_inputs(x0, eps)
    plan.pr.pol.b_bs = 0                                         # every restart uses b[0]
    g = plan.launch_grad()
    for r in range(3):
        _, g1, out1 = _grad_run(gp, dict(singles[r], b=spec["b"][0]), terms, x0, eps, mu)
        assert torch.equal(plan.ret[r], out1[4]) and torch.equal(g["W"][r], g1["W"])


def test_batched_call_is_reproducible_and_replays():
    gp, spec, _, terms, m0, S0, H, P, mu = _batch_case("rbf", 3)
    x0, eps = _draw(m0, S0, P, H, seed=36)
    plan, first, out = _grad_run(gp, spec, terms, x0, eps, mu, R=3)
    second = {k: v.clone() for k, v in plan.launch_grad().items()}
    assert all(torch.equal(first[k], second[k]) for k in first)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        plan.launch_grad()
    for v in list(plan.gbuf.values()) + [plan.traj, plan.ret]:
        v.zero_()
    graph.replay()
    torch.cuda.synchronize()
    assert all(torch.equal(first[k], plan.gbuf[k]) for k in first)
    assert torch.equal(out[0], plan.traj) and torch.equal(out[4], plan.ret)


@pytest.mark.parametrize("kind", ["rbf", "linear"])
def test_evaluator_is_the_sampled_objective(kind):
    pilco, _, _ = _pilco(kind, 40)
    P, seed = 300, 11
    c = pilco.controller
    f = policy_opt.initial_flats(c, 2)[1]
    x0, eps = pilco._particle_inputs(pilco.m_init, pilco.S_init, pilco.horizon, P, seed, "test")
    v = np.random.RandomState(41).randn(f.size)
    h = 1e-5
    ev = policy_opt.ParticleEvaluator(pilco, 3, x0, eps)
    loss, grad = ev(np.stack([f, f + h * v, f - h * v]))
    saved = c.get_flat()
    c.set_flat(f)
    ref = pilco.sample_policy_gradient(pilco.m_init, pilco.S_init, pilco.horizon, num_samples=P, seed=seed)
    c.set_flat(saved)
    scale = np.abs(ref.grad).max()
    lerr, gerr = abs(loss[0] + ref.value) / abs(ref.value), np.abs(grad[0] + ref.grad).max() / scale
    fd = (loss[1] - loss[2]) / (2 * h)
    gv = float(grad[0] @ v)
    print("%s evaluator vs sample_policy_gradient: loss %.1e, grad %.1e of scale; directional difference rel %.1e"
          % (kind, lerr, gerr, abs(fd - gv) / abs(gv)))
    assert lerr <= 1e-12 and gerr <= 1e-12
    if kind == "linear":                                        # the same unbatched kernels on the same arrays
        assert loss[0] == -ref.value and np.array_equal(grad[0], -ref.grad)
    assert abs(fd - gv) <= 1e-6 * abs(gv)


def _start_values(pilco, flats0, P, seed):
    x0, eps = pilco._particle_inputs(pilco.m_init, pilco.S_init, pilco.horizon, P, seed, "test")
    loss, _ = policy_opt.ParticleEvaluator(pilco, flats0.shape[0], x0, eps)(flats0)
    return -loss, x0, eps


@pytest.mark.parametrize("kind", ["rbf", "linear"])
def test_optimize_policy_sampled(kind):
    pilco, _, _ = _pilco(kind, 42)
    P, seed, restarts, maxiter = 300, 13, 3, 30
    state = np.random.get_state()
    flats0 = policy_opt.initial_flats(pilco.controller, restarts)
    start, x0, eps = _start_values(pilco, flats0, P, seed)
    best_flat, best, finals = policy_opt.optimize(pilco, maxiter=maxiter, restarts=restarts, flats0=flats0,
                                                  evaluator=partial(policy_opt.ParticleEvaluator, x0=x0, eps=eps))
    finals = np.asarray(finals)
    print("%s: sampled value per restart %s -> %s, best %.6f" % (kind, start, finals, best))
    assert np.all(finals >= start) and finals[0] > start[0]
    assert best == finals.max()                                 # (select_best: ties go to the lowest index)
    win = int(np.flatnonzero(finals == best)[0])
    again = -policy_opt.ParticleEvaluator(pilco, 1, x0, eps)(best_flat[None])[0][0]
    assert abs(again - finals[win]) <= 1e-12 * abs(best)
    runs = []
    for _ in range(2):                                          # the method itself, from the same np.random state
        np.random.set_state(state)
        pilco.controller.set_flat(flats0[0])
        value = pilco.optimize_policy_sampled(maxiter=maxiter, restarts=restarts, num_samples=P, seed=seed)
        runs.append(pilco.controller.get_flat().copy())
        assert value == best
        # the controller holds the winner (an RBF policy's lengthscales go through the softplus and back)
        assert np.abs(runs[-1] - best_flat).max() <= 1e-12 * np.abs(best_flat).max()
        held = pilco.sample_policy_gradient(pilco.m_init, pilco.S_init, pilco.horizon, num_samples=P, seed=seed).value
        assert abs(held - best) <= 1e-12 * abs(best)
    assert np.array_equal(runs[0], runs[1])
    assert pilco.mgpr.models[0].kernel.lengthscales.trainable     # the model's trainables are restored


def test_optimize_policy_sampled_smgpr_and_appended_data():
    from pilco.models import PILCO
    from pilco.controllers import LinearController
    np.random.seed(43)
    X, Y = _pilco_data(43, n=300, Ds=4)
    sp = PILCO((X, Y), num_induced_points=40, controller=LinearController(4, 1), horizon=5)
    f0 = sp.controller.get_flat()[None]
    start = _start_values(sp, f0, 200, 3)[0][0]
    value = sp.optimize_policy_sampled(maxiter=10, restarts=2, num_samples=200, seed=3)
    print("SMGPR: sampled value %.6f -> %.6f" % (start, value))
    assert np.isfinite(value) and value > start
    pilco, X, Y = _pilco("rbf", 44)
    pilco.mgpr.device_gp()                                      # factorised on the first 60 rows, then 20 appended
    pilco.mgpr.set_data((X, Y))
    f0 = pilco.controller.get_flat()[None]
    start = _start_values(pilco, f0, 200, 4)[0][0]
    assert pilco.mgpr.last_update == "append"
    value = pilco.optimize_policy_sampled(maxiter=10, restarts=2, num_samples=200, seed=4)
    print("after appended data: sampled value %.6f -> %.6f" % (start, value))
    assert np.isfinite(value) and value > start
