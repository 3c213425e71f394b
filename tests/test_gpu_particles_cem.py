"""GPU tests of the batched forward-only rollouts and the cross-entropy method (DESIGN.md section 31): the batched
forward bitwise against the scheduled gradient calls' forward and against single calls, chunking, rerun and graph
replay; the update fed the device's own values against the numpy oracle; the whole loop against the particle oracle
and the numpy update; monotonicity; SafePILCO's risk channel; PILCO.plan(optimizer="cem"); the example."""
import os
import sys

import numpy as np
import pytest
import torch

import cem_oracle as co
import particle_oracle as po
import particle_schedule_oracle as pso
from particle_cases import _angle_case, _dyn_np
from pilco_b200 import _lib, controllers, engine, rewards
from pilco_b200.models.pilco import PILCO
from util import ROOT

pytestmark = pytest.mark.gpu

LO, HI = -np.pi / 2, np.pi / 2


def _draw(E, P, H, seed):
    rng = np.random.RandomState(seed)
    return 0.8 * rng.randn(P, E), rng.randn(P, H, E), rng.randn(P, H, E)


def _var(E, seed=0):
    return 0.01 + 0.03 * np.random.RandomState(seed + 100).rand(E)


def _grad_plan(gp, spec, terms, P, H, mu, consistent, R, dims, v):
    kw = dict(mult_mu=mu, R=R, angles=list(dims) or None, measurement_noise=v, schedule=True)
    if consistent:
        return engine.ConsistentGradPlan(gp, spec, terms, P, H, **kw)
    return engine.ParticlePlan(gp, spec, terms, P, H, grad=True, **kw)


class _Batch:
    """the batched forward on a plan's description and output buffers (its own workspace and value)"""

    def __init__(self, plan, consistent, R):
        key = ("scheduled", "consistent" if consistent else "step", "batch")
        self.pr = _lib.Particles.from_buffer_copy(plan.pr)
        wsb = plan._entry(key, pr=self.pr, R=R).query()
        assert wsb > 0
        self.ws = torch.empty(wsb // 8 + 2, dtype=torch.float64, device=engine.device())
        self.pr.ws, self.pr.ws_bytes = self.ws.data_ptr(), wsb
        self.value = torch.zeros(R, dtype=torch.float64, device=engine.device())
        self.call = plan._entry(key, pr=self.pr, R=R, value=self.value.data_ptr())

    def __call__(self):
        self.call()


FORWARD = [(False, False), (False, True), (True, False), (True, True)]      # consistent, angles and noise


@pytest.mark.parametrize("consistent,mapped", FORWARD, ids=["stepwise", "stepwise-angles-noise", "consistent",
                                                            "consistent-angles-noise"])
def test_batched_forward_is_the_gradient_calls_forward_and_its_single_calls(consistent, mapped):
    E, U, R, H, mu = 4, 1, 3, 5, 1.5
    dims = [1] if mapped else []
    gp, spec, _, terms = _angle_case(E, dims, U, "linear", joint=True)
    P = 150 if consistent else 400
    x0, eps, nu = _draw(E, P, H, seed=P + H + mapped)
    v = _var(E) if mapped else None
    rng = np.random.RandomState(5)
    W, b = 0.5 * rng.randn(R, H, U, E + len(dims)), rng.randn(R, H, U)
    plan = _grad_plan(gp, dict(spec, W=W, b=b), terms, P, H, mu, consistent, R, dims, v)
    plan.set_inputs(x0, eps, nu if mapped else None)
    g = plan.launch_grad()
    torch.cuda.synchronize()
    ref, vref = [t.clone() for t in plan.outputs()], g["value"].clone()
    batch = _Batch(plan, consistent, R)
    for t in plan.outputs():
        t.zero_()
    batch()
    torch.cuda.synchronize()
    assert all(torch.equal(a, c) for a, c in zip(plan.outputs(), ref))
    assert torch.equal(batch.value, vref)
    for r in range(R):                                                # restart r: the single scheduled rollout
        one = engine.ParticlePlan(gp, dict(spec, W=W[r], b=b[r]), terms, P, H, mult_mu=mu, consistent=consistent,
                                  angles=dims or None, measurement_noise=v, schedule=True)
        one.set_inputs(x0, eps, nu if mapped else None)
        one.launch()
        torch.cuda.synchronize()
        assert all(torch.equal(a[r], c) for a, c in zip(ref, one.outputs())), r
    batch()                                                           # a rerun
    torch.cuda.synchronize()
    assert all(torch.equal(a, c) for a, c in zip(plan.outputs(), ref)) and torch.equal(batch.value, vref)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        batch()
    for t in list(plan.outputs()) + [batch.value]:
        t.zero_()
    graph.replay()
    torch.cuda.synchronize()
    assert all(torch.equal(a, c) for a, c in zip(plan.outputs(), ref)) and torch.equal(batch.value, vref)


def _cem_case(E=3, dims=(), H=5, seed=0, feedback=True):
    """gp, a scheduled spec (shared W, initial b), the oracle's policy dict and the terms"""
    gp, spec, pols, terms = _angle_case(E, list(dims), 1, "linear", seed=seed)
    rng = np.random.RandomState(seed + 3)
    Dh = E + len(dims)
    W = 0.3 * rng.randn(H, 1, Dh) if feedback else np.zeros((H, 1, Dh))
    sspec = dict(spec, W=W, b=0.4 * rng.randn(H, 1), schedule=True)
    return gp, sspec, dict(pols[0], W=W), terms


def _cem_plan(gp, spec, terms, P, H, K, ke, iters, x0, eps, xi, mu=0.0, **kw):
    plan = engine.CemPlan(gp, spec, terms, P, H, K, ke, iters, mult_mu=mu, **kw)
    plan.set_inputs(x0, eps, xi[:iters])
    plan.launch()
    torch.cuda.synchronize()
    return plan


def test_consistent_chunking_is_bitwise():
    E, H, P, K = 3, 4, 60, 24
    gp, spec, _, terms = _cem_case(E, (), H, seed=2)
    x0, eps, _ = _draw(E, P, H, seed=3)
    xi = np.random.RandomState(4).randn(2, K, H, 1)
    whole = _cem_plan(gp, spec, terms, P, H, K, 5, 2, x0, eps, xi, consistent=True)
    need = engine.CemPlan(gp, spec, terms, P, H, K, 5, 2, consistent=True, max_ws_bytes=1 << 40).ws.numel() * 8
    chunked = _cem_plan(gp, spec, terms, P, H, K, 5, 2, x0, eps, xi, consistent=True, max_ws_bytes=need // 4)
    assert whole.chunk == K and 1 < chunked.chunk < K // 2
    for a, c in zip(whole.outputs() + (whole.value, whole.mean, whole.std, whole.best_b, whole.best_value, whole.trace),
                    chunked.outputs() + (chunked.value, chunked.mean, chunked.std, chunked.best_b, chunked.best_value,
                                         chunked.trace)):
        assert torch.equal(a, c)


def test_update_on_device_values_against_the_oracle():
    """fed the device's own values: the elite sets, mean / std and best against the numpy update, and the populations
    bitwise clip(mean + std xi) of the distribution they were drawn from"""
    E, H, P, K, ke, alpha = 3, 5, 64, 256, 20, 0.1
    gp, spec, _, terms = _cem_case(E, (), H, seed=1)
    x0, eps, _ = _draw(E, P, H, seed=7)
    xi = np.random.RandomState(8).randn(2, K, H, 1)
    one = _cem_plan(gp, spec, terms, P, H, K, ke, 1, x0, eps, xi, alpha=alpha)
    two = _cem_plan(gp, spec, terms, P, H, K, ke, 2, x0, eps, xi, alpha=alpha)
    mean0, std0 = spec["b"][:H], np.full((H, 1), np.pi / 4)
    assert np.array_equal(one.cand.cpu().numpy(), co.draw(mean0, std0, xi[0], LO, HI))
    value = one.value.cpu().numpy()
    ref = co.update(one.cand.cpu().numpy(), value, mean0, std0, ke, alpha, LO, HI, -np.inf, mean0)
    order = one.uws.view(torch.int32)[:K].cpu().numpy()
    assert np.array_equal(order, ref["order"])
    assert set(order[:ke]) == set(ref["elites"])
    for k, t in (("mean", one.mean), ("std", one.std), ("best", one.best_b)):
        got = t.cpu().numpy()
        assert np.abs(got - ref[k]).max() <= 1e-14 * max(1.0, np.abs(ref[k]).max()), k
    assert float(one.best_value[0]) == ref["best_value"]
    assert np.array_equal(one.trace[0].cpu().numpy(), ref["trace"])
    nxt = co.draw(one.mean.cpu().numpy(), one.std.cpu().numpy(), xi[1], LO, HI)
    assert np.array_equal(two.cand.cpu().numpy(), nxt)


def _oracle_cem(dyn, pol, terms, x0, eps, xi, mean0, K, ke, iters, alpha, mu):
    """the particle oracle scores every candidate, the numpy update advances them -> per-iteration states and the
    smallest margin an elite set or a best-so-far decision had"""
    mean, std = mean0.copy(), np.full_like(mean0, np.pi / 4)
    cand = co.draw(mean, std, xi[0], LO, HI)
    best_value, best, states, margin = -np.inf, mean0.copy(), [], np.inf
    for i in range(iters):
        value = np.empty(K)
        for k in range(K):
            p = dict(pol, b=cand[k])
            with pso.schedule(p):
                value[k] = po.particle_rollout(dyn, p, terms, x0, eps, mu)[4].mean()
        s = np.sort(value)[::-1]
        margin = min(margin, s[ke - 1] - s[ke] if ke < K else np.inf,
                     abs(s[0] - best_value) if np.isfinite(best_value) else np.inf)
        out = co.update(cand, value, mean, std, ke, alpha, LO, HI, best_value, best,
                        xi[i + 1] if i + 1 < iters else None)
        mean, std, best_value, best, cand = out["mean"], out["std"], out["best_value"], out["best"], out["cand"]
        states.append(dict(mean=mean, std=std, best=best, best_value=best_value, trace=out["trace"]))
    return states, margin


def test_whole_loop_against_the_oracle():
    """K = 64, P = 8, H = 5, 3 iterations, at a seed whose elite and best decisions are all decided by more than 1e-9"""
    E, H, P, K, ke, iters, alpha, mu = 3, 5, 8, 64, 8, 3, 0.1, 0.0
    for seed in range(20):
        gp, spec, pol, terms = _cem_case(E, (), H, seed=seed)
        x0, eps, _ = _draw(E, P, H, seed=seed + 40)
        xi = np.random.RandomState(seed + 50).randn(iters, K, H, 1)
        states, margin = _oracle_cem(_dyn_np(gp), pol, terms, x0, eps, xi, spec["b"][:H], K, ke, iters, alpha, mu)
        if margin > 1e-9:
            break
    assert margin > 1e-9
    print("CEM whole loop: seed %d, smallest decision margin %.2e" % (seed, margin))
    for i in range(iters):
        plan = _cem_plan(gp, spec, terms, P, H, K, ke, i + 1, x0, eps, xi, alpha=alpha)
        ref = states[i]
        for k, t in (("mean", plan.mean), ("std", plan.std), ("best", plan.best_b)):
            got = t.cpu().numpy()
            err = np.abs(got - ref[k]).max() / max(1.0, np.abs(ref[k]).max())
            assert err <= 1e-10, (i, k, err)
        assert abs(float(plan.best_value[0]) - ref["best_value"]) <= 1e-10 * max(1.0, abs(ref["best_value"]))
        assert np.abs(plan.trace[i].cpu().numpy() - ref["trace"]).max() <= 1e-10 * max(1.0, np.abs(ref["trace"]).max())


def test_best_value_is_monotone_and_beats_the_warm_start():
    E, dims, H, P, K, ke = 3, (1,), 6, 32, 128, 12
    gp, spec, _, terms = _cem_case(E, dims, H, seed=4, feedback=False)
    x0, eps, nu = _draw(E, P, H, seed=11)
    v = _var(E, 2)
    xi = np.random.RandomState(12).randn(4, K, H, 1)
    best = []
    for iters in range(1, 5):
        plan = engine.CemPlan(gp, spec, terms, P, H, K, ke, iters, angles=list(dims), measurement_noise=v)
        plan.set_inputs(x0, eps, xi[:iters], nu=nu)
        plan.launch()
        torch.cuda.synchronize()
        best.append(float(plan.best_value[0]))
    assert all(a <= c for a, c in zip(best, best[1:]))
    assert best[-1] == float(plan.trace[:, 0].max())
    warm = dict(spec, b=np.clip(spec["b"], LO, HI))
    out = engine.particles_rollout(gp, warm, terms, engine.dev(x0), engine.dev(eps), angles=list(dims),
                                   measurement_noise=v, nu=engine.dev(nu), schedule=True)
    start = float(out[4].mean())
    print("CEM best value per iteration %s, warm start %.6f" % (np.round(best, 6), start))
    assert best[0] >= start - 1e-12 * max(1.0, abs(start))


def test_safe_pilco_plans_with_the_risk_channel():
    """RiskOfCollision is a box term: the gradient planner refuses it, CEM plans with it and beats the zero-action
    schedule on the same particles"""
    from safe_pilco_extension.rewards_safe import RiskOfCollision
    from safe_pilco_extension.safe_pilco import SafePILCO
    from pilco.rewards import LinearReward
    np.random.seed(0)
    rng = np.random.RandomState(1)
    X = np.hstack([rng.uniform(-1, 1, (60, 4)), rng.uniform(-1, 1, (60, 1))])
    Y = 0.1 * np.stack([X[:, 1], X[:, 4], X[:, 3], -X[:, 4]], 1)
    H = 6
    sp = SafePILCO((X, Y), controller=controllers.TimeVaryingLinearController(4, 1, H, feedback=False), horizon=H,
                   reward_add=LinearReward(4, np.array([1.0, 0.0, 0.0, 0.0])),
                   reward_mult=RiskOfCollision(4, [-0.05, -0.05], [0.05, 0.05]), mu=-4.0)
    x = np.array([0.0, 0.0, 0.0, 0.0])
    with pytest.raises(ValueError, match="box"):
        sp.plan(x, num_samples=32, seed=0)
    u = np.asarray(sp.plan(x, num_samples=32, seed=0, optimizer="cem", maxiter=4, population=256, elites=20))
    assert u.shape == (1, 1) and np.all(np.isfinite(u))
    plan = sp.cem_plan
    terms, mu = sp.reward_spec()
    zero = dict(sp.controller.policy_spec(), b=np.zeros((H, 1)))
    ret = engine.particles_rollout(sp.mgpr.device_gp(), zero, terms, plan.x0, plan.eps_buf, mult_mu=mu,
                                   schedule=True)[4]
    z, best = float(ret.mean()), float(plan.best_value[0])
    print("SafePILCO CEM plan: in-sample value %.6f, zero-action schedule %.6f" % (best, z))
    assert best > z


def _mpc_pilco(H=8, seed=0):
    np.random.seed(seed)
    rng = np.random.RandomState(seed)
    X = np.hstack([rng.randn(60, 2) * 0.5, rng.uniform(-1, 1, (60, 1))])
    Y = np.stack([0.1 * X[:, 1], 0.1 * (-np.sin(X[:, 0]) + X[:, 2])], 1)
    c = controllers.TimeVaryingLinearController(2, 1, H, max_action=1.5, feedback=False)
    pilco = PILCO((X, Y), controller=c, horizon=H, reward=rewards.ExponentialReward(2, t=np.array([0.5, 0.0])),
                  m_init=np.zeros((1, 2)), S_init=0.01 * np.eye(2))
    for m in pilco.mgpr.models:
        m.likelihood.variance.assign(1e-3)
    return pilco


def test_class_plan_is_seeded_acts_within_bounds_and_shifts():
    pilco = _mpc_pilco()
    c = pilco.controller
    flat0 = c.get_flat().copy()
    x = np.array([0.1, -0.2])
    kw = dict(num_samples=32, seed=3, optimizer="cem", maxiter=3, population=64, elites=8)
    u = np.asarray(pilco.plan(x, **kw))
    plan = pilco.cem_plan
    best = plan.best_b.cpu().numpy()
    assert u.shape == (1, 1) and np.all(np.abs(u) <= 1.5)
    assert np.allclose(u, 1.5 * np.sin(best[0]), rtol=0, atol=1e-12)          # u_0 = maxa sin(b_0)
    assert np.array_equal(np.asarray(c.b), np.concatenate([best[1:], best[-1:]]))
    x0, eps = pilco._particle_inputs(x.reshape(1, 2), np.zeros((2, 2)), 8, 32, 3, "plan")
    assert torch.equal(plan.x0, x0) and torch.equal(plan.eps_buf, eps)        # the L-BFGS-B planner's particles
    assert float(plan.best_value[0]) >= float(plan.trace[0, 0])
    c.set_flat(flat0)
    u2 = np.asarray(pilco.plan(x, **kw))
    assert np.array_equal(u, u2)


def test_example_runs_two_mpc_steps():
    sys.path.insert(0, os.path.join(ROOT, "examples"))
    import pendulum_cem_numpy as ex
    random_returns, mpc_returns = ex.run(episodes=1, T=2, random_episodes=2)
    assert len(mpc_returns) == 1 and np.isfinite(mpc_returns[0]) and 0.0 <= mpc_returns[0] <= 2.0
