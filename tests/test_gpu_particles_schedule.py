"""GPU tests of the time-varying linear policy in the particle rollouts (pilco_particles_scheduled_*, DESIGN.md section
28) through engine.ParticlePlan / ConsistentGradPlan / particles_rollout(schedule=True) and PILCO.plan(num_samples=...):
a constant schedule against the stationary call (bitwise forward and value, per-step gradients summing to its
gradient), the numpy and torch oracles on random schedules with the features the samplers combine, a central
difference, restarts against single calls and graph replay, the one-step moments against the moment-matching
RolloutPlan(schedule=True), and receding-horizon planning on the sampled return."""
import os
import sys

import numpy as np
import pytest
import torch

from pilco_b200 import controllers, engine, rewards
from pilco_b200.models.pilco import PILCO
import particle_grad_oracle as pgo
import particle_oracle as po
import particle_schedule_oracle as pso
from particle_cases import _angle_case, _dyn_np
from util import _rel, scaled_err

pytestmark = pytest.mark.gpu


def _draw(E, P, H, seed):
    rng = np.random.RandomState(seed)
    return 0.8 * rng.randn(P, E), rng.randn(P, H, E), rng.randn(P, H, E), rng.randn(P, H, E)


def _var(E, seed=0):
    return 0.01 + 0.03 * np.random.RandomState(seed + 100).rand(E)


def _schedule(spec, H, R=None, seed=0):
    """a random schedule W [R?,H,U,Dh], b [R?,H,U] around the stationary spec's scale"""
    rng = np.random.RandomState(seed + 11)
    lead = () if R is None else (R,)
    U, Dh = spec["U"], spec["Ds"]
    return 0.5 * rng.randn(*lead, H, U, Dh), rng.randn(*lead, H, U)


def _make(gp, spec, terms, P, H, mu, sampler="stepwise", estimator="pathwise", R=1, dims=(), v=None, x=None,
          schedule=True, grad=True):
    if sampler == "consistent" and grad:
        return engine.ConsistentGradPlan(gp, spec, terms, P, H, mult_mu=mu, R=R, angles=list(dims) or None,
                                         measurement_noise=v, exploration=x, estimator=estimator, schedule=schedule)
    return engine.ParticlePlan(gp, spec, terms, P, H, mult_mu=mu, grad=grad, R=R, consistent=sampler == "consistent",
                               estimator=estimator, angles=list(dims) or None, measurement_noise=v, exploration=x,
                               resample=sampler == "resampled", schedule=schedule)


def _run(plan, x0, eps, nu, xi, grad=True):
    plan.set_inputs(x0, eps, nu if plan.nz is not None else None, xi if plan.resample else None)
    g = {k: t.clone() for k, t in plan.launch_grad().items()} if grad else {}
    if not grad:
        plan.launch()
    torch.cuda.synchronize()
    return [t.clone() for t in plan.outputs()], g


CONSTANT = [  # sampler, estimator, angles, noise, exploration
    ("stepwise", "pathwise", (), False, None),
    ("stepwise", "pathwise", (1,), True, 0.4),
    ("stepwise", "score", (1,), True, None),
    ("consistent", "pathwise", (), False, 0.3),
    ("consistent", "pathwise", (1,), True, None),
    ("consistent", "score", (1,), True, None),
    ("resampled", "pathwise", (), False, None),
]


@pytest.mark.parametrize("sampler,estimator,dims,noise,x", CONSTANT)
def test_constant_schedule_is_the_stationary_call(sampler, estimator, dims, noise, x):
    """W_t = W and b_t = b: the outputs and value bitwise, sum_t of the per-step gradients the stationary gradient up
    to the order of the sums; R = 2 restarts, and the forward-only call at R = 1"""
    E, U, R, H, mu = 4, 1, 2, 5, 1.5
    gp, spec, _, terms = _angle_case(E, list(dims), U, "linear", joint=sampler != "resampled", R=R)
    P = 150 if sampler == "consistent" else 400
    x0, eps, nu, xi = _draw(E, P, H, seed=P + H)
    v = _var(E) if noise else None
    rep = lambda a: np.repeat(a[:, None], H, 1)
    sspec = dict(spec, W=rep(spec["W"]), b=rep(spec["b"]))
    kw = dict(sampler=sampler, estimator=estimator, R=R, dims=dims, v=v, x=x)
    out0, g0 = _run(_make(gp, spec, terms, P, H, mu, schedule=False, **kw), x0, eps, nu, xi)
    out1, g1 = _run(_make(gp, sspec, terms, P, H, mu, **kw), x0, eps, nu, xi)
    assert all(torch.equal(a, b) for a, b in zip(out0, out1))
    assert torch.equal(g0["value"], g1["value"])
    assert g1["W"].shape == (R, H, U, E + len(dims)) and g1["b"].shape == (R, H, U)
    for k in ("W", "b"):
        ref = g0[k].cpu().numpy()
        err = np.abs(g1[k].sum(1).cpu().numpy() - ref).max() / np.abs(ref).max()
        print("constant schedule %s/%s dims=%s noise=%s x=%s: sum_t g%s_t vs stationary %.1e" % (sampler, estimator,
                                                                                             dims, noise, x, k, err))
        assert err <= 1e-13, (k, err)
    if sampler == "resampled" or (sampler == "stepwise" and estimator == "pathwise"):    # forward-only, R = 1
        one = lambda s: dict(s, W=s["W"][0], b=s["b"][0])
        fw = dict(sampler=sampler, dims=dims, v=v, grad=False)
        a, _ = _run(_make(gp, one(spec), terms, P, H, mu, schedule=False, **fw), x0, eps, nu, xi, grad=False)
        b, _ = _run(_make(gp, one(sspec), terms, P, H, mu, **fw), x0, eps, nu, xi, grad=False)
        assert all(torch.equal(p, q) for p, q in zip(a, b))


SHAPES = {"small": (4, [1], 1), "swimmer": (8, [], 2)}          # E, angles, U
PARITY = [  # shape, sampler, estimator, noise, exploration
    ("small", "stepwise", "pathwise", True, 0.4),
    ("small", "stepwise", "score", True, None),
    ("small", "consistent", "pathwise", True, None),
    ("small", "consistent", "score", False, None),
    ("small", "resampled", "pathwise", False, None),
    ("swimmer", "stepwise", "pathwise", False, None),
    ("swimmer", "stepwise", "score", False, None),
    ("swimmer", "consistent", "pathwise", False, 0.3),
]


@pytest.mark.parametrize("shape,sampler,estimator,noise,x", PARITY)
def test_oracle_parity(shape, sampler, estimator, noise, x):
    """random W_t, b_t: the forward against the numpy oracle (the torch oracle's for the refit), the gradients against
    the torch oracle, at the tolerances of the stationary particle tests"""
    E, dims, U = SHAPES[shape]
    dims = [] if sampler == "resampled" else dims
    gp, spec, pols, terms = _angle_case(E, dims, U, "linear", joint=sampler != "resampled")
    P, H, mu = 200, 5, 1.5
    x0, eps, nu, xi = _draw(E, P, H, seed=P + H + 1)
    v = _var(E, 1) if noise else None
    W, b = _schedule(spec, H)
    sspec, pol = dict(spec, W=W, b=b), dict(pols[0], W=W, b=b)
    plan = _make(gp, sspec, terms, P, H, mu, sampler, estimator, dims=dims, v=v, x=x)
    out, g = _run(plan, x0, eps, nu, xi)
    g = {k: t.cpu().numpy() for k, t in g.items()}
    out = [t.cpu().numpy() for t in out]
    dyn = _dyn_np(gp)
    kw = dict(angle_dims=dims or None, nu=nu if noise else None, v=v)
    with pso.schedule(pol):
        ref_out, val, ref, own = _oracle(dyn, pol, terms, x0, eps, xi, mu, sampler, estimator, x, out, kw)
    errs = [scaled_err(o, r) if r.size and np.abs(r).max() > 0 else float(np.abs(o).max(initial=0.0))
            for o, r in zip(out, ref_out)]
    err, verr = _rel(g, ref), abs(float(g["value"][0]) - val) / max(abs(val), 1e-300)
    print("scheduled %s %s/%s noise=%s x=%s: forward %.1e, gradient %.1e of scale, value %.1e (own %.1e)"
          % (shape, sampler, estimator, noise, x, max(errs), err, verr, own))
    assert g["W"].shape == (H, U, E + len(dims)) and g["b"].shape == (H, U)
    assert max(errs) <= max(1e-9, 10.0 * own)
    assert err <= max(1e-8, 10.0 * own) and verr <= max(1e-9, 10.0 * own)


def _oracle(dyn, pol, terms, x0, eps, xi, mu, sampler, estimator, x, out, kw):
    """(forward outputs, value, gradient, the oracle's own rounding spread) of one sampler and estimator"""
    own = 0.0
    if sampler == "resampled":
        r = pgo.resampled_rollout(dyn, pol, terms, x0, eps, xi, mu)
        ref_out = [r[k] for k in ("traj", "act", "rew", "risk", "ret")]
        val, ref = r["value"], r["grad"]
    else:
        f = po.consistent_rollout if sampler == "consistent" else po.particle_rollout
        ref_out = f(dyn, pol, terms, x0, eps, mu, **kw)
        if sampler == "consistent":
            own = scaled_err(f(dyn, pol, terms, x0, eps, mu, swap=True, **kw)[0], ref_out[0])
        if estimator == "score":
            sg = pgo.score_grad(dyn, pol, terms, out[0], eps, mu, consistent=sampler == "consistent", **kw)
            ref, val = (sg[0] if sampler == "consistent" else sg), float(out[4].mean())
        elif sampler == "consistent":
            res = pgo.consistent_value_and_grad(dyn, pol, terms, x0, eps, mu, b=x, **kw)
            val, ref = res[0], res[1]
            own = max(own, _rel(pgo.consistent_value_and_grad(dyn, pol, terms, x0, eps, mu, swap=True, b=x, **kw)[1],
                                ref))
        else:
            val, ref = pgo.value_and_grad(dyn, pol, terms, x0, eps, mu, b=x, **kw)[:2]
    return ref_out, val, ref, own


def test_central_difference_along_a_schedule_direction():
    E, dims, U = 4, [1], 1
    gp, spec, _, terms = _angle_case(E, dims, U, "linear", joint=True)
    P, H, mu = 500, 6, 1.5
    x0, eps, nu, _ = _draw(E, P, H, seed=9)
    v = _var(E, 2)
    W, b = _schedule(spec, H, seed=4)
    plan = _make(gp, dict(spec, W=W, b=b), terms, P, H, mu, dims=dims, v=v)
    _, g = _run(plan, x0, eps, nu, None)
    val = lambda W, b: float(engine.particles_rollout(gp, dict(spec, W=W, b=b), terms, x0, eps, mult_mu=mu, angles=dims,
                                                      measurement_noise=v, nu=nu, schedule=True)[4].mean())
    rng = np.random.RandomState(3)
    dW, db = rng.randn(*W.shape), rng.randn(*b.shape)
    h = 1e-5
    fd = (val(W + h * dW, b + h * db) - val(W - h * dW, b - h * db)) / (2 * h)
    gd = float((g["W"].cpu().numpy() * dW).sum() + (g["b"].cpu().numpy() * db).sum())
    print("scheduled directional derivative: central difference %.12e, pathwise %.12e" % (fd, gd))
    assert abs(fd - gd) <= 1e-6 * abs(gd)


@pytest.mark.parametrize("sampler,estimator", [("stepwise", "pathwise"), ("stepwise", "score"),
                                               ("consistent", "pathwise"), ("resampled", "pathwise")])
def test_restarts_are_their_single_calls_and_replay_bitwise(sampler, estimator):
    E, dims, U, R = 4, ([] if sampler == "resampled" else [1]), 1, 3
    gp, spec, _, terms = _angle_case(E, dims, U, "linear", joint=sampler != "resampled")
    P, H, mu = 300, 5, 1.5
    x0, eps, nu, xi = _draw(E, P, H, seed=21)
    v = None if sampler == "resampled" else _var(E, 3)
    W, b = _schedule(spec, H, R=R, seed=6)
    kw = dict(sampler=sampler, estimator=estimator, dims=dims, v=v)
    plan = _make(gp, dict(spec, W=W, b=b), terms, P, H, mu, R=R, **kw)
    out, g = _run(plan, x0, eps, nu, xi)
    for r in range(R):
        o1, g1 = _run(_make(gp, dict(spec, W=W[r], b=b[r]), terms, P, H, mu, **kw), x0, eps, nu, xi)
        assert all(torch.equal(a[r], c) for a, c in zip(out, o1)), r
        assert all(torch.equal(g[k][r], g1[k].reshape(g[k][r].shape)) for k in g), r
    plan.launch_grad()                                              # a rerun
    torch.cuda.synchronize()
    assert all(torch.equal(a, c) for a, c in zip(plan.outputs(), out))
    assert all(torch.equal(plan.gbuf[k], g[k]) for k in g)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        plan.launch_grad()
    for t in list(plan.gbuf.values()) + [plan.traj, plan.ret]:
        t.zero_()
    graph.replay()
    torch.cuda.synchronize()
    assert all(torch.equal(a, c) for a, c in zip(plan.outputs(), out))
    assert all(torch.equal(plan.gbuf[k], g[k]) for k in g)


def test_one_step_moments_match_the_moment_matching_plan():
    """H = 1 under an unsquashed linear schedule from a Gaussian x0: the sample mean and covariance of x_1 against
    RolloutPlan(schedule=True)'s moment-matched ones (exact in the first two moments at one step)"""
    E, U = 3, 1
    gp, spec, _, terms = _angle_case(E, [], U, "linear")
    W, b = _schedule(spec, 2, seed=8)
    sspec = dict(spec, W=0.3 * W, b=0.3 * b, squash=False)
    m0, S0 = 0.1 * np.ones(E), 0.05 * np.eye(E) + 0.01
    mm = engine.RolloutPlan(gp, sspec, terms, m0, S0, 1, schedule=True)
    mm.forward()
    M1, S1 = mm.traj_m[0, 1].cpu().numpy(), mm.traj_S[0, 1].cpu().numpy()
    P = 1 << 17
    g = torch.Generator(device=engine.device())
    g.manual_seed(17)
    x0 = engine.dev(m0)[None] + torch.randn((P, E), dtype=engine.F64, device=engine.device(), generator=g) \
        @ engine.dev(np.linalg.cholesky(S0)).T
    eps = torch.randn((P, 1, E), dtype=engine.F64, device=engine.device(), generator=g)
    traj = engine.particles_rollout(gp, sspec, terms, x0, eps, schedule=True)[0]
    worst = po.moment_check(traj[:, 1].cpu().numpy(), M1, S1)
    print("scheduled one-step moments at P=2^17: worst %.2f standard errors" % worst)
    assert worst <= 5.0


def _pilco(H=8, seed=0):
    np.random.seed(seed)
    rng = np.random.RandomState(seed)
    X = np.hstack([rng.randn(60, 2) * 0.5, rng.uniform(-1, 1, (60, 1))])
    Y = np.stack([0.1 * X[:, 1], 0.1 * (-np.sin(X[:, 0]) + X[:, 2])], 1)
    c = controllers.TimeVaryingLinearController(2, 1, H, max_action=1.0, feedback=False)
    pilco = PILCO((X, Y), controller=c, horizon=H, reward=rewards.ExponentialReward(2, t=np.array([0.5, 0.0])),
                  m_init=np.zeros((1, 2)), S_init=0.01 * np.eye(2))
    for m in pilco.mgpr.models:
        m.likelihood.variance.assign(1e-3)
    return pilco


def test_plan_on_samples_acts_shifts_and_is_deterministic():
    pilco = _pilco()
    c = pilco.controller
    m_init, S_init = np.array(pilco.m_init), np.array(pilco.S_init)
    flat0 = c.get_flat().copy()
    seen = []
    shift = c.shift
    c.shift = lambda: (seen.append(c.get_flat().copy()), shift())
    x = np.array([0.1, -0.2])
    np.random.seed(5)
    u = np.asarray(pilco.plan(x, maxiter=8, restarts=2, num_samples=64, seed=3))
    assert u.shape == (1, 1) and np.all(np.isfinite(u))
    b = seen[0].reshape(8, 1)
    assert np.allclose(u, np.sin(b[0]), rtol=0, atol=1e-12)          # u_0 = maxa sin(b_0)
    assert np.array_equal(np.asarray(c.b), np.concatenate([b[1:], b[-1:]]))
    assert np.array_equal(pilco.m_init, m_init) and np.array_equal(pilco.S_init, S_init)
    assert not np.array_equal(seen[0], flat0)
    after = c.get_flat().copy()
    c.set_flat(flat0)
    np.random.seed(5)
    u2 = np.asarray(pilco.plan(x, maxiter=8, restarts=2, num_samples=64, seed=3))
    assert np.array_equal(u, u2) and np.array_equal(seen[1], seen[0]) and np.array_equal(c.get_flat(), after)
    u3 = np.asarray(pilco.plan(x, 0.01 * np.eye(2), maxiter=4, restarts=1, num_samples=32, seed=4, consistent=True))
    assert u3.shape == (1, 1) and np.all(np.isfinite(u3))


def test_mpc_on_samples_on_the_example_pendulum_beats_random_actions():
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "examples"))
    import pendulum_mpc_numpy
    random_returns, mpc_returns = pendulum_mpc_numpy.run(episodes=1, T=20, horizon=8, restarts=2, maxiter=8,
                                                         verbose=False, num_samples=64)
    print("sampled MPC return %s, random %s" % (mpc_returns, random_returns))
    assert np.all(np.isfinite(mpc_returns))
    assert np.mean(mpc_returns) > np.mean(random_returns), (mpc_returns, random_returns)
