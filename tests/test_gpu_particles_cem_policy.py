"""GPU tests of the batched forward-only rollouts of stationary policies and the cross-entropy method over policy
parameters (DESIGN.md section 33): the batched forward bitwise against the batched gradient calls' forward and against
single forward calls, independent of R, of the chunking and of graph replay; the search's every iteration against the
numpy update fed the device's values and normals; PILCO.optimize_policy_sampled(optimizer="cem") against
sample_policy_gradient's value, with SafePILCO's risk channel, angles and measurement noise; the example."""
import ctypes as C
import os
import sys

import numpy as np
import pytest
import torch

import cem_oracle as co
from particle_cases import _angle_case
from pilco_b200 import _lib, controllers, engine, policy_opt, rewards
from pilco_b200._lib import check, lib
from pilco_b200.models.pilco import PILCO
from util import ROOT

pytestmark = pytest.mark.gpu


def _policies(kind, R, Dh, U, seed, bf=12):
    """a spec of R policies and each restart's unbatched spec"""
    rng = np.random.RandomState(seed)
    maxa = 0.8 + 0.4 * np.arange(U)
    if kind == "linear":
        W, b = 0.5 * rng.randn(R, U, Dh), rng.randn(R, U)
        spec = dict(kind=_lib.POLICY_LINEAR, Ds=Dh, U=U, squash=True, max_action=maxa, W=W, b=b)
        return spec, [dict(spec, W=W[r], b=b[r]) for r in range(R)]
    if kind == "rbf":
        pgp = engine.gp_factorize(rng.rand(R, bf, Dh) * 2.0 - 1.0, 0.3 * rng.randn(R, bf, U),
                                  1.0 + 0.2 * rng.rand(R, U, Dh), np.ones((R, U)), 1e-4 * np.ones((R, U)),
                                  need_iK=False, mode=1)
        spec = dict(kind=_lib.POLICY_RBF, Ds=Dh, U=U, squash=True, max_action=maxa, gp=pgp)
        # restart r's factor bits, as an unbatched policy
        return spec, [dict(spec, gp=engine.DeviceGP(pgp.X[r], pgp.ell[r], pgp.sf2[r], pgp.beta[r], mode=1))
                      for r in range(R)]
    hidden = (16, 8)
    n = engine.mlp_theta_size(Dh, U, hidden)
    theta = 0.4 * rng.randn(R, n)
    spec = dict(kind=_lib.POLICY_MLP, Ds=Dh, U=U, squash=True, max_action=maxa, hidden=hidden, theta=theta)
    return spec, [dict(spec, theta=theta[r]) for r in range(R)]


def _inputs(E, P, H, seed):
    rng = np.random.RandomState(seed)
    return 0.8 * rng.randn(P, E), rng.randn(P, H, E), rng.randn(P, H, E)


def _grad_plan(gp, spec, terms, P, H, mu, consistent, R, dims, v):
    kw = dict(mult_mu=mu, R=R, angles=list(dims) or None, measurement_noise=v)
    if consistent:
        return engine.ConsistentGradPlan(gp, spec, terms, P, H, **kw)
    return engine.ParticlePlan(gp, spec, terms, P, H, grad=True, **kw)


CASES = [(k, c, d, nz) for k in ("linear", "rbf") for c in (False, True) for d, nz in (((), False), ((1,), False),
                                                                                      ((), True), ((1,), True))]
CASES += [("mlp", c, (), False) for c in (False, True)]


@pytest.mark.parametrize("kind,consistent,dims,noisy", CASES,
                         ids=["%s-%s-A%d%s" % (k, "consistent" if c else "stepwise", len(d), "-noise" if nz else "")
                              for k, c, d, nz in CASES])
def test_batched_forward_is_the_gradient_calls_forward_and_its_single_calls(kind, consistent, dims, noisy):
    E, U, R, H, mu = 4, 1, 3, 5, 1.5
    gp, _, _, terms = _angle_case(E, list(dims), U, "linear", joint=True)
    P = 100 if consistent else 300
    Dh = E + len(dims)
    spec, singles = _policies(kind, R, Dh, U, seed=11 + len(dims) + 2 * noisy)
    x0, eps, nu = _inputs(E, P, H, seed=P + H + len(dims))
    v = 0.01 + 0.03 * np.random.RandomState(3).rand(E) if noisy else None
    nu = nu if noisy else None
    grad = _grad_plan(gp, spec, terms, P, H, mu, consistent, R, dims, v)
    grad.set_inputs(x0, eps, nu)
    g = grad.launch_grad()
    torch.cuda.synchronize()
    ref, vref = [t.clone() for t in grad.outputs()], g["value"].clone()
    plan = engine.ParticleBatchPlan(gp, spec, terms, P, H, R, mult_mu=mu, consistent=consistent,
                                    angles=list(dims) or None, measurement_noise=v)
    plan.set_inputs(x0, eps, nu)
    assert plan.chunk == R
    value = plan.launch()
    torch.cuda.synchronize()
    assert torch.equal(value, vref)
    assert all(torch.equal(a, c) for a, c in zip(plan.outputs(), ref))
    for r in range(R):                                                # restart r: the single forward call
        one = engine.ParticlePlan(gp, singles[r], terms, P, H, mult_mu=mu, consistent=consistent,
                                  angles=list(dims) or None, measurement_noise=v)
        one.set_inputs(x0, eps, nu)
        one.launch()
        torch.cuda.synchronize()
        assert all(torch.equal(a[r], c) for a, c in zip(ref, one.outputs())), r
    graph = torch.cuda.CUDAGraph()                                     # replay against eager
    with torch.cuda.graph(graph):
        plan.launch()
    for t in list(plan.outputs()) + [plan.value]:
        t.zero_()
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(plan.value, vref) and all(torch.equal(a, c) for a, c in zip(plan.outputs(), ref))


@pytest.mark.parametrize("kind", ["linear", "rbf", "mlp"])
@pytest.mark.parametrize("consistent", [False, True], ids=["stepwise", "consistent"])
def test_value_depends_on_neither_R_nor_the_chunking(kind, consistent):
    E, U, R, H, P = 3, 1, 7, 4, 40
    gp, _, _, terms = _angle_case(E, [], U, "linear")
    spec, singles = _policies(kind, R, E, U, seed=5)
    x0, eps, _ = _inputs(E, P, H, seed=9)
    whole = engine.ParticleBatchPlan(gp, spec, terms, P, H, R, consistent=consistent)
    whole.set_inputs(x0, eps)
    vw = whole.launch().clone()
    for Rc in (1, 3):
        small = engine.ParticleBatchPlan(gp, spec, terms, P, H, R, consistent=consistent,
                                         max_ws_bytes=whole.bytes_needed(Rc))
        assert small.chunk == Rc and len(small.chunks) == -(-R // Rc)
        small.set_inputs(x0, eps)
        assert torch.equal(small.launch(), vw), Rc
    for r in (0, R - 1):                                               # R = 1
        one = engine.ParticleBatchPlan(gp, _batch_of_one(singles[r]), terms, P, H, 1, consistent=consistent)
        one.set_inputs(x0, eps)
        assert torch.equal(one.launch(), vw[r:r + 1]), r
    torch.cuda.synchronize()


def _batch_of_one(spec):
    """an unbatched policy spec as a batch of one"""
    if spec["kind"] == _lib.POLICY_LINEAR:
        return dict(spec, W=spec["W"][None], b=spec["b"][None])
    if spec["kind"] == _lib.POLICY_MLP:
        return dict(spec, theta=spec["theta"][None])
    g = spec["gp"]
    one = engine.DeviceGP(g.X[None], g.ell[None], g.sf2[None], g.beta[None], mode=1, batched=True)
    return dict(spec, gp=one)


# ---- the search ----------------------------------------------------------------------------------------------------------
def _pilco(kind="linear", seed=0, H=6, **kw):
    np.random.seed(seed)
    rng = np.random.RandomState(seed)
    X = np.hstack([rng.randn(60, 2) * 0.5, rng.uniform(-1, 1, (60, 1))])
    Y = np.stack([0.1 * X[:, 1], 0.1 * (-np.sin(X[:, 0]) + X[:, 2])], 1)
    Dh = 2 + len(kw.get("angle_dims") or [])
    c = {"linear": lambda: controllers.LinearController(Dh, 1, max_action=1.5),
         "rbf": lambda: controllers.RbfController(Dh, 1, 8, max_action=1.5),
         "mlp": lambda: controllers.MlpController(Dh, 1, (8,), max_action=1.5)}[kind]()
    p = PILCO((X, Y), controller=c, horizon=H, reward=rewards.ExponentialReward(2, t=np.array([0.5, 0.0])),
              m_init=np.zeros((1, 2)), S_init=0.01 * np.eye(2), **kw)
    for m in p.mgpr.models:
        m.likelihood.variance.assign(1e-3)
    return p


def _search(p, K, ke, iters, S, seed, std=0.3):
    x0, eps = p._particle_inputs(p.m_init, p.S_init, p.horizon, S, seed, "test")
    s = policy_opt.CemPolicySearch(p, K, ke, iters, S, seed, std0=std)
    s.set_inputs(x0, eps)
    return s


@pytest.mark.parametrize("kind", ["linear", "rbf", "mlp"])
def test_every_iteration_against_the_numpy_update(kind):
    """iteration i of a search of i + 1 iterations: population i is bitwise mean + std xi (row 0 the mean) of the
    previous distribution with xi the counter-based normals at iteration i; the update fed the device's values equals
    the oracle's"""
    p = _pilco(kind)
    K, ke, iters, S, seed, alpha = 48, 6, 3, 16, 7, policy_opt.CemPolicySearch.ALPHA
    n = p.controller.get_flat().size
    mean = p.controller.get_flat().copy()
    std, bv, best = np.full(n, 0.3), -np.inf, mean.copy()
    for i in range(iters):
        s = _search(p, K, ke, i + 1, S, seed)
        s.launch()
        torch.cuda.synchronize()
        xi = engine.normals(torch.empty(K, n, dtype=torch.float64, device=engine.device()), seed, s.STREAM,
                            torch.full((1,), i, dtype=torch.int64, device=engine.device())).cpu().numpy()
        assert np.array_equal(s.xi.cpu().numpy(), xi)
        cand = s.cand.cpu().numpy()
        assert np.array_equal(cand, co.draw(mean[None], std[None], xi[:, None], -np.inf, np.inf)[:, 0]), i
        value = s.plan.value.cpu().numpy()
        ref = co.update(cand[:, None], value, mean[None], std[None], ke, alpha, -np.inf, np.inf, bv, best[None])
        got_mean, got_std = s.mean.cpu().numpy(), s.std.cpu().numpy()
        for k, got in (("mean", got_mean), ("std", got_std)):
            assert np.abs(got - ref[k][0]).max() <= 1e-14 * max(1.0, np.abs(ref[k]).max()), (i, k)
        assert np.array_equal(s.best.cpu().numpy(), ref["best"][0]) and float(s.best_value[0]) == ref["best_value"]
        assert np.array_equal(s.trace[i].cpu().numpy(), ref["trace"])
        mean, std, bv, best = got_mean, got_std, ref["best_value"], ref["best"][0]
    again = _search(p, K, ke, iters, S, seed)
    again.run()                                                       # graph replay after the eager warm-up
    torch.cuda.synchronize()
    for a, c in ((again.best, s.best), (again.best_value, s.best_value), (again.trace, s.trace), (again.mean, s.mean),
                 (again.std, s.std)):
        assert torch.equal(a, c)


def _value_at(p, flat, S, seed):
    c = p.controller
    keep = c.get_flat().copy()
    c.set_flat(flat)
    v = p.sample_policy_gradient(p.m_init, p.S_init, p.horizon, num_samples=S, seed=seed).value
    c.set_flat(keep)
    return v


@pytest.mark.parametrize("kind", ["linear", "rbf", "mlp"])
def test_class_value_is_sample_policy_gradients_and_beats_the_start(kind):
    p = _pilco(kind, seed=1)
    S, seed = 64, 5
    start = _value_at(p, p.controller.get_flat(), S, seed)
    kw = dict(optimizer="cem", maxiter=4, num_samples=S, seed=seed, population=128, elites=12, cem_std=0.3)
    v = p.optimize_policy_sampled(**kw)
    flat = p.controller.get_flat().copy()
    after = p.sample_policy_gradient(p.m_init, p.S_init, p.horizon, num_samples=S, seed=seed).value
    print("CEM %s: start %.9f, in-sample best %.9f" % (kind, start, v))
    tol = 1e-10 * max(1.0, abs(after)) if kind == "rbf" else 0.0     # RBF: the controller factorises on its own path
    assert abs(v - after) <= tol
    assert v >= start - tol and np.isfinite(v)
    s = p.cem_search
    assert s.trace.shape == (4, 2) and float(s.best_value[0]) == v == float(s.trace[:, 0].max())
    p2 = _pilco(kind, seed=1)
    assert p2.optimize_policy_sampled(**kw) == v and np.array_equal(p2.controller.get_flat(), flat)   # seeded


def test_safe_pilco_trains_with_the_risk_channel():
    """RiskOfCollision is a box term: the default optimizer refuses it; CEM trains the stationary policy with it"""
    from safe_pilco_extension.rewards_safe import RiskOfCollision
    from safe_pilco_extension.safe_pilco import SafePILCO
    from pilco.rewards import LinearReward
    np.random.seed(0)
    rng = np.random.RandomState(1)
    X = np.hstack([rng.uniform(-1, 1, (60, 4)), rng.uniform(-1, 1, (60, 1))])
    Y = 0.1 * np.stack([X[:, 1], X[:, 4], X[:, 3], -X[:, 4]], 1)
    sp = SafePILCO((X, Y), controller=controllers.LinearController(4, 1), horizon=6,
                   reward_add=LinearReward(4, np.array([1.0, 0.0, 0.0, 0.0])),
                   reward_mult=RiskOfCollision(4, [-0.05, -0.05], [0.05, 0.05]), mu=-4.0)
    with pytest.raises(ValueError, match="box"):
        sp.optimize_policy_sampled(num_samples=32, seed=0)
    flat0 = sp.controller.get_flat().copy()
    v = sp.optimize_policy_sampled(optimizer="cem", num_samples=32, seed=0, maxiter=4, population=128, elites=12)
    s = sp.cem_search
    start = _rerun(sp, s, flat0)
    print("SafePILCO CEM: start %.6f, in-sample best %.6f" % (start, v))
    assert np.isfinite(v) and v >= start
    assert v == _rerun(sp, s, sp.controller.get_flat())


def _rerun(p, s, flat):
    """ParticleBatchPlan at one flat vector over the search's x0, eps (and nu) -> its value"""
    c = p.controller
    keep = c.get_flat().copy()
    c.set_flat(flat)
    spec = c.policy_spec(flat[None]) if not isinstance(c, controllers.RbfController) else p.policy_spec(flat[None])
    c.set_flat(keep)
    terms, mu = p.reward_spec()
    q = s.plan
    plan = engine.ParticleBatchPlan(p.mgpr.device_gp(), spec, terms, q.P, q.H, 1, mult_mu=mu,
                                    consistent=q.consistent, angles=p.angle_dims, measurement_noise=p._noise_var())
    plan.set_inputs(q.x0, q.eps_buf, q.nu_buf if q.nz is not None else None)
    v = float(plan.launch()[0])
    return v


@pytest.mark.parametrize("kind", ["linear", "rbf"])
@pytest.mark.parametrize("feature", ["angles", "noise"])
def test_angles_and_measurement_noise(kind, feature):
    kw = dict(angle_dims=[0]) if feature == "angles" else dict(measurement_noise="model")
    p = _pilco(kind, seed=2, **kw)
    flat0 = p.controller.get_flat().copy()
    v = p.optimize_policy_sampled(optimizer="cem", num_samples=32, seed=4, maxiter=3, population=96, elites=10,
                                  cem_std=0.3)
    s = p.cem_search
    assert (s.plan.nz is not None) == (feature == "noise") and (s.plan.ang is not None) == (feature == "angles")
    start, at = _rerun(p, s, flat0), _rerun(p, s, p.controller.get_flat())
    print("CEM %s with %s: start %.9f, in-sample best %.9f" % (kind, feature, start, v))
    if kind == "rbf":
        assert abs(v - at) <= 1e-10 * max(1.0, abs(at))
    else:
        assert v == at
    assert v >= start


def test_consistent_sampler_and_a_nan_candidate_never_wins():
    p = _pilco("linear", seed=3)
    v = p.optimize_policy_sampled(optimizer="cem", num_samples=16, seed=2, maxiter=2, population=32, elites=4,
                                  consistent=True)
    assert v == p.sample_policy_gradient(p.m_init, p.S_init, p.horizon, num_samples=16, seed=2, consistent=True).value
    s = _search(p, 16, 4, 1, 8, 3)
    s.launch()
    s.plan.value[3] = float("nan")                                     # the update alone, fed a NaN at row 3
    s.plan.value[5] = 1e9
    s.best_value.fill_(-float("inf"))
    check(lib.pilco_cem_update(C.byref(s.updates[0]), s.uws.data_ptr(), s.uws_bytes, engine.stream_ptr()), "cem")
    torch.cuda.synchronize()
    order = s.uws.view(torch.int32)[:16].cpu().numpy()
    assert order[0] == 5 and order[-1] == 3 and float(s.best_value[0]) == 1e9
    assert torch.equal(s.best, s.cand[5])
    s.plan.value.fill_(float("nan"))                                  # every candidate NaN: the best stays the start
    s.best_value.fill_(-float("inf"))
    s.best.copy_(s.mean0)
    check(lib.pilco_cem_update(C.byref(s.updates[0]), s.uws.data_ptr(), s.uws_bytes, engine.stream_ptr()), "cem")
    torch.cuda.synchronize()
    assert float(s.best_value[0]) == -float("inf") and torch.equal(s.best, s.mean0)


def test_example_runs():
    sys.path.insert(0, os.path.join(ROOT, "examples"))
    import safe_cars_cem_numpy as ex
    out = ex.run(J=2, N=1, T=10, maxiter=2, population=64, elites=8, num_samples=16)
    assert all(np.isfinite(r) for r in out)
