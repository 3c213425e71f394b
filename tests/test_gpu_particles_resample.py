"""Gaussian-resampled particle rollouts on the device (pilco_particles_resampled_* through
engine.ParticlePlan(resample=True), DESIGN.md section 26): parity with the torch oracle
(tests/particle_grad_oracle.py's resampled_rollout) on the same x0, eps and xi, the call without resampling at H <= 1,
restarts against single calls, bitwise reproducibility and CUDA-graph replay, the fitted moments against the
moment-matching trajectory at every step, a central difference of the value, and the class-level options."""
import numpy as np
import pytest
import torch

from pilco_b200 import engine, _lib
from particle_cases import _batch_case, _case, _draw, _dyn_np, _linear_pilco, _oracle_pol, _pilco
import particle_grad_oracle as pgo
from util import make_gp_problem

pytestmark = pytest.mark.gpu

CASES = ["linear_squash", "linear_nosquash", "metric_rbf", "fitc", "joint_terms"]


def _get(name):
    if name == "joint_terms":
        gp, spec, pol, terms, m0, S0, H, P, mu = _case("linear_squash")
        terms = terms[:2] + [dict(kind=_lib.REWARD_EXP_SA, coef=0.7, W=np.eye(5) + 0.1, t=0.2 * np.ones(5)),
                             dict(kind=_lib.REWARD_LINEAR_SA, coef=-0.4, W=np.linspace(-1.0, 1.0, 5), t=None)]
        return gp, spec, pol, terms, m0, S0, H, P, mu
    return _case(name)


def _run(gp, spec, terms, x0, eps, xi, mu, R=1):
    plan = engine.ParticlePlan(gp, spec, terms, x0.shape[0], eps.shape[1], mult_mu=mu, grad=True, R=R, resample=True)
    plan.set_inputs(x0, eps, xi=xi)
    g = {k: t.clone() for k, t in plan.launch_grad().items()}
    out = [t.clone() for t in plan.outputs()] + [plan.step_mean.clone(), plan.step_cov.clone()]
    return plan, g, out


def _scaled(a, b):
    a, b = np.asarray(a), np.asarray(b)
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-300)) if b.size else 0.0


@pytest.mark.parametrize("name", CASES)
def test_parity_with_oracle(name):
    gp, spec, pol, terms, m0, S0, H, P, mu = _get(name)
    P = min(P, 300)
    x0, eps = _draw(m0, S0, P, H, seed=P + H + 1)
    xi = np.random.RandomState(P + H + 2).randn(P, H, m0.shape[0])
    _, g, out = _run(gp, spec, terms, x0, eps, xi, mu)
    ref = pgo.resampled_rollout(_dyn_np(gp), _oracle_pol(spec, pol), terms, x0, eps, xi, mu)
    tol = 1e-6 if name == "fitc" else 1e-9
    errs = {k: _scaled(o.cpu().numpy(), ref[k]) for k, o in zip(("traj", "act", "rew", "risk", "ret", "step_mean",
                                                                   "step_cov"), out)}
    errs["value"] = abs(float(g["value"].item()) - ref["value"]) / max(abs(ref["value"]), 1e-300)
    scale = max(float(np.abs(r).max()) for r in ref["grad"].values())
    errs["grad"] = max(float(np.abs(g[k].cpu().numpy().reshape(r.shape) - r).max()) for k, r in ref["grad"].items()) \
        / max(scale, 1e-300)
    print("resampled %s (P=%d, H=%d) vs oracle: %s" % (name, P, H, ", ".join("%s %.1e" % kv for kv in errs.items())))
    assert max(errs.values()) <= tol, errs


@pytest.mark.parametrize("H", [0, 1])
def test_short_horizons_are_the_call_without_resampling(H):
    gp, spec, pol, terms, m0, S0, _, P, mu = _case("metric_rbf")
    P = 500
    x0, eps = _draw(m0, S0, P, H, seed=3)
    xi = np.random.RandomState(4).randn(P, H, m0.shape[0])
    _, g, out = _run(gp, spec, terms, x0, eps, xi, mu)
    plan = engine.ParticlePlan(gp, spec, terms, P, H, mult_mu=mu, grad=True)
    plan.set_inputs(x0, eps)
    g0 = plan.launch_grad()
    out0 = plan.outputs()
    for k in g0:
        assert torch.equal(g[k], g0[k]), k
    for a, b in zip(out[1:5], out0[1:5]):
        assert torch.equal(a, b)
    assert torch.equal(out[0][:, 0], out0[0][:, 0])
    if H == 0:
        assert torch.equal(out[0], out0[0])


def test_restarts_are_the_single_calls_and_reproducible():
    gp, spec, singles, terms, m0, S0, H, P, mu = _batch_case("rbf", 3)
    x0, eps = _draw(m0, S0, P, H, seed=21)
    xi = np.random.RandomState(22).randn(P, H, m0.shape[0])
    plan, g, out = _run(gp, spec, terms, x0, eps, xi, mu, R=3)
    for r, one in enumerate(singles):
        _, g1, out1 = _run(gp, one, terms, x0, eps, xi, mu)
        for k in g1:
            assert torch.equal(g[k][r], g1[k].reshape(g[k][r].shape)), (r, k)
        for a, b in zip(out, out1):
            assert torch.equal(a[r], b.reshape(a[r].shape)), r
    again = {k: t.clone() for k, t in plan.launch_grad().items()}
    for k in g:
        assert torch.equal(again[k], g[k]), k
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            plan.launch_grad()
    graph.replay()
    torch.cuda.synchronize()
    for k in g:
        assert torch.equal(plan.gbuf[k], g[k]), k
    assert torch.equal(plan.step_cov, out[6]) and torch.equal(plan.traj, out[0])


def test_moments_match_moment_matching_at_every_step():
    """linear unsquashed policy: the refitted particles are Gaussian, so PILCO's moment matching of that Gaussian is
    exact and the fitted moments converge to RolloutPlan's (m_t, S_t) at every t"""
    X, Y, ell, sf2, sn2 = make_gp_problem(100, 5, 4, seed=6)
    gp = engine.gp_factorize(X, 0.1 * Y, ell, 0.1 * sf2, 1e-3 * np.ones(4))
    rng = np.random.RandomState(7)
    W, b = 0.5 * rng.randn(1, 4), rng.randn(1)
    spec = dict(kind=_lib.POLICY_LINEAR, Ds=4, U=1, squash=False, max_action=np.ones(1), W=W, b=b)
    terms = [dict(kind=_lib.REWARD_EXP, coef=1.0, W=np.eye(4), t=0.5 * np.ones(4))]
    m0, S0, H, P, K = X[0, :4], 0.05 * np.eye(4), 10, 1 << 16, 16
    mm = engine.RolloutPlan(gp, spec, terms, m0, S0, H)
    tm, tS, _ = mm.forward()
    tm, tS = tm[0].cpu().numpy(), tS[0].cpu().numpy()
    plan = engine.ParticlePlan(gp, spec, terms, P, H, resample=True)
    means, covs = [], []
    for k in range(K):
        g = torch.Generator(device=engine.device())
        g.manual_seed(100 + k)
        x0 = engine.dev(m0)[None] + torch.randn((P, 4), dtype=engine.F64, device=engine.device(), generator=g) \
            @ engine.dev(np.linalg.cholesky(S0)).T
        eps = torch.randn((P, H, 4), dtype=engine.F64, device=engine.device(), generator=g)
        xi = torch.randn((P, H, 4), dtype=engine.F64, device=engine.device(), generator=g)
        plan.set_inputs(x0, eps, xi=xi)
        plan.launch()
        means.append(plan.step_mean.cpu().numpy()); covs.append(plan.step_cov.cpu().numpy())
    means, covs = np.stack(means), np.stack(covs)
    worst = 0.0
    for t in range(H + 1):
        for est, ref in ((means[:, t], tm[t]), (covs[:, t], tS[t])):
            se = est.std(0, ddof=1) / np.sqrt(K)
            z = np.abs(est.mean(0) - ref) / np.maximum(se, 1e-300)
            worst = max(worst, float(z.max()))
    print("resampled moments vs moment matching, %d x %d particles, H=%d: worst %.2f standard errors" % (K, P, H, worst))
    assert worst <= 5.0


def test_value_central_difference():
    gp, spec, pol, terms, m0, S0, H, P, mu = _case("linear_squash")
    terms = [t for t in terms if t["kind"] != _lib.REWARD_BOX]
    P = 2000
    x0, eps = _draw(m0, S0, P, H, seed=41)
    xi = np.random.RandomState(42).randn(P, H, m0.shape[0])
    _, g, _ = _run(gp, spec, terms, x0, eps, xi, mu)
    rng = np.random.RandomState(43)
    vW, vb = rng.randn(*spec["W"].shape), rng.randn(*np.shape(spec["b"]))
    gv = float((g["W"].cpu().numpy().reshape(vW.shape) * vW).sum() + (g["b"].cpu().numpy().reshape(vb.shape) * vb).sum())
    h = 1e-5

    def value(s):
        sp = dict(spec, W=spec["W"] + s * vW, b=spec["b"] + s * vb)
        return float(_run(gp, sp, terms, x0, eps, xi, mu)[1]["value"].item())
    cd = (value(h) - value(-h)) / (2 * h)
    print("resampled value: central difference %.12e, g'v %.12e" % (cd, gv))
    assert abs(cd - gv) <= 1e-6 * max(abs(gv), 1e-12)


def test_class_level():
    pilco, X = _linear_pilco()
    a = pilco.sample_trajectories(X[0, :2], 0.01 * np.eye(2), 4, num_samples=64, seed=5)
    b = pilco.sample_trajectories(X[0, :2], 0.01 * np.eye(2), 4, num_samples=64, seed=5, resample=True)
    assert np.array_equal(a.states[:, 0], b.states[:, 0]) and np.array_equal(a.actions[:, 0], b.actions[:, 0])
    x0, eps = pilco._particle_inputs(X[0, :2], 0.01 * np.eye(2), 4, 64, 5, "test")
    x0r, epsr, xi = pilco._particle_inputs(X[0, :2], 0.01 * np.eye(2), 4, 64, 5, "test", True)
    assert torch.equal(x0, x0r) and torch.equal(eps, epsr) and xi.shape == eps.shape
    for kw in (dict(consistent=True), dict(estimator="score"), dict(exploration=0.5)):
        with pytest.raises(ValueError, match="resample"):
            pilco.sample_policy_gradient(X[0, :2], 0.01 * np.eye(2), 4, num_samples=64, seed=5, resample=True, **kw)
    with pytest.raises(ValueError, match="resample"):
        pilco.sample_trajectories(X[0, :2], 0.01 * np.eye(2), 4, num_samples=64, resample=True, consistent=True)
    with pytest.raises(ValueError, match="resample"):
        pilco.optimize_policy_sampled(maxiter=2, num_samples=64, resample=True, consistent=True)
    m, v = pilco.sample_reward_moments(X[0, :2], 0.01 * np.eye(2), 4, num_samples=64, seed=5, resample=True)
    assert np.all(np.isfinite(m)) and np.all(np.isfinite(v))


def test_optimize_policy_sampled_resampled():
    pilco, X, Y = _pilco("linear", 61)
    start = pilco.sample_policy_gradient(pilco.m_init, pilco.S_init, pilco.horizon, num_samples=300, seed=7,
                                         resample=True).value
    value = pilco.optimize_policy_sampled(maxiter=10, restarts=8, num_samples=300, seed=7, resample=True)
    print("resampled optimize_policy_sampled: start %.6f, optimised %.6f" % (start, value))
    assert np.isfinite(value) and value >= start - 1e-12
