"""Score-function gradient of the particle return on the device (pilco_particles_rollout_score_grad through
engine.ParticlePlan(estimator="score") and PILCO.sample_policy_gradient(estimator="score")): parity with the torch
oracle given the device's trajectories, x0 and eps (tests/score_grad_oracle.py), the forward outputs and value against
the pathwise call, restarts against single calls, bitwise reproducibility and CUDA-graph replay, a call past one VJP
call's row limit, unbiasedness against the moment-matching and pathwise gradients, box terms against a central
difference of the sampled return, and the class API."""
import numpy as np
import pytest
import torch

from pilco_b200 import engine, _lib
from score_grad_oracle import score_grad
from test_gpu_particles import BOX2, _case, _draw, _dyn_np, _pilco_data
from test_gpu_particles_grad import _oracle_pol
from test_gpu_particles_opt import _batch_case
from util import make_gp_problem, make_rollout_problem

pytestmark = pytest.mark.gpu


def _run(gp, spec, terms, x0, eps, mu, estimator="score", R=1):
    plan = engine.ParticlePlan(gp, spec, terms, x0.shape[0], eps.shape[1], mult_mu=mu, grad=True, R=R,
                               estimator=estimator)
    plan.set_inputs(x0, eps)
    g = {k: v.clone() for k, v in plan.launch_grad().items()}
    return plan, g, [t.clone() for t in plan.outputs()]


def _parity(gp, spec, pol, terms, x0, eps, mu):
    plan, g, out = _run(gp, spec, terms, x0, eps, mu)
    ref = score_grad(_dyn_np(gp), _oracle_pol(spec, pol), terms, out[0].cpu().numpy(), eps, mu)
    g = {k: v.cpu().numpy() for k, v in g.items()}
    scale = max(float(np.abs(r).max()) for r in ref.values())
    if scale == 0.0:
        return g, ref, 0.0
    return g, ref, max(float(np.abs(g[k] - ref[k]).max()) for k in ref) / scale


@pytest.mark.parametrize("name", ["metric_rbf", "linear_squash", "linear_nosquash", "fitc", "n1_d16_h0"])
def test_parity_with_score_oracle(name):
    gp, spec, pol, terms, m0, S0, H, P, mu = _case(name)
    x0, eps = _draw(m0, S0, P, H, seed=P + H + 2)
    g, ref, err = _parity(gp, spec, pol, terms, x0, eps, mu)
    print("score gradient %s (P=%d, H=%d) vs oracle: %.1e of the gradient's scale" % (name, P, H, err))
    if H < 2:
        assert all(not g[k].any() for k in ref)
    assert err <= (1e-6 if name == "fitc" else 1e-8)


def test_parity_at_one_particle_and_zero_at_one_step():
    gp, spec, pol, terms, m0, S0, H, P, mu = _case("linear_squash")
    x0, eps = _draw(m0, S0, 1, H, seed=40)                      # P = 1: no baseline, w = G
    g, ref, err = _parity(gp, spec, pol, terms, x0, eps, mu)
    print("score gradient at P = 1 vs oracle: %.1e of the gradient's scale" % err)
    assert err <= 1e-8 and any(ref[k].any() for k in ref)
    for name in ("linear_squash", "metric_rbf"):                # H = 1: no transition can move a reward
        gp, spec, pol, terms, m0, S0, H, P, mu = _case(name)
        x0, eps = _draw(m0, S0, P, 1, seed=41)
        _, g, out = _run(gp, spec, terms, x0, eps, mu)
        _, gp_, out_p = _run(gp, spec, terms, x0, eps, mu, estimator="pathwise")
        assert all(not g[k].any() for k in g if k != "value")
        assert torch.equal(g["value"], gp_["value"]) and all(torch.equal(a, b) for a, b in zip(out, out_p))


@pytest.mark.parametrize("name", ["metric_rbf", "linear_squash"])
def test_forward_and_value_bitwise_equal_pathwise(name):
    gp, spec, pol, terms, m0, S0, H, P, mu = _case(name)
    x0, eps = _draw(m0, S0, P, H, seed=42)
    _, g, out = _run(gp, spec, terms, x0, eps, mu)
    _, gp_, out_p = _run(gp, spec, terms, x0, eps, mu, estimator="pathwise")
    assert all(torch.equal(a, b) for a, b in zip(out, out_p))
    assert torch.equal(g["value"], gp_["value"])
    assert any(not torch.equal(g[k], gp_[k]) for k in g if k != "value")


@pytest.mark.parametrize("kind", ["linear", "rbf"])
def test_restarts_bitwise_equal_single_calls(kind):
    gp, spec, singles, terms, m0, S0, H, P, mu = _batch_case(kind, 3)
    x0, eps = _draw(m0, S0, P, H, seed=43)
    _, g, out = _run(gp, spec, terms, x0, eps, mu, R=3)
    _, gpath, out_p = _run(gp, spec, terms, x0, eps, mu, R=3, estimator="pathwise")
    assert all(torch.equal(a, b) for a, b in zip(out, out_p)) and torch.equal(g["value"], gpath["value"])
    for r in range(3):
        _, g1, out1 = _run(gp, singles[r], terms, x0, eps, mu)
        for what, a, b in zip(("traj", "act", "step_reward", "step_risk", "ret"), out, out1):
            assert torch.equal(a[r], b), (r, what)
        for k in g1:
            assert torch.equal(g[k][r], g1[k].reshape(g[k][r].shape)), (r, k)


def test_run_to_run_and_graph_replay_are_bitwise_equal():
    gp, spec, pol, terms, m0, S0, H, P, mu = _case("metric_rbf")
    x0, eps = _draw(m0, S0, P, H, seed=44)
    plan, first, out = _run(gp, spec, terms, x0, eps, mu)
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


def test_past_one_vjp_call_agrees_with_oracle():
    """39 steps x 60000 rows are more than one pilco_gp_predict_vjp call takes (65535 * 32 rows): two groups"""
    X, Y, ell, sf2, sn2 = make_gp_problem(20, 3, 2, seed=45)
    gp = engine.gp_factorize(X, 0.1 * Y, ell, 0.1 * sf2, 1e-3 * np.ones(2))
    rng = np.random.RandomState(46)
    W, b = 0.5 * rng.randn(1, 2), rng.randn(1)
    spec = dict(kind=_lib.POLICY_LINEAR, Ds=2, U=1, squash=True, max_action=np.array([1.1]), W=W, b=b)
    pol = dict(kind=_lib.POLICY_LINEAR, squash=True, maxa=np.array([1.1]), W=W, b=b)
    terms = [dict(kind=_lib.REWARD_EXP, coef=1.0, W=np.eye(2), t=0.5 * np.ones(2)),
             dict(kind=_lib.REWARD_LINEAR, coef=0.2, W=np.ones(2), t=None)]
    P, H = 60000, 40
    assert P * (H - 1) > 65535 * 32
    x0, eps = _draw(X[0, :2], 0.05 * np.eye(2), P, H, seed=47)
    g, ref, err = _parity(gp, spec, pol, terms, x0, eps, 0.0)
    print("score gradient P=%d H=%d (two VJP calls) vs oracle: %.1e of the gradient's scale" % (P, H, err))
    assert err <= 1e-8


def _seeded(P, H, Ds, m0, S0, seed):
    d = engine.device()
    gen = torch.Generator(device=d)
    gen.manual_seed(seed)
    F = engine.dev(np.linalg.cholesky(S0))
    x0 = engine.dev(m0)[None] + torch.randn((P, Ds), dtype=engine.F64, device=d, generator=gen) @ F.T
    return x0, torch.randn((P, H, Ds), dtype=engine.F64, device=d, generator=gen)


def _zscores(a, b=None, ref=None):
    """largest |mean| / standard error of a - b (paired draws) or of a against the constant ref"""
    worst = 0.0
    for k in a:
        d = np.stack(a[k]) - (np.stack(b[k]) if b is not None else ref[k])
        worst = max(worst, float(np.max(np.abs(d.mean(0)) / (d.std(0, ddof=1) / np.sqrt(d.shape[0])))))
    return worst


def test_expected_score_gradient_is_the_moment_matching_gradient():
    """Linear unsquashed policy, one linear reward, H = 2, where moment matching is exact (as the pathwise test)"""
    pb = make_rollout_problem(200, 4, 1, 10, 1, seed=23)
    gp = engine.gp_factorize(pb["X"], pb["Y"], pb["ell"], pb["sf2"], pb["sn2"])
    rng = np.random.RandomState(24)
    spec = dict(kind=_lib.POLICY_LINEAR, Ds=4, U=1, squash=False, max_action=np.ones(1), W=0.5 * rng.randn(1, 4),
                b=0.1 * rng.randn(1))
    terms = [dict(kind=_lib.REWARD_LINEAR, coef=1.0, W=rng.randn(4), t=None)]
    m0, S0 = pb["m0"], 0.05 * np.eye(4)
    plan = engine.RolloutPlan(gp, spec, terms, m0, S0, 2, R=1, grad=True)
    plan.forward()
    mm = {k: v[0].cpu().numpy() for k, v in plan.backward().items() if k in ("W", "b")}
    P = 1 << 14
    pp = engine.ParticlePlan(gp, spec, terms, P, 2, grad=True, estimator="score")
    draws = {k: [] for k in mm}
    for s in range(16):
        x0, eps = _seeded(P, 2, 4, m0, S0, 100 + s)
        pp.x0.copy_(x0); pp.eps_buf.copy_(eps)
        g = pp.launch_grad()
        for k in draws:
            draws[k].append(g[k].cpu().numpy().copy())
    worst = _zscores(draws, ref=mm)
    print("score gradient (16 x 2^14 particles) vs moment matching: worst %.2f standard errors" % worst)
    assert worst <= 5.0


def test_expected_score_gradient_is_the_expected_pathwise_gradient():
    gp, spec, pol, terms, m0, S0, H, P, mu = _case("metric_rbf")
    terms = [t for t in terms if t["kind"] != _lib.REWARD_BOX]  # smooth terms: the pathwise estimate is unbiased
    P = 1 << 12
    plans = {e: engine.ParticlePlan(gp, spec, terms, P, H, mult_mu=mu, grad=True, estimator=e)
             for e in ("score", "pathwise")}
    draws = {e: {k: [] for k in ("X", "Y", "ell")} for e in plans}
    for s in range(16):
        x0, eps = _seeded(P, H, spec["Ds"], m0, S0, 200 + s)
        for e, plan in plans.items():
            plan.x0.copy_(x0); plan.eps_buf.copy_(eps)
            g = plan.launch_grad()
            for k in draws[e]:
                draws[e][k].append(g[k].cpu().numpy().copy())
    worst = _zscores(draws["score"], draws["pathwise"])
    print("score vs pathwise gradient, paired over 16 x 2^12 particles: worst %.2f standard errors" % worst)
    assert worst <= 5.0


def _box_case():
    """SafePILCO-like: a linear policy, a linear additive reward and one box as the only MULT term"""
    X, Y, ell, sf2, sn2 = make_gp_problem(100, 5, 4, seed=6)
    gp = engine.gp_factorize(X, 0.1 * Y, ell, 0.1 * sf2, 1e-3 * np.ones(4))
    rng = np.random.RandomState(48)
    W, b = 0.5 * rng.randn(1, 4), rng.randn(1)
    spec = dict(kind=_lib.POLICY_LINEAR, Ds=4, U=1, squash=True, max_action=np.array([1.3]), W=W, b=b)
    terms = [dict(kind=_lib.REWARD_LINEAR, coef=0.3, W=rng.randn(4), t=None),
             dict(kind=_lib.REWARD_BOX, coef=1.0, channel=_lib.CHANNEL_MULT, W=BOX2, t=None)]
    return gp, spec, terms, X[0, :4], 0.05 * np.eye(4), 6, -4.0


def test_box_terms_central_difference_of_sampled_return():
    gp, spec, terms, m0, S0, H, mu = _box_case()
    P, K, h = 1 << 14, 16, 2e-3                                 # 2^18 particles in all
    rng = np.random.RandomState(49)
    vW, vb = rng.randn(*spec["W"].shape), rng.randn(*spec["b"].shape)
    plans = {e: engine.ParticlePlan(gp, spec, terms, P, H, mult_mu=mu, grad=True, estimator=e)
             for e in ("score", "pathwise")}
    shifted = [engine.ParticlePlan(gp, dict(spec, W=spec["W"] + s * h * vW, b=spec["b"] + s * h * vb), terms, P, H,
                                   mult_mu=mu) for s in (1.0, -1.0)]
    diffs, active = {e: [] for e in plans}, 0.0
    for k in range(K):
        x0, eps = _seeded(P, H, 4, m0, S0, 300 + k)
        vals = []
        for sp in shifted:
            sp.set_inputs(x0, eps)
            sp.launch()
            vals.append(float(sp.ret.mean()))
        for e, plan in plans.items():
            plan.x0.copy_(x0); plan.eps_buf.copy_(eps)
            g = plan.launch_grad()
            gv = float((g["W"].cpu().numpy() * vW).sum() + (g["b"].cpu().numpy() * vb).sum())
            diffs[e].append((vals[0] - vals[1]) / (2 * h) - gv)
        active += float(plans["score"].risk_buf.mean())
    zs = {}
    for e, d in diffs.items():
        d = np.array(d)
        zs[e] = abs(d.mean()) / (d.std(ddof=1) / np.sqrt(K))
        print("box terms, %s: central difference - g'v = %.3e +- %.3e (%.2f combined standard errors), mean risk %.3f"
              % (e, d.mean(), d.std(ddof=1) / np.sqrt(K), zs[e], active / K))
    assert 0.0 < active / K < 1.0
    assert zs["score"] <= 4.0
    assert zs["pathwise"] > 4.0                                 # the check tells the biased estimate (no box) apart


def test_removing_the_box_term_moves_only_the_score_gradient():
    gp, spec, terms, m0, S0, H, mu = _box_case()
    x0, eps = _draw(m0, S0, 2000, H, seed=50)
    res = {}
    for name, tt in (("with", terms), ("without", terms[:1])):
        for e in ("score", "pathwise"):
            res[name, e] = _run(gp, spec, tt, x0, eps, mu, estimator=e)[1]
    assert all(torch.equal(res["with", "pathwise"][k], res["without", "pathwise"][k]) for k in ("W", "b"))
    assert not torch.equal(res["with", "score"]["W"], res["without", "score"]["W"])


def _check_class(pilco, m, S, n, S_, seed):
    a = pilco.sample_policy_gradient(m, S, n, num_samples=S_, seed=seed, estimator="score")
    p = pilco.sample_policy_gradient(m, S, n, num_samples=S_, seed=seed)
    assert np.array_equal(a.returns, p.returns) and a.value == p.value
    assert a.grad.shape == pilco.controller.get_flat().shape and np.all(np.isfinite(a.grad))
    assert not np.array_equal(a.grad, p.grad)
    b = pilco.sample_policy_gradient(m, S, n, num_samples=S_, seed=seed, estimator="score")
    assert np.array_equal(a.grad, b.grad)
    return a, p


def test_class_api():
    from pilco.models import PILCO
    from pilco.controllers import RbfController
    np.random.seed(26)
    X, Y = _pilco_data(26)
    pilco = PILCO((X[:60], Y[:60]), controller=RbfController(3, 1, 10, max_action=1.2), horizon=6)
    _check_class(pilco, X[0, :3], 0.05 * np.eye(3), 6, 300, 5)


def test_smgpr_and_safe_pilco():
    from pilco.models import PILCO
    from pilco.controllers import LinearController
    from safe_pilco_extension.safe_pilco import SafePILCO
    from safe_pilco_extension.rewards_safe import RiskOfCollision
    from pilco.rewards import LinearReward
    np.random.seed(27)
    X, Y = _pilco_data(27, n=300, Ds=4)
    sp = PILCO((X, Y), num_induced_points=40, controller=LinearController(4, 1), horizon=5)
    _check_class(sp, X[0, :4], 0.05 * np.eye(4), 5, 100, 2)
    pilco = SafePILCO((X, Y), controller=LinearController(4, 1), horizon=5, reward_add=LinearReward(4, np.ones(4)),
                      reward_mult=RiskOfCollision(4, [0.0, 0.1], [0.6, 0.9]), mu=-4.0)
    _check_class(pilco, X[0, :4], 0.05 * np.eye(4), 5, 300, 3)
