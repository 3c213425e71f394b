"""Score-function gradient over consistent function samples on the device (pilco_particles_consistent_score_grad_rollout
through engine.ConsistentGradPlan(estimator="score"), DESIGN.md section 25): parity with the torch oracle
(tests/particle_grad_oracle.py's score_grad(consistent=True)) given the device's trajectories, x0, eps and nu, the
forward outputs and value against the consistent pathwise call, restarts against single calls, bitwise reproducibility
and CUDA-graph replay, H = 2 against section 16's score gradient, unbiasedness against the consistent pathwise gradient,
and box terms against a central difference of the sampled return."""
import numpy as np
import pytest
import torch

from pilco_b200 import engine, _lib
from particle_cases import _angle_case, _batch_case, _box_case, _case, _draw, _dyn_np, _oracle_pol, _seeded
from particle_grad_oracle import score_grad
from util import _zscores

pytestmark = pytest.mark.gpu

CASES = ["metric_rbf", "linear_squash", "linear_nosquash", "fitc", "n1_d16_h0"]
SHAPES = {                                                      # E, dims, U, policy, joint terms, measurement noise
    "angles_a1": (4, [1], 1, "rbf", False, False),
    "angles_a2_noise": (6, [1, 2], 1, "linear", True, True),
    "u2_joint_box": (4, [], 2, "linear", True, False),
}


def _run(gp, spec, terms, x0, eps, mu, estimator="score", R=1, angles=None, v=None, nu=None):
    plan = engine.ConsistentGradPlan(gp, spec, terms, x0.shape[0], eps.shape[1], mult_mu=mu, R=R, angles=angles,
                                     measurement_noise=v, estimator=estimator)
    plan.set_inputs(x0, eps, nu)
    g = {k: t.clone() for k, t in plan.launch_grad().items()}
    return plan, g, [t.clone() for t in plan.outputs()]


def _rel(g, ref):
    scale = max(float(np.abs(r).max()) for r in ref.values())
    if scale == 0.0:
        return 0.0, scale
    return max(float(np.abs(g[k].reshape(ref[k].shape) - ref[k]).max()) for k in ref) / scale, scale


def _parity(gp, spec, pol, terms, x0, eps, mu, angles=None, v=None, nu=None):
    plan, g, out = _run(gp, spec, terms, x0, eps, mu, angles=angles, v=v, nu=nu)
    g = {k: t.cpu().numpy() for k, t in g.items()}
    args = (_dyn_np(gp), _oracle_pol(spec, pol), terms, out[0].cpu().numpy(), eps, mu)
    kw = dict(angle_dims=angles, nu=nu, v=v, consistent=True)
    ref, ratio = score_grad(*args, **kw)
    err, scale = _rel(g, ref)
    own = _rel(score_grad(*args, swap=True, **kw)[0], ref)[0] if scale > 0.0 else 0.0
    return g, ref, err, own, ratio


@pytest.mark.parametrize("name", CASES)
def test_parity_with_oracle(name):
    gp, spec, pol, terms, m0, S0, H, P, mu = _case(name)
    P = min(P, 300)                                             # (the oracle's cost)
    x0, eps = _draw(m0, S0, P, H, seed=P + H + 5)
    g, ref, err, own, ratio = _parity(gp, spec, pol, terms, x0, eps, mu)
    print("consistent score gradient %s (P=%d, H=%d) vs oracle: %.1e of the gradient's scale; the oracle against "
          "itself with its sums reordered: %.1e; smallest pivot d2 / (tau sf2) %.1e" % (name, P, H, err, own, ratio))
    if H < 2:
        assert all(not g[k].any() for k in ref)
    assert err <= max(1e-9, 10.0 * own)


@pytest.mark.parametrize("name", sorted(SHAPES))
def test_parity_with_oracle_angles_noise_joint_terms(name):
    E, dims, U, kind, joint, noisy = SHAPES[name]
    gp, spec, pols, terms = _angle_case(E, dims, U, kind, joint=joint)
    P, H, mu = 200, 6, 1.5
    rng = np.random.RandomState(P + H + E)
    x0, eps, nu = 0.8 * rng.randn(P, E), rng.randn(P, H, E), rng.randn(P, H, E)
    v = 0.01 + 0.03 * rng.rand(E) if noisy else None
    g, ref, err, own, ratio = _parity(gp, spec, pols[0], terms, x0, eps, mu, angles=dims, v=v, nu=nu if noisy else None)
    print("consistent score gradient %s vs oracle: %.1e of the gradient's scale (own %.1e), smallest pivot d2 / "
          "(tau sf2) %.1e" % (name, err, own, ratio))
    assert err <= max(1e-9, 10.0 * own)


@pytest.mark.parametrize("name", ["metric_rbf", "linear_squash", "n1_d16_h0"])
def test_forward_and_value_bitwise_equal_pathwise(name):
    gp, spec, pol, terms, m0, S0, H, P, mu = _case(name)
    x0, eps = _draw(m0, S0, min(P, 500), H, seed=42)
    _, g, out = _run(gp, spec, terms, x0, eps, mu)
    _, gp_, out_p = _run(gp, spec, terms, x0, eps, mu, estimator="pathwise")
    assert all(torch.equal(a, b) for a, b in zip(out, out_p))
    assert torch.equal(g["value"], gp_["value"])
    if H > 1:
        assert any(not torch.equal(g[k], gp_[k]) for k in g if k != "value")


def test_forward_and_value_bitwise_equal_pathwise_with_angles_and_noise():
    E, dims, U, kind, joint, _ = SHAPES["angles_a2_noise"]
    gp, spec, _, terms = _angle_case(E, dims, U, kind, joint=joint)
    rng = np.random.RandomState(7)
    x0, eps, nu = 0.8 * rng.randn(300, E), rng.randn(300, 5, E), rng.randn(300, 5, E)
    v = 0.02 * np.ones(E)
    _, g, out = _run(gp, spec, terms, x0, eps, 1.5, angles=dims, v=v, nu=nu)
    _, gp_, out_p = _run(gp, spec, terms, x0, eps, 1.5, estimator="pathwise", angles=dims, v=v, nu=nu)
    assert all(torch.equal(a, b) for a, b in zip(out, out_p)) and torch.equal(g["value"], gp_["value"])


@pytest.mark.parametrize("kind", ["linear", "rbf"])
def test_restarts_bitwise_equal_single_calls(kind):
    gp, spec, singles, terms, m0, S0, H, P, mu = _batch_case(kind, 3)
    x0, eps = _draw(m0, S0, P, H, seed=43)
    _, g, out = _run(gp, spec, terms, x0, eps, mu, R=3)
    assert g["value"].shape == (3,)
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
    for v in list(plan.gbuf.values()) + [plan.traj, plan.ret, plan.gws]:
        v.zero_()
    graph.replay()
    torch.cuda.synchronize()
    assert all(torch.equal(first[k], plan.gbuf[k]) for k in first)
    assert torch.equal(out[0], plan.traj) and torch.equal(out[4], plan.ret)


@pytest.mark.parametrize("name", ["metric_rbf", "linear_squash"])
def test_two_steps_is_the_step_wise_score_gradient(name):
    """H = 2: step 0 is the same transition in both samplers, and the cotangents are bitwise ps_cot_kernel's; the two
    calls are different VJP siblings, so they agree to rounding.  The score gradient is a sum over particles that
    cancels strongly, which amplifies rounding: the bar is 1e-12 of scale or ten times the distance of section 16's call
    from its oracle (particle_grad_oracle.score_grad) on the same particles, whichever is larger"""
    gp, spec, pol, terms, m0, S0, H, P, mu = _case(name)
    x0, eps = _draw(m0, S0, P, 2, seed=45)
    _, g, out = _run(gp, spec, terms, x0, eps, mu)
    plan = engine.ParticlePlan(gp, spec, terms, P, 2, mult_mu=mu, grad=True, estimator="score")
    plan.set_inputs(x0, eps)
    ref = {k: t.cpu().numpy() for k, t in plan.launch_grad().items() if k != "value"}
    err, scale = _rel({k: t.cpu().numpy() for k, t in g.items()}, ref)
    own = _rel(ref, score_grad(_dyn_np(gp), _oracle_pol(spec, pol), terms, plan.traj.cpu().numpy(), eps, mu))[0]
    print("H = 2 %s: consistent score vs step-wise score gradient %.1e of scale (the step-wise call against its oracle: "
          "%.1e)" % (name, err, own))
    assert torch.equal(out[0][:, :2], plan.traj[:, :2])          # step 0 is the same transition, bitwise
    assert scale > 0.0 and err <= max(1e-12, 10.0 * own)


def test_expected_gradient_is_the_consistent_pathwise_gradient():
    """the metric case at H = 10 without box terms, paired over 16 x 2^12 particles"""
    gp, spec, pol, terms, m0, S0, H, P, mu = _case("metric_rbf")
    terms = [t for t in terms if t["kind"] != _lib.REWARD_BOX]
    P = 1 << 12
    plans = {e: engine.ConsistentGradPlan(gp, spec, terms, P, H, mult_mu=mu, estimator=e) for e in ("score", "pathwise")}
    draws = {e: {k: [] for k in ("X", "Y", "ell")} for e in plans}
    for s in range(16):
        x0, eps = _seeded(P, H, spec["Ds"], m0, S0, 500 + s)
        for e, plan in plans.items():
            plan.x0.copy_(x0); plan.eps_buf.copy_(eps)
            g = plan.launch_grad()
            for k in draws[e]:
                draws[e][k].append(g[k].cpu().numpy().copy())
        if s == 0:                                              # the pivots of a subset, from the oracle
            sub = 200
            ratio = score_grad(_dyn_np(gp), _oracle_pol(spec, pol), terms, plans["score"].traj[:sub].cpu().numpy(),
                               eps[:sub].cpu().numpy(), mu, consistent=True)[1]
    worst = _zscores(draws["score"], draws["pathwise"])
    print("consistent score vs pathwise gradient, paired over 16 x 2^12 particles: worst %.2f standard errors; "
          "smallest pivot d2 / (tau sf2) over %d particles %.1e" % (worst, sub, ratio))
    assert ratio > 1e2 and worst <= 5.0


def test_box_terms_central_difference_of_sampled_return():
    gp, spec, terms, m0, S0, H, mu = _box_case()
    P, K, h = 1 << 14, 16, 1e-2                                 # 2^18 particles in all
    rng = np.random.RandomState(49)
    vW, vb = rng.randn(*spec["W"].shape), rng.randn(*spec["b"].shape)
    plans = {e: engine.ConsistentGradPlan(gp, spec, terms, P, H, mult_mu=mu, estimator=e) for e in ("score", "pathwise")}
    shifted = [engine.ParticlePlan(gp, dict(spec, W=spec["W"] + s * h * vW, b=spec["b"] + s * h * vb), terms, P, H,
                                   mult_mu=mu, consistent=True) for s in (1.0, -1.0)]
    diffs, active = {e: [] for e in plans}, 0.0
    for k in range(K):
        x0, eps = _seeded(P, H, 4, m0, S0, 600 + k)
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
        print("consistent box terms, %s: central difference - g'v = %.3e +- %.3e (%.2f combined standard errors), "
              "mean risk %.3f" % (e, d.mean(), d.std(ddof=1) / np.sqrt(K), zs[e], active / K))
    assert 0.0 < active / K < 1.0
    assert zs["score"] <= 4.0
    assert zs["pathwise"] > 4.0                                 # the check tells the biased estimate (no box) apart
