"""The consistent sampler's pathwise gradient on the device (pilco_particles_rollout_consistent_grad through
engine.ConsistentGradPlan, PILCO.sample_policy_gradient / optimize_policy_sampled(..., consistent=True)): forward
outputs bitwise those of pilco_particles_rollout_consistent, parity with the torch autograd oracle
(tests/consistent_grad_oracle.py) given the same x0 and eps, a directional central difference of the device value, a
finite gradient at a revisited input, batched restarts bitwise equal to unbatched calls, bitwise reproducibility and
CUDA-graph replay, the workspace budget, and the class API."""
from functools import partial

import numpy as np
import pytest
import torch

from pilco_b200 import engine, _lib, policy_opt
from consistent_grad_oracle import value_and_grad
from test_gpu_particles import _case, _draw, _dyn_np, _pilco_data
from test_gpu_particles_consistent import _revisit_problem
from test_gpu_particles_grad import _oracle_pol
from test_gpu_particles_opt import _batch_case, _pilco
from util import make_rollout_problem

pytestmark = pytest.mark.gpu

CASES = ["metric_rbf", "linear_squash", "linear_nosquash", "fitc", "n1_d16_h0"]


def _grad_run(gp, spec, terms, x0, eps, mu, R=1):
    plan = engine.ConsistentGradPlan(gp, spec, terms, x0.shape[0], eps.shape[1], mult_mu=mu, R=R)
    plan.set_inputs(x0, eps)
    g = {k: v.clone() for k, v in plan.launch_grad().items()}
    return plan, g, [t.clone() for t in plan.outputs()]


@pytest.mark.parametrize("name", CASES)
def test_forward_outputs_bitwise_equal_consistent_rollout(name):
    gp, spec, pol, terms, m0, S0, H, P, mu = _case(name)
    x0, eps = _draw(m0, S0, P, H, seed=P + H + 2)
    _, _, out = _grad_run(gp, spec, terms, x0, eps, mu)
    ref = engine.particles_rollout(gp, spec, terms, x0, eps, mult_mu=mu, consistent=True)
    for what, a, b in zip(("traj", "act", "step_reward", "step_risk", "ret"), out, ref):
        assert torch.equal(a, b), what


@pytest.mark.parametrize("name", CASES)
def test_parity_with_autograd_oracle(name):
    gp, spec, pol, terms, m0, S0, H, P, mu = _case(name)
    P = min(P, 300)                                             # (the oracle's cost)
    x0, eps = _draw(m0, S0, P, H, seed=P + H + 3)
    _, g, _ = _grad_run(gp, spec, terms, x0, eps, mu)
    g = {k: v.cpu().numpy() for k, v in g.items()}
    args = (_dyn_np(gp), _oracle_pol(spec, pol), terms, x0, eps, mu)
    v, ref, ratio = value_and_grad(*args)
    scale = max(float(np.abs(r).max()) for r in ref.values())
    if scale == 0.0:                                            # H = 0: nothing depends on the policy
        assert all(not g[k].any() for k in ref)
        err = own = 0.0
    else:
        err = max(float(np.abs(g[k].reshape(ref[k].shape) - ref[k]).max()) for k in ref) / scale
        _, sw, _ = value_and_grad(*args, swap=True)
        own = max(float(np.abs(sw[k] - ref[k]).max()) for k in ref) / scale
    verr = abs(float(g["value"][0]) - v) / max(abs(v), 1e-300)
    print("consistent gradient %s (P=%d, H=%d) vs autograd oracle: %.1e of the gradient's scale, value %.1e; the "
          "oracle against itself with its sums reordered: %.1e; smallest pivot d2 / (tau sf2) %.1e"
          % (name, P, H, err, verr, own, ratio))
    # the bar of DESIGN.md section 14: 1e-9 of scale or ten times the oracle's own sensitivity to rounding
    assert err <= max(1e-9, 10.0 * own) and verr <= max(1e-9, 10.0 * own)


def test_directional_finite_difference_of_device_value():
    """the metric RBF problem, whose smallest pivot is about 1e5 tau sf2: the draw is well conditioned"""
    pb = make_rollout_problem(300, 10, 2, 50, 1, seed=5)
    gp = engine.gp_factorize(pb["X"], pb["Y"], pb["ell"], pb["sf2"], pb["sn2"])
    terms = [t for t in _case("metric_rbf")[3] if t["kind"] != _lib.REWARD_BOX]
    Xc, Yc, lc = pb["Xc"][0], pb["Yc"][0], pb["lc"][0]
    U, H, P, mu = Yc.shape[1], 10, 1000, 1.5
    x0, eps = _draw(pb["m0"], pb["S0"], P, H, seed=41)

    def run(Xc, Yc, lc):
        pgp = engine.gp_factorize(Xc, Yc, lc, np.ones(U), 1e-4 * np.ones(U), need_iK=False, mode=1)
        spec = dict(kind=_lib.POLICY_RBF, Ds=10, U=U, squash=True, max_action=pb["maxa"], gp=pgp)
        return {k: v.cpu().numpy() for k, v in _grad_run(gp, spec, terms, x0, eps, mu)[1].items()}
    g = run(Xc, Yc, lc)
    rng = np.random.RandomState(42)
    v = {k: rng.randn(*g[k].shape) for k in ("X", "Y", "ell")}
    h = 1e-5
    vp = run(Xc + h * v["X"], Yc + h * v["Y"], lc + h * v["ell"])["value"][0]
    vm = run(Xc - h * v["X"], Yc - h * v["Y"], lc - h * v["ell"])["value"][0]
    fd = (vp - vm) / (2 * h)
    gv = sum(float((g[k] * v[k]).sum()) for k in v)
    print("consistent directional derivative: central difference %.12e, g'v %.12e, rel %.1e"
          % (fd, gv, abs(fd - gv) / abs(gv)))
    # the value carries the sampler's rounding sensitivity (about 1e-11 relative, DESIGN.md section 14), which over
    # 2h limits the central difference to a few 1e-6; the tight check is the autograd parity above
    assert abs(fd - gv) <= 1e-5 * abs(gv)


def test_revisited_input_gives_a_finite_gradient():
    """every step of a particle has the same input (the degenerate pivots of DESIGN.md section 14): the tau rule holds
    their own noise constant, so the gradient stays finite"""
    H = 20
    gp, spec, terms, x0, eps = _revisit_problem(H, 1024, seed=43)
    spec = dict(spec, b=np.array([1.2]))            # a constant action 5 sin(1.2), still outside the data's range
    plan, g, out = _grad_run(gp, spec, terms, x0, eps, 0.0)
    print("revisited input: value %.6e, |grad W| %.3e, |grad b| %.3e"
          % (float(g["value"][0]), float(g["W"].abs().max()), float(g["b"].abs().max())))
    assert all(bool(torch.isfinite(v).all()) for v in g.values()) and bool(torch.isfinite(out[0]).all())
    assert float(g["b"].abs().max()) > 0.0


@pytest.mark.parametrize("kind,R", [("rbf", 1), ("rbf", 3), ("rbf", 5), ("linear", 3), ("linear", 5), ("fitc", 3)])
def test_batched_restarts_bitwise_equal_unbatched(kind, R):
    gp, spec, singles, terms, m0, S0, H, P, mu = _batch_case(kind, R)
    x0, eps = _draw(m0, S0, P, H, seed=44)
    _, g, out = _grad_run(gp, spec, terms, x0, eps, mu, R=R)
    assert g["value"].shape == (R,) and out[0].shape == (R, P, H + 1, spec["Ds"])
    for r in range(R):
        _, g1, out1 = _grad_run(gp, singles[r], terms, x0, eps, mu)
        for what, a, b in zip(("traj", "act", "step_reward", "step_risk", "ret"), out, out1):
            assert torch.equal(a[r], b), (r, what)
        for k in g1:
            assert torch.equal(g[k][r], g1[k].reshape(g[k][r].shape)), (r, k)
    assert len(set(float(v) for v in g["value"])) == R


def test_shared_policy_array_with_zero_stride():
    gp, spec, singles, terms, m0, S0, H, P, mu = _batch_case("linear", 3)
    x0, eps = _draw(m0, S0, P, H, seed=45)
    plan = engine.ConsistentGradPlan(gp, spec, terms, P, H, mult_mu=mu, R=3)
    plan.set_inputs(x0, eps)
    plan.pr.pol.b_bs = 0                                         # every restart uses b[0]
    g = plan.launch_grad()
    for r in range(3):
        _, g1, out1 = _grad_run(gp, dict(singles[r], b=spec["b"][0]), terms, x0, eps, mu)
        assert torch.equal(plan.ret[r], out1[4]) and torch.equal(g["W"][r], g1["W"])


def test_run_to_run_and_graph_replay_are_bitwise_equal():
    gp, spec, pol, terms, m0, S0, H, P, mu = _case("metric_rbf")
    x0, eps = _draw(m0, S0, P, H, seed=46)
    plan, first, out = _grad_run(gp, spec, terms, x0, eps, mu)
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


def test_workspace_budget_is_checked_before_any_launch():
    gp, spec, pol, terms, m0, S0, H, P, mu = _case("linear_squash")
    need = engine.ConsistentGradPlan(gp, spec, terms, 100, H, mult_mu=mu).gws.numel() * 8
    with pytest.raises(ValueError, match=r"num_samples=\d+ would fit"):
        engine.ConsistentGradPlan(gp, spec, terms, 1000, H, mult_mu=mu, max_ws_bytes=need)
    with pytest.raises(ValueError, match="gradient"):
        engine.ParticlePlan(gp, spec, terms, P, H, grad=True, consistent=True)


def test_sample_policy_gradient_consistent_class_api():
    from pilco.models import PILCO
    from pilco.controllers import RbfController
    np.random.seed(47)
    X, Y = _pilco_data(47)
    pilco = PILCO((X[:60], Y[:60]), controller=RbfController(3, 1, 10, max_action=1.2), horizon=6)
    m, S = X[0, :3], 0.05 * np.eye(3)
    a = pilco.sample_policy_gradient(m, S, 6, num_samples=300, seed=5, consistent=True)
    tr = pilco.sample_trajectories(m, S, 6, num_samples=300, seed=5, consistent=True)
    assert np.array_equal(a.returns, tr.returns)
    assert abs(a.value - tr.returns.mean()) <= 1e-14 * abs(tr.returns.mean())
    assert a.grad.shape == pilco.controller.get_flat().shape and np.all(np.isfinite(a.grad))
    b = pilco.sample_policy_gradient(m, S, 6, num_samples=300, seed=5, consistent=True)
    assert np.array_equal(a.grad, b.grad)
    marg = pilco.sample_policy_gradient(m, S, 6, num_samples=300, seed=5)
    assert not np.array_equal(a.grad, marg.grad)
    cos = float(a.grad @ marg.grad / (np.linalg.norm(a.grad) * np.linalg.norm(marg.grad)))
    print("cosine between the consistent and step-wise particle gradients: %.3f" % cos)
    pilco.mgpr.set_data((X, Y))                                 # appended data: the updated factorisation
    c = pilco.sample_policy_gradient(m, S, 6, num_samples=300, seed=5, consistent=True)
    assert pilco.mgpr.last_update == "append" and not np.array_equal(c.grad, a.grad) and np.all(np.isfinite(c.grad))
    assert np.array_equal(c.returns, pilco.sample_trajectories(m, S, 6, num_samples=300, seed=5, consistent=True).returns)


def test_sample_policy_gradient_consistent_smgpr_and_safe_pilco():
    from pilco.models import PILCO
    from pilco.controllers import LinearController
    from safe_pilco_extension.safe_pilco import SafePILCO
    from safe_pilco_extension.rewards_safe import RiskOfCollision
    from pilco.rewards import LinearReward
    np.random.seed(48)
    X, Y = _pilco_data(48, n=300, Ds=4)
    sp = PILCO((X, Y), num_induced_points=40, controller=LinearController(4, 1), horizon=5)
    res = sp.sample_policy_gradient(X[0, :4], 0.05 * np.eye(4), 5, num_samples=100, seed=2, consistent=True)
    assert res.grad.shape == (5,) and np.all(np.isfinite(res.grad))
    pilco = SafePILCO((X, Y), controller=LinearController(4, 1), horizon=5, reward_add=LinearReward(4, np.ones(4)),
                      reward_mult=RiskOfCollision(4, [0.0, 0.1], [0.6, 0.9]), mu=-4.0)
    res = pilco.sample_policy_gradient(X[0, :4], 0.05 * np.eye(4), 5, num_samples=300, seed=3, consistent=True)
    tr = pilco.sample_trajectories(X[0, :4], 0.05 * np.eye(4), 5, num_samples=300, seed=3, consistent=True)
    assert np.array_equal(res.returns, tr.returns) and tr.risks.any()      # box terms: in the value only
    assert abs(res.value - tr.returns.mean()) <= 1e-14 * abs(tr.returns.mean())
    assert np.all(np.isfinite(res.grad))


def _start_values(pilco, flats0, P, seed):
    x0, eps = pilco._particle_inputs(pilco.m_init, pilco.S_init, pilco.horizon, P, seed, "test")
    loss, _ = policy_opt.ParticleEvaluator(pilco, flats0.shape[0], x0, eps, consistent=True)(flats0)
    return -loss, x0, eps


@pytest.mark.parametrize("kind", ["rbf", "linear"])
def test_optimize_policy_sampled_consistent(kind):
    pilco, _, _ = _pilco(kind, 49)
    P, seed, restarts, maxiter = 300, 13, 3, 30
    state = np.random.get_state()
    flats0 = policy_opt.initial_flats(pilco.controller, restarts)
    start, x0, eps = _start_values(pilco, flats0, P, seed)
    best_flat, best, finals = policy_opt.optimize(
        pilco, maxiter=maxiter, restarts=restarts, flats0=flats0,
        evaluator=partial(policy_opt.ParticleEvaluator, x0=x0, eps=eps, consistent=True))
    finals = np.asarray(finals)
    print("%s consistent: sampled value per restart %s -> %s, best %.6f" % (kind, start, finals, best))
    assert np.all(finals >= start) and best == finals.max()
    np.random.set_state(state)
    pilco.controller.set_flat(flats0[0])
    value = pilco.optimize_policy_sampled(maxiter=maxiter, restarts=restarts, num_samples=P, seed=seed, consistent=True)
    assert value == best and value >= start[0]
    held = pilco.sample_policy_gradient(pilco.m_init, pilco.S_init, pilco.horizon, num_samples=P, seed=seed,
                                        consistent=True).value
    assert abs(held - best) <= 1e-12 * abs(best)
    assert pilco.mgpr.models[0].kernel.lengthscales.trainable


def test_optimize_policy_sampled_consistent_smgpr():
    from pilco.models import PILCO
    from pilco.controllers import LinearController
    np.random.seed(50)
    X, Y = _pilco_data(50, n=300, Ds=4)
    sp = PILCO((X, Y), num_induced_points=40, controller=LinearController(4, 1), horizon=5)
    f0 = sp.controller.get_flat()[None]
    start = _start_values(sp, f0, 200, 3)[0][0]
    value = sp.optimize_policy_sampled(maxiter=10, restarts=2, num_samples=200, seed=3, consistent=True)
    print("SMGPR consistent: sampled value %.6f -> %.6f" % (start, value))
    assert np.isfinite(value) and value >= start
