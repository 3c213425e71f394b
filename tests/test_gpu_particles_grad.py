"""Pathwise gradient of the particle return on the device (pilco_particles_rollout_grad through
engine.ParticlePlan(grad=True) and PILCO.sample_policy_gradient; pilco_gp_predict_vjp through engine.gp_predict_vjp):
the predict VJP against its closed form on the device factors, parity with the torch autograd oracle given the same x0
and eps (tests/particle_grad_oracle.py), the forward outputs against pilco_particles_rollout, a directional finite
difference of the device value, the link to the moment-matching gradient where moment matching is exact, bitwise
reproducibility and CUDA-graph replay, and the class API."""
import numpy as np
import pytest
import torch

from pilco_b200 import engine, _lib
from particle_grad_oracle import predict_vjp, value_and_grad
from particle_cases import _case, _draw, _dyn_np, _oracle_pol, _pilco_data
from util import make_gp_problem, make_rollout_problem

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("n,D,E,T", [(1, 1, 1, 1), (37, 3, 2, 30), (37, 16, 3, 4099), (300, 12, 10, 1000),
                                     (300, 1, 16, 30), (600, 16, 16, 4099), (2000, 12, 4, 1000), (2000, 3, 2, 4099)])
def test_predict_vjp_against_closed_form(n, D, E, T):
    X, Y, ell, sf2, sn2 = make_gp_problem(n, D, E, seed=n + D)
    gp = engine.gp_factorize(X, Y, ell, sf2, sn2)
    rng = np.random.RandomState(T)
    Xs, gm, gv = rng.rand(T, D) * 1.4 - 0.2, rng.randn(T, E), rng.randn(T, E)
    out = engine.gp_predict_vjp(gp, Xs, gm, gv).cpu().numpy()
    dyn = _dyn_np(gp)
    worst = 0.0
    for lo in range(0, T, 128):                                 # (the closed form holds [rows, n, D] at once)
        ref, scale = predict_vjp(dyn, Xs[lo:lo + 128], gm[lo:lo + 128], gv[lo:lo + 128])
        worst = max(worst, float(np.max(np.abs(out[lo:lo + 128] - ref) / scale)))
    print("predict VJP n=%d D=%d E=%d T=%d vs closed form: %.1e of sum |terms|" % (n, D, E, T, worst))
    assert worst <= 1e-12
    if T > 1:                                                   # bitwise independent of T and of the row
        k = max(1, T // 3)
        part = engine.gp_predict_vjp(gp, Xs[:k], gm[:k], gv[:k])
        assert torch.equal(part, torch.as_tensor(out[:k], device=part.device))
        perm = rng.permutation(T)
        pm = engine.gp_predict_vjp(gp, Xs[perm], gm[perm], gv[perm]).cpu().numpy()
        assert np.array_equal(pm, out[perm])


def _device_grad(gp, spec, terms, x0, eps, mu):
    plan = engine.ParticlePlan(gp, spec, terms, x0.shape[0], eps.shape[1], mult_mu=mu, grad=True)
    plan.set_inputs(x0, eps)
    g = plan.launch_grad()
    return plan, {k: v.cpu().numpy() for k, v in g.items()}


@pytest.mark.parametrize("name", ["metric_rbf", "linear_squash", "linear_nosquash", "fitc", "n1_d16_h0"])
def test_parity_with_autograd_oracle(name):
    gp, spec, pol, terms, m0, S0, H, P, mu = _case(name)
    x0, eps = _draw(m0, S0, P, H, seed=P + H + 1)
    _, g = _device_grad(gp, spec, terms, x0, eps, mu)
    v, ref = value_and_grad(_dyn_np(gp), _oracle_pol(spec, pol), terms, x0, eps, mu)
    scale = max(float(np.abs(r).max()) for r in ref.values())
    if scale == 0.0:                                            # H = 0: nothing depends on the policy
        assert all(not g[k].any() for k in ref)
        err = 0.0
    else:
        err = max(float(np.abs(g[k] - ref[k]).max()) for k in ref) / scale
    verr = abs(float(g["value"][0]) - v) / max(abs(v), 1e-300)
    print("particle gradient %s (P=%d, H=%d) vs autograd oracle: %.1e of the gradient's scale, value %.1e"
          % (name, P, H, err, verr))
    assert err <= (1e-6 if name == "fitc" else 1e-8) and verr <= 1e-9


@pytest.mark.parametrize("name", ["metric_rbf", "linear_squash"])
def test_forward_outputs_bitwise_equal_rollout(name):
    gp, spec, pol, terms, m0, S0, H, P, mu = _case(name)
    x0, eps = _draw(m0, S0, P, H, seed=3)
    plan, _ = _device_grad(gp, spec, terms, x0, eps, mu)
    ref = engine.particles_rollout(gp, spec, terms, x0, eps, mult_mu=mu)
    for a, b in zip(plan.outputs(), ref):
        assert torch.equal(a, b)


def test_directional_finite_difference_of_device_value():
    pb = make_rollout_problem(300, 10, 2, 50, 1, seed=5)
    gp = engine.gp_factorize(pb["X"], pb["Y"], pb["ell"], pb["sf2"], pb["sn2"])
    terms = [t for t in _case("metric_rbf")[3] if t["kind"] != _lib.REWARD_BOX]
    Xc, Yc, lc = pb["Xc"][0], pb["Yc"][0], pb["lc"][0]
    U, H, P, mu = Yc.shape[1], 10, 1000, 1.5
    x0, eps = _draw(pb["m0"], pb["S0"], P, H, seed=21)

    def run(Xc, Yc, lc):
        pgp = engine.gp_factorize(Xc, Yc, lc, np.ones(U), 1e-4 * np.ones(U), need_iK=False, mode=1)
        spec = dict(kind=_lib.POLICY_RBF, Ds=10, U=U, squash=True, max_action=pb["maxa"], gp=pgp)
        return _device_grad(gp, spec, terms, x0, eps, mu)[1]
    g = run(Xc, Yc, lc)
    rng = np.random.RandomState(22)
    v = {k: rng.randn(*g[k].shape) for k in ("X", "Y", "ell")}
    h = 1e-5
    vp = run(Xc + h * v["X"], Yc + h * v["Y"], lc + h * v["ell"])["value"][0]
    vm = run(Xc - h * v["X"], Yc - h * v["Y"], lc - h * v["ell"])["value"][0]
    fd = (vp - vm) / (2 * h)
    gv = sum(float((g[k] * v[k]).sum()) for k in v)
    print("directional derivative: central difference %.12e, g'v %.12e, rel %.1e" % (fd, gv, abs(fd - gv) / abs(gv)))
    assert abs(fd - gv) <= 1e-6 * abs(gv)


def test_expected_pathwise_gradient_is_the_moment_matching_gradient():
    """Linear unsquashed policy, one linear reward, H = 2: E[return] = w'm0 + w'E[x1] and moment matching gets E[x1]
    exactly, so the mean of the pathwise gradient over independent draws is pilco_rollout_backward's gradient."""
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
    P, d = 1 << 14, engine.device()
    pp = engine.ParticlePlan(gp, spec, terms, P, 2, grad=True)
    F = engine.dev(np.linalg.cholesky(S0))
    draws = {k: [] for k in mm}
    for s in range(16):
        gen = torch.Generator(device=d)
        gen.manual_seed(100 + s)
        pp.x0.copy_(engine.dev(m0)[None] + torch.randn((P, 4), dtype=engine.F64, device=d, generator=gen) @ F.T)
        pp.eps_buf.copy_(torch.randn((P, 2, 4), dtype=engine.F64, device=d, generator=gen))
        g = pp.launch_grad()
        for k in draws:
            draws[k].append(g[k].cpu().numpy().copy())
    worst = 0.0
    for k, ref in mm.items():
        a = np.stack(draws[k])
        z = np.abs(a.mean(0) - ref) / (a.std(0, ddof=1) / np.sqrt(a.shape[0]))
        worst = max(worst, float(z.max()))
    print("pathwise gradient (16 x 2^14 particles) vs moment matching: worst %.2f standard errors" % worst)
    assert worst <= 5.0


def test_run_to_run_and_graph_replay_are_bitwise_equal():
    gp, spec, pol, terms, m0, S0, H, P, mu = _case("metric_rbf")
    x0, eps = _draw(m0, S0, P, H, seed=25)
    plan = engine.ParticlePlan(gp, spec, terms, P, H, mult_mu=mu, grad=True)
    plan.set_inputs(x0, eps)
    first = {k: v.clone() for k, v in plan.launch_grad().items()}
    second = {k: v.clone() for k, v in plan.launch_grad().items()}
    assert all(torch.equal(first[k], second[k]) for k in first)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        plan.launch_grad()
    for v in plan.gbuf.values():
        v.zero_()
    graph.replay()
    torch.cuda.synchronize()
    assert all(torch.equal(first[k], plan.gbuf[k]) for k in first)


def test_class_api():
    from pilco.models import PILCO
    from pilco.controllers import RbfController
    from pilco_b200 import policy_opt
    np.random.seed(26)
    X, Y = _pilco_data(26)
    pilco = PILCO((X[:60], Y[:60]), controller=RbfController(3, 1, 10, max_action=1.2), horizon=6)
    m, S = X[0, :3], 0.05 * np.eye(3)
    a = pilco.sample_policy_gradient(m, S, 6, num_samples=300, seed=5)
    tr = pilco.sample_trajectories(m, S, 6, num_samples=300, seed=5)
    assert np.array_equal(a.returns, tr.returns)
    assert abs(a.value - tr.returns.mean()) <= 1e-14 * abs(tr.returns.mean())
    flat = pilco.controller.get_flat()
    assert a.grad.shape == flat.shape and np.all(np.isfinite(a.grad))
    b = pilco.sample_policy_gradient(m, S, 6, num_samples=300, seed=5)
    assert np.array_equal(a.grad, b.grad)
    reward, grad = pilco.policy_gradient()
    loss, ev = policy_opt.PolicyEvaluator(pilco, 1)(flat[None])
    scale = np.abs(ev[0]).max()
    print("policy_gradient vs policy_opt's evaluator: reward %.1e, grad %.1e of scale"
          % (abs(reward + loss[0]), np.abs(grad + ev[0]).max() / scale))
    assert abs(reward + loss[0]) <= 1e-12 * abs(loss[0]) and np.abs(grad + ev[0]).max() <= 1e-12 * scale
    cos = float(a.grad @ grad / (np.linalg.norm(a.grad) * np.linalg.norm(grad)))
    print("cosine between the particle and moment-matching gradients: %.3f" % cos)
    # appended data: both follow the MGPR's updated factorisation
    pilco.mgpr.set_data((X, Y))
    c = pilco.sample_policy_gradient(m, S, 6, num_samples=300, seed=5)
    assert pilco.mgpr.last_update == "append" and not np.array_equal(c.grad, a.grad)
    r2, g2 = pilco.policy_gradient()
    assert np.all(np.isfinite(g2)) and r2 != reward


def test_smgpr_and_safe_pilco():
    from pilco.models import PILCO
    from pilco.controllers import LinearController
    from safe_pilco_extension.safe_pilco import SafePILCO
    from safe_pilco_extension.rewards_safe import RiskOfCollision
    from pilco.rewards import LinearReward
    np.random.seed(27)
    X, Y = _pilco_data(27, n=300, Ds=4)
    sp = PILCO((X, Y), num_induced_points=40, controller=LinearController(4, 1), horizon=5)
    res = sp.sample_policy_gradient(X[0, :4], 0.05 * np.eye(4), 5, num_samples=100, seed=2)
    r, g = sp.policy_gradient()
    assert res.grad.shape == g.shape == (5,) and np.all(np.isfinite(res.grad)) and np.all(np.isfinite(g))
    pilco = SafePILCO((X, Y), controller=LinearController(4, 1), horizon=5, reward_add=LinearReward(4, np.ones(4)),
                      reward_mult=RiskOfCollision(4, [0.0, 0.1], [0.6, 0.9]), mu=-4.0)
    res = pilco.sample_policy_gradient(X[0, :4], 0.05 * np.eye(4), 5, num_samples=300, seed=3)
    tr = pilco.sample_trajectories(X[0, :4], 0.05 * np.eye(4), 5, num_samples=300, seed=3)
    assert np.array_equal(res.returns, tr.returns) and tr.risks.any()
    assert abs(res.value - tr.returns.mean()) <= 1e-14 * abs(tr.returns.mean())
    r, g = pilco.policy_gradient()
    assert np.all(np.isfinite(res.grad)) and np.all(np.isfinite(g))
