"""PILCO's exploration objective in the particle rollouts on the device (pilco_particles_explore_* through
engine.ParticlePlan / ConsistentGradPlan with ``exploration``, pilco_particles_reward_moments through
engine.particle_reward_moments, and the PILCO class's sample_reward_moments and exploration keywords; DESIGN.md
section 24): value, step_var and gradients against torch autograd on the oracle (tests/particle_grad_oracle.py)
with the same x0, eps and nu, central differences of the device value, the bitwise properties (NULL and b = 0 against
the calls without exploration, restarts, graph replay), the chunked forward's moments, and the sampled variance at
step 0 against the moment-matching prediction."""
import numpy as np
import pytest
import torch

from pilco_b200 import engine, _lib
from particle_cases import _angle_case, _dyn_np, _oracle_pol, _pilco, _safe_pilco
from particle_grad_oracle import consistent_value_and_grad, value_and_grad
from particle_oracle import sample_moments
from util import _rel

pytestmark = pytest.mark.gpu

SHAPES = {                                                      # E, dims, U, policy, FITC, joint terms, noise
    "linear": (4, [], 1, "linear", False, False, False),
    "rbf": (4, [], 1, "rbf", False, False, False),
    "cartpole": (4, [1], 1, "rbf", False, False, False),
    "double_pendulum_noisy": (6, [1, 2], 1, "linear", False, True, True),
    "joint_terms": (4, [], 2, "linear", False, True, False),
    "fitc": (4, [1], 1, "rbf", True, False, False),
}


def _draw(E, P, H, seed):
    rng = np.random.RandomState(seed)
    return 0.8 * rng.randn(P, E), rng.randn(P, H, E), rng.randn(P, H, E)


def _run(gp, spec, terms, x0, eps, nu, v, mu, dims, b, R=1, consistent=False):
    kw = dict(mult_mu=mu, R=R, angles=dims, measurement_noise=v, exploration=b)
    if consistent:
        plan = engine.ConsistentGradPlan(gp, spec, terms, x0.shape[0], eps.shape[1], **kw)
    else:
        plan = engine.ParticlePlan(gp, spec, terms, x0.shape[0], eps.shape[1], grad=True, **kw)
    plan.set_inputs(x0, eps, nu if v is not None else None)
    g = plan.launch_grad()
    return plan, {k: t.cpu().numpy() for k, t in g.items()}


@pytest.mark.parametrize("name", sorted(SHAPES))
@pytest.mark.parametrize("consistent", [False, True])
def test_value_step_var_and_gradient_match_autograd_oracle(name, consistent):
    E, dims, U, kind, fitc, joint, noisy = SHAPES[name]
    gp, spec, pols, terms = _angle_case(E, dims, U, kind, fitc, joint)
    P, H, mu, b = 200, 5, 1.5, 0.7
    x0, eps, nu = _draw(E, P, H, seed=P + H + 3)
    v = 0.01 + 0.02 * np.random.RandomState(4).rand(E) if noisy else None
    plan, g = _run(gp, spec, terms, x0, eps, nu, v, mu, dims, b, consistent=consistent)
    args = (_dyn_np(gp), _oracle_pol(spec, pols[0]), terms, x0, eps, mu)
    f = consistent_value_and_grad if consistent else value_and_grad
    out = f(*args, angle_dims=dims, nu=nu, v=v, b=b)
    val, ref, sv = out[0], out[1], out[-1]
    own = 0.0
    if consistent:
        own = _rel(consistent_value_and_grad(*args, swap=True, angle_dims=dims, nu=nu, v=v, b=b)[1], ref)
    err = _rel(g, ref)
    verr = abs(float(g["value"][0]) - val) / max(abs(val), 1e-300)
    serr = float(np.abs(plan.step_var[0, :H].cpu().numpy() - sv).max() / np.abs(sv).max())
    print("explore %s consistent=%s vs autograd oracle: grad %.1e, value %.1e, step_var %.1e (own %.1e)"
          % (name, consistent, err, verr, serr, own))
    bar = 1e-6 if fitc else 1e-9
    assert err <= max(bar, 10.0 * own) and verr <= max(1e-9, 10.0 * own) and serr <= max(1e-9, 10.0 * own)


@pytest.mark.parametrize("b", [0.5, -0.5])
def test_device_value_matches_central_differences(b):
    E, dims, U = 4, [1], 1
    gp, spec, _, terms = _angle_case(E, dims, U, "linear", joint=True)
    x0, eps, _ = _draw(E, 400, 6, seed=9)
    _, g = _run(gp, spec, terms, x0, eps, None, None, 1.5, dims, b)
    val = lambda W, bb: float(_run(gp, dict(spec, W=W, b=bb), terms, x0, eps, None, None, 1.5, dims, b)[1]["value"][0])
    rng = np.random.RandomState(3)
    dW, db = rng.randn(*spec["W"].shape), rng.randn(*spec["b"].shape)
    h = 1e-5
    fd = (val(spec["W"] + h * dW, spec["b"] + h * db) - val(spec["W"] - h * dW, spec["b"] - h * db)) / (2 * h)
    gd = float((g["W"] * dW).sum() + (g["b"] * db).sum())
    print("b=%g directional derivative: central difference %.12e, pathwise %.12e" % (b, fd, gd))
    assert abs(fd - gd) <= 1e-6 * abs(gd)


@pytest.mark.parametrize("name", ["linear", "cartpole", "double_pendulum_noisy", "joint_terms"])
@pytest.mark.parametrize("consistent", [False, True])
def test_zero_b_is_bitwise_the_call_without_exploration(name, consistent):
    """b = 0 with step_var: every output and gradient is bitwise the noisy / angle / plain call's"""
    E, dims, U, kind, fitc, joint, noisy = SHAPES[name]
    gp, spec, _, terms = _angle_case(E, dims, U, kind, fitc, joint)
    x0, eps, nu = _draw(E, 300, 5, seed=11)
    v = 0.02 * np.ones(E) if noisy else None
    outs = []
    for b in (None, 0.0):
        plan, g = _run(gp, spec, terms, x0, eps, nu, v, 0.5, dims, b, consistent=consistent)
        outs.append(([t.cpu().numpy() for t in plan.outputs()], g))
        if b is not None:
            assert float(plan.step_var[0].min()) > 0.0
    for a, c in zip(outs[0][0], outs[1][0]):
        assert np.array_equal(a, c)
    assert all(np.array_equal(outs[0][1][k], outs[1][1][k]) for k in outs[0][1])


def test_zero_spread_is_bitwise_b_zero():
    """S0 = 0 at H = 1: every particle has the same reward, sigma_0 = 0, so b = 0.5 changes nothing"""
    E = 4
    gp, spec, _, terms = _angle_case(E, [], 1, "linear", joint=True)
    x0 = np.tile(0.3 * np.ones(E), (100, 1))
    eps = np.random.RandomState(2).randn(100, 1, E)
    p0, g0 = _run(gp, spec, terms, x0, eps, None, None, 0.5, [], 0.0)
    p1, g1 = _run(gp, spec, terms, x0, eps, None, None, 0.5, [], 0.5)
    assert float(p1.step_var[0, 0]) <= 1e-12
    assert all(np.array_equal(g0[k], g1[k]) for k in g0)


@pytest.mark.parametrize("consistent", [False, True])
def test_restarts_are_independent_and_graph_replay_is_bitwise(consistent):
    E, U, R = 4, 1, 3
    gp, spec, _, terms = _angle_case(E, [], U, "linear", joint=True, R=R)
    x0, eps, _ = _draw(E, 150, 4, seed=5)
    plan, g = _run(gp, spec, terms, x0, eps, None, None, 0.5, [], 0.6, R=R, consistent=consistent)
    sv = plan.step_var.cpu().numpy()
    for r in range(R):
        one = dict(spec, W=spec["W"][r], b=spec["b"][r])
        p1, g1 = _run(gp, one, terms, x0, eps, None, None, 0.5, [], 0.6, consistent=consistent)
        assert np.array_equal(p1.step_var[0].cpu().numpy(), sv[r])
        assert all(np.array_equal(g1[k].reshape(-1), g[k][r].reshape(-1)) for k in g1)
    gr = torch.cuda.CUDAGraph()
    torch.cuda.synchronize()
    with torch.cuda.graph(gr):
        plan.launch_grad()
    plan.gbuf["value"].zero_(); plan.step_var.zero_()
    gr.replay()
    torch.cuda.synchronize()
    assert np.array_equal(plan.step_var.cpu().numpy(), sv)
    assert all(np.array_equal(plan.gbuf[k].cpu().numpy(), g[k]) for k in g)


def test_reward_moments_over_chunked_forward_match_gradient_call():
    """pilco_particles_reward_moments over a chunked consistent forward gives the unchunked gradient call's step_var"""
    E, dims, U = 4, [1], 1
    gp, spec, _, terms = _angle_case(E, dims, U, "linear", joint=True)
    P, H = 300, 5
    x0, eps, _ = _draw(E, P, H, seed=13)
    plan, _ = _run(gp, spec, terms, x0, eps, None, None, 0.5, dims, 0.0, consistent=True)
    ref = plan.step_var[0, :H].cpu().numpy()
    one = engine.consistent_workspace_bytes(gp, E + len(dims), U, 1, H, dims)
    out = engine.particles_rollout(gp, spec, terms, x0, eps, mult_mu=0.5, consistent=True, angles=dims,
                                   max_ws_bytes=int(one * 97))
    mean, var = engine.particle_reward_moments(terms, out[0], out[1], angles=dims)
    err = float(np.abs(var.cpu().numpy() - ref).max() / np.abs(ref).max())
    print("chunked moments vs gradient call's step_var: %.1e" % err)
    assert err <= 1e-13
    want = sample_moments(terms, out[0].cpu().numpy(), out[1].cpu().numpy(), dims)
    assert np.allclose(mean.cpu().numpy(), want[0], rtol=1e-12, atol=1e-14)
    assert np.allclose(var.cpu().numpy(), want[1], rtol=1e-11, atol=0.0)


def test_sample_reward_moments_against_predicted_variance():
    """step 0 at 2^20 particles: the sampled variance against predict_reward_moments' closed form (exact at step 0 for
    the linear controller's unsquashed-free state terms); mean equals the trajectories' mean reward"""
    pilco, _, _ = _pilco("linear", 3)
    m, S = pilco.m_init, 0.05 * np.eye(3)
    N = 1 << 20
    mean, var = pilco.sample_reward_moments(m, S, 3, num_samples=N, seed=5)
    pm, pv = pilco.predict_reward_moments(m, S, 3)
    traj = pilco.sample_trajectories(m, S, 3, num_samples=N, seed=5)
    assert np.allclose(mean, traj.rewards.mean(0), rtol=1e-12, atol=1e-15)
    x0 = traj.states[:, 0]
    terms, _ = pilco.reward_spec()
    q = np.zeros(N)
    from particle_oracle import point_value
    for t in terms:
        r = point_value(t, x0)
        q += t.get("coef", 1.0) ** 2 * (r - r.mean()) ** 2
    se = q.std() / np.sqrt(N)
    print("step-0 reward variance: sampled %.10e, predicted %.10e, SE %.1e" % (var[0], pv[0], se))
    assert abs(var[0] - pv[0]) <= 5.0 * se


def test_class_api():
    pilco, _, _ = _pilco("linear", 4)
    m, S = pilco.m_init, 0.05 * np.eye(3)
    a = pilco.sample_policy_gradient(m, S, 4, num_samples=200, seed=1)
    b = pilco.sample_policy_gradient(m, S, 4, num_samples=200, seed=1, exploration=0.0)
    assert a.value == b.value and np.array_equal(a.grad, b.grad) and np.array_equal(a.returns, b.returns)
    c = pilco.sample_policy_gradient(m, S, 4, num_samples=200, seed=1, exploration=0.5)
    assert c.value > a.value and np.array_equal(a.returns, c.returns)
    with pytest.raises(ValueError, match="pathwise"):
        pilco.sample_policy_gradient(m, S, 4, num_samples=200, seed=1, estimator="score", exploration=0.5)
    start = pilco.sample_policy_gradient(pilco.m_init, pilco.S_init, pilco.horizon, num_samples=64, seed=2,
                                         exploration=0.5).value
    best = pilco.optimize_policy_sampled(maxiter=10, restarts=8, num_samples=64, seed=2, exploration=0.5)
    again = pilco.sample_policy_gradient(pilco.m_init, pilco.S_init, pilco.horizon, num_samples=64, seed=2,
                                         exploration=0.5).value
    print("optimize_policy_sampled(exploration=0.5): start %.6f, best %.6f, re-evaluated %.6f" % (start, best, again))
    assert np.isfinite(best) and best >= start - 1e-9 and abs(again - best) <= 1e-9 * max(1.0, abs(best))
    safe = _safe_pilco()
    mean, var = safe.sample_reward_moments(safe.m_init, 0.05 * np.eye(4), 3, num_samples=500, seed=3)
    traj = safe.sample_trajectories(safe.m_init, 0.05 * np.eye(4), 3, num_samples=500, seed=3)
    add = [t for t in safe.reward_spec()[0] if t.get("channel", 0) == _lib.CHANNEL_ADD]
    want = sample_moments(add, traj.states, traj.actions)
    assert np.allclose(var, want[1], rtol=1e-11) and np.allclose(mean, traj.rewards.mean(0), rtol=1e-12)
    g = safe.sample_policy_gradient(safe.m_init, 0.05 * np.eye(4), 3, num_samples=500, seed=3, exploration=0.5)
    assert np.all(np.isfinite(g.grad))
