"""GPU tests of function samples from random-feature draws (pilco_particles_features_*, DESIGN.md section 30) through
engine.feature_draws, particles_rollout and ConsistentGradPlan: the draw and the rollouts against the oracles given
the normals (linear, RBF and MLP policies; angles, noise and exploration), a central difference, restarts against
single calls, forward outputs of the gradient call, independence of P and of a particle's row, reruns and graph
replay, the sampler's statistics (near and far from the data, a revisited input, the exact consistent sampler), and
the PILCO class methods' num_features."""
import numpy as np
import pytest
import torch

from pilco_b200 import _lib, controllers, engine, rewards
from pilco_b200.models.pilco import PILCO
import particle_features_oracle as pfo
import particle_mlp_oracle as pmo
from particle_cases import _angle_case, _dyn_np, _oracle_pol, _pilco, _revisit_problem
from util import scaled_err

pytestmark = pytest.mark.gpu


def _normals(gp, P, F, seed):
    rng = np.random.RandomState(seed)
    return rng.randn(gp.E, F, gp.D), rng.randn(P, gp.E, 2 * F), rng.randn(P, gp.E, gp.n)


def _draws(gp, P, F, seed=0):
    zeta, w, eps_y = _normals(gp, P, F, seed)
    return engine.feature_draws(gp, P, F, zeta, w, eps_y), (zeta, w, eps_y)


def _np(draws):
    return draws.omega.cpu().numpy(), draws.w.cpu().numpy(), draws.v.cpu().numpy()


SHAPES = {"small": (3, 1, 150), "metric": (10, 2, 300), "swimmer": (8, 2, 150)}      # E, U, n


@pytest.mark.parametrize("shape", ["small", "metric"])
def test_draw_matches_the_oracle_and_does_not_depend_on_P(shape):
    E, U, n = SHAPES[shape]
    gp, _, _, _ = _angle_case(E, [], U, n=n)
    P, F = 300, 64
    draws, (zeta, w, eps_y) = _draws(gp, P, F)
    omega, v = pfo.draw(_dyn_np(gp), gp.sn2.cpu().numpy(), zeta, w, eps_y)
    assert np.array_equal(draws.omega.cpu().numpy(), omega)
    assert scaled_err(draws.v.cpu().numpy(), v) <= 1e-10
    part = engine.feature_draws(gp, 7, F, zeta, w[5:12], eps_y[5:12])
    assert torch.equal(part.v, draws.v[5:12])


def _inputs(gp, P, H, seed, Dx=None):
    rng = np.random.RandomState(seed + 100)
    return 0.5 * rng.randn(P, Dx or gp.E), rng.randn(P, H, gp.E)


PARITY = [  # shape, policy kind, angles, noise
    ("small", "linear", [], False),
    ("small", "rbf", [], False),
    ("small", "linear", [0], True),
    ("small", "rbf", [1], False),
    ("swimmer", "linear", [], False),
    ("swimmer", "rbf", [2, 3], True),
]


@pytest.mark.parametrize("shape,kind,angles,noisy", PARITY)
def test_forward_and_gradient_against_the_oracles(shape, kind, angles, noisy):
    E, U, n = SHAPES[shape]
    gp, spec, pols, terms = _angle_case(E, angles, U, kind, joint=True, n=n)
    P, H, F = 64, 6, 48
    draws, _ = _draws(gp, P, F, seed=1)
    om, w, v = _np(draws)
    x0, nu = _inputs(gp, P, H, 2)
    var = 0.01 * np.ones(E) if noisy else None
    nz = dict(measurement_noise=var, nu=nu if noisy else None)
    dyn = _dyn_np(gp)
    out = engine.particles_rollout(gp, spec, terms, x0, None, mult_mu=1.5, consistent=True, angles=angles or None,
                                   features=draws, horizon=H, **nz)
    ref = pfo.rollout(dyn, om, w, v, pols[0], terms, x0, H, 1.5, angles or None, nu if noisy else None, var)
    # a fixed bar of 1e-10 of scale (the issue's floor; no reordered-oracle bar is computed): the kernels and the
    # oracle sum in different orders; the largest difference is printed
    errs = [scaled_err(o.cpu().numpy(), r) for o, r in zip(out, ref)]
    print("forward parity, largest scaled difference %.3g" % max(errs))
    assert max(errs) <= 1e-10, errs
    plan = engine.ConsistentGradPlan(gp, spec, terms, P, H, mult_mu=1.5, angles=angles or None, num_features=F,
                                     measurement_noise=var)
    plan.set_inputs(x0, None, nu=nu if noisy else None, features=draws)
    g = {k: t.clone() for k, t in plan.launch_grad().items()}
    for o, c in zip(out, plan.outputs()):
        assert torch.equal(o, c)                                         # the grad call's forward is the forward
    val, gref, _ = pfo.value_and_grad(dyn, om, w, v, _oracle_pol(spec, pols[0]), terms, x0, H, 1.5, angles or None,
                                      nu if noisy else None, var)
    assert abs(float(g["value"][0]) - val) <= 1e-10 * max(1.0, abs(val))
    for k, ref_g in gref.items():
        assert scaled_err(g[k].cpu().numpy().reshape(np.shape(ref_g)), ref_g) <= 1e-8, k


@pytest.mark.parametrize("kind", ["linear", "rbf"])
def test_exploration_bonus_against_the_oracle(kind):
    """b != 0: value = mean return + b sum_t sigma_t, its gradient (the bonus's share goes through pf_vjp_kernel's
    x~_bar) and sigma_t^2 against the torch oracle"""
    E, U, n = SHAPES["small"]
    gp, spec, pols, terms = _angle_case(E, [], U, kind, joint=True, n=n)
    P, H, F, b = 48, 5, 32, 0.7
    draws, _ = _draws(gp, P, F, seed=15)
    om, w, v = _np(draws)
    x0, _ = _inputs(gp, P, H, 16)
    plan = engine.ConsistentGradPlan(gp, spec, terms, P, H, num_features=F, exploration=b)
    plan.set_inputs(x0, None, features=draws)
    g = plan.launch_grad()
    val, gref, hist = pfo.value_and_grad(_dyn_np(gp), om, w, v, _oracle_pol(spec, pols[0]), terms, x0, H, b=b)
    assert abs(float(g["value"][0]) - val) <= 1e-10 * max(1.0, abs(val))
    assert scaled_err(plan.step_var[0, :H].cpu().numpy(), hist["step_var"]) <= 1e-10
    for k, ref_g in gref.items():
        assert scaled_err(g[k].cpu().numpy().reshape(np.shape(ref_g)), ref_g) <= 1e-8, k


def test_central_difference_restarts_and_exploration():
    E, U, n = SHAPES["small"]
    R, P, H, F = 3, 50, 5, 32
    gp, spec, pols, terms = _angle_case(E, [], U, "linear", n=n, R=R)
    draws, _ = _draws(gp, P, F, seed=3)
    x0, _ = _inputs(gp, P, H, 4)
    plan = engine.ConsistentGradPlan(gp, spec, terms, P, H, R=R, num_features=F, exploration=0.0)
    plan.set_inputs(x0, None, features=draws)
    g = {k: t.clone() for k, t in plan.launch_grad().items()}
    outs = [t.clone() for t in plan.outputs()]
    for r in range(R):                                                   # restart r is the single call with policy r
        one = dict(spec, W=spec["W"][r], b=spec["b"][r])
        p1 = engine.ConsistentGradPlan(gp, one, terms, P, H, num_features=F, exploration=0.0)
        p1.set_inputs(x0, None, features=draws)
        g1 = p1.launch_grad()
        for k in g1:
            assert torch.equal(g1[k].reshape(-1), g[k][r].reshape(-1)), k
        for o, c in zip(outs, p1.outputs()):
            assert torch.equal(o[r], c)
    one = dict(spec, W=spec["W"][0], b=spec["b"][0])
    dW = np.random.RandomState(5).randn(*one["W"].shape)
    ret = lambda Wx: float(engine.particles_rollout(gp, dict(one, W=Wx), terms, x0, None, consistent=True,
                                                    features=draws, horizon=H)[4].mean())
    h = 1e-6
    fd = (ret(one["W"] + h * dW) - ret(one["W"] - h * dW)) / (2 * h)
    gd = float((g["W"][0].cpu().numpy() * dW).sum())
    assert abs(fd - gd) <= 1e-6 * max(abs(gd), 1e-3), (fd, gd)


@pytest.mark.parametrize("hidden", [(16,), (24, 12)])
def test_mlp_policy_against_the_oracles(hidden):
    E, U, n = SHAPES["small"]
    gp, lin, _, terms = _angle_case(E, [], U, "linear", joint=True, n=n)
    rng = np.random.RandomState(9)
    theta = 0.5 * rng.randn(engine.mlp_theta_size(E, U, hidden))
    spec = dict(kind=_lib.POLICY_MLP, Ds=E, U=U, squash=True, max_action=lin["max_action"], hidden=hidden, theta=theta)
    pol = dict(kind=_lib.POLICY_MLP, squash=True, maxa=np.asarray(lin["max_action"]), Ds=E, U=U, hidden=hidden,
               theta=theta)
    P, H, F = 40, 5, 32
    draws, _ = _draws(gp, P, F, seed=6)
    om, w, v = _np(draws)
    x0, _ = _inputs(gp, P, H, 7)
    dyn = _dyn_np(gp)
    with pmo.mlp_policies():
        out = engine.particles_rollout(gp, spec, terms, x0, None, consistent=True, features=draws, horizon=H)
        ref = pfo.rollout(dyn, om, w, v, pol, terms, x0, H)
        for o, r in zip(out, ref):
            assert scaled_err(o.cpu().numpy(), r) <= 1e-10
        plan = engine.ConsistentGradPlan(gp, spec, terms, P, H, num_features=F)
        plan.set_inputs(x0, None, features=draws)
        g = plan.launch_grad()
        val, gref, _ = pfo.value_and_grad(dyn, om, w, v, pol, terms, x0, H)
    assert abs(float(g["value"][0]) - val) <= 1e-10 * max(1.0, abs(val))
    assert scaled_err(g["theta"].cpu().numpy().reshape(-1), np.asarray(gref["theta"]).reshape(-1)) <= 1e-8


def test_particles_do_not_depend_on_P_or_their_row_and_graphs_replay():
    E, U, n = SHAPES["small"]
    gp, spec, pols, terms = _angle_case(E, [], U, "rbf", n=n)
    P, H, F = 90, 7, 40
    zeta, w, eps_y = _normals(gp, P, F, 8)
    draws = engine.feature_draws(gp, P, F, zeta, w, eps_y)
    x0, _ = _inputs(gp, P, H, 9)
    full = engine.particles_rollout(gp, spec, terms, x0, None, consistent=True, features=draws, horizon=H)
    again = engine.particles_rollout(gp, spec, terms, x0, None, consistent=True, features=draws, horizon=H)
    for a, b in zip(full, again):
        assert torch.equal(a, b)
    idx = np.array([17, 3, 64])                                          # a subset, reordered
    sub = engine.feature_draws(gp, 3, F, zeta, w[idx], eps_y[idx])
    part = engine.particles_rollout(gp, spec, terms, x0[idx], None, consistent=True, features=sub, horizon=H)
    for a, b in zip(part, full):
        assert torch.equal(a, b[idx])
    chunked = engine.particles_rollout(gp, spec, terms, x0, None, consistent=True, features=draws, horizon=H,
                                       max_ws_bytes=engine.consistent_workspace_bytes(gp, E, U, 25, H,
                                                                                      num_features=F))
    for a, b in zip(chunked, full):
        assert torch.equal(a, b)
    plan = engine.ConsistentGradPlan(gp, spec, terms, P, H, num_features=F)
    plan.set_inputs(x0, None, features=draws)
    ref = {k: t.clone() for k, t in plan.launch_grad().items()}
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        plan.launch_grad()
    for k in plan.gbuf:
        plan.gbuf[k].zero_()
    graph.replay()
    torch.cuda.synchronize()
    for k in ref:
        assert torch.equal(ref[k], plan.gbuf[k]), k


def _constant_policy(E, U, b):
    return dict(kind=_lib.POLICY_LINEAR, Ds=E, U=U, squash=False, max_action=np.ones(U), W=np.zeros((U, E)),
                b=np.full(U, b))


@pytest.mark.parametrize("where", ["near", "far"])
def test_one_step_variance_is_the_conditional_closed_form(where):
    """2^16 particles at one x~: Var(x_1 - x_0) against |phi - k iK Phi(X)|^2 + sn2 |iK k|^2 given omega (near the
    data) or sf2 (far from it), 5 standard errors of the sample variance"""
    E, U, n = SHAPES["small"]
    gp, _, _, terms = _angle_case(E, [], U, n=n)
    P, F = 1 << 16, 256
    draws, _ = _draws(gp, P, F, seed=10)
    X = gp.X.cpu().numpy()
    xt = X[5] if where == "near" else X[5] + 30.0
    x0 = np.tile(xt[:E], (P, 1))
    spec = _constant_policy(E, U, float(xt[E]))
    out = engine.particles_rollout(gp, spec, terms, x0, None, consistent=True, features=draws, horizon=1)
    dx = (out[0][:, 1] - out[0][:, 0]).cpu().numpy()
    sv = dx.var(0, ddof=1)
    dyn = _dyn_np(gp)
    var = pfo.conditional_variance(dyn, gp.sn2.cpu().numpy(), draws.omega.cpu().numpy(), xt[None])[0]
    if where == "far":
        assert np.abs(var - dyn["sf2"]).max() <= 1e-12 * dyn["sf2"].max()
    assert np.all(np.abs(sv - var) <= 5 * var * np.sqrt(2.0 / (P - 1))), (sv, var)


def test_revisited_input_grows_as_H_squared():
    """section 14's construction: every step of a particle has the same input, so x_H - x_0 = H f and the variance
    ratio is H^2"""
    H, P = 20, 4096
    gp, spec, terms, x0, _ = _revisit_problem(H, P, 11)
    draws, _ = _draws(gp, P, 128, seed=12)
    traj = engine.particles_rollout(gp, spec, terms, x0, None, consistent=True, features=draws,
                                    horizon=H)[0].cpu().numpy()
    v1, vH = (traj[:, 1] - traj[:, 0]).var(0), (traj[:, H] - traj[:, 0]).var(0)
    assert np.all(np.abs(vH / v1 / H ** 2 - 1.0) <= 1e-6), vH / v1


def test_moments_match_the_exact_consistent_sampler():
    """F = 4096, 2^14 particles, H = 5: per-step sample means and variances within 5 standard errors of the exact
    consistent sampler's (independent normals for the two)"""
    E, U, n = SHAPES["small"]
    gp, spec, _, terms = _angle_case(E, [], U, "linear", n=60)
    P, H, F = 1 << 14, 5, 4096
    draws, _ = _draws(gp, P, F, seed=13)
    x0, eps = _inputs(gp, P, H, 14)
    x0 = 0.1 * x0
    a = engine.particles_rollout(gp, spec, terms, x0, None, consistent=True, features=draws, horizon=H)[0].cpu().numpy()
    b = engine.particles_rollout(gp, spec, terms, x0, eps, consistent=True)[0].cpu().numpy()
    for t in range(1, H + 1):
        ma, mb, va, vb = a[:, t].mean(0), b[:, t].mean(0), a[:, t].var(0, ddof=1), b[:, t].var(0, ddof=1)
        se_m = np.sqrt((va + vb) / P)
        se_v = np.sqrt(2.0 / (P - 1)) * np.sqrt(va ** 2 + vb ** 2)
        assert np.all(np.abs(ma - mb) <= 5 * se_m), (t, ma, mb)
        assert np.all(np.abs(va - vb) <= 5 * se_v), (t, va, vb)


# ---- the class API ---------------------------------------------------------------------------------------------------
def _mlp_pilco():
    rng = np.random.RandomState(4)
    X = np.hstack([rng.randn(60, 2) * 0.5, rng.uniform(-1, 1, (60, 1))])
    Y = np.stack([0.1 * X[:, 1], 0.1 * (-np.sin(X[:, 0]) + X[:, 2])], 1)
    c = controllers.MlpController(2, 1, hidden=(16, 16), max_action=1.0)
    pilco = PILCO((X, Y), controller=c, horizon=6, reward=rewards.ExponentialReward(2, t=np.array([0.5, 0.0])),
                  m_init=np.zeros((1, 2)), S_init=0.01 * np.eye(2))
    for m in pilco.mgpr.models:
        m.likelihood.variance.assign(1e-3)
    return pilco


@pytest.mark.parametrize("kind", ["linear", "rbf", "mlp"])
def test_optimize_policy_sampled_raises_the_sampled_return(kind):
    pilco = _mlp_pilco() if kind == "mlp" else _pilco(kind, 2)[0]
    kw = dict(consistent=True, num_features=128)
    spg = lambda: pilco.sample_policy_gradient(pilco.m_init, pilco.S_init, pilco.horizon, num_samples=64, seed=11, **kw)
    v0 = spg().value
    best = pilco.optimize_policy_sampled(maxiter=15, restarts=3, num_samples=64, seed=11, **kw)
    v1 = spg().value
    print("%s optimize_policy_sampled(num_features=128): in-sample value %.6f -> %.6f (re-evaluated %.6f)"
          % (kind, v0, best, v1))
    assert best > v0 and abs(v1 - best) <= 1e-9 * max(1.0, abs(best))


def test_class_methods_draw_in_the_documented_order():
    """the same seed gives the same x0 with and without num_features; num_features=None is today's call bit for bit;
    the trajectories, moments and gradient of one seed agree with each other and with the engine on the same draws"""
    pilco = _pilco("linear", 3)[0]
    m, S, n, N, seed = pilco.m_init, pilco.S_init, 5, 200, 21
    exact = pilco.sample_trajectories(m, S, n, num_samples=N, seed=seed, consistent=True)
    none = pilco.sample_trajectories(m, S, n, num_samples=N, seed=seed, consistent=True, num_features=None)
    feat = pilco.sample_trajectories(m, S, n, num_samples=N, seed=seed, consistent=True, num_features=64)
    for a, b in zip(exact, none):
        assert np.array_equal(a, b)
    assert np.array_equal(feat.states[:, 0], exact.states[:, 0])
    x0, draws = pilco._feature_inputs(m, S, n, N, seed, 64, "test")
    terms, mu = pilco.reward_spec()
    ref = engine.particles_rollout(pilco.mgpr.device_gp(), pilco.policy_spec(), terms, x0, None, mult_mu=mu,
                                   consistent=True, features=draws, horizon=n)
    for a, b in zip(feat, ref):
        assert np.array_equal(a, b.cpu().numpy())
    mean, _ = pilco.sample_reward_moments(m, S, n, num_samples=N, seed=seed, consistent=True, num_features=64)
    assert np.abs(mean - feat.rewards.mean(0)).max() <= 1e-12 * max(1.0, np.abs(mean).max())
    g = pilco.sample_policy_gradient(m, S, n, num_samples=N, seed=seed, consistent=True, num_features=64)
    assert np.array_equal(g.returns, feat.returns) and np.all(np.isfinite(g.grad))
