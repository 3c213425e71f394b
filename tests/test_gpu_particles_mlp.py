"""GPU tests of tanh MLP policies in the particle rollouts (pilco_particles_mlp_*, DESIGN.md section 29) through
engine.ParticlePlan / ConsistentGradPlan / particles_rollout and PILCO.optimize_policy_sampled with an MlpController:
the numpy and torch oracles on every sampler, a central difference, restarts against single calls, reruns and graph
replay, a particle's outputs against P and its row, exploration at b = 0, and policy optimisation on samples."""
import numpy as np
import pytest
import torch

from pilco_b200 import _lib, controllers, engine, rewards
from pilco_b200.models.pilco import PILCO
import particle_grad_oracle as pgo
import particle_mlp_oracle as pmo
import particle_oracle as po
from particle_cases import _angle_case, _dyn_np
from util import scaled_err

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _mlp_oracle():
    """the shared particle oracles serve MLP policy dicts (tests/particle_mlp_oracle.py)"""
    with pmo.mlp_policies():
        yield


def _theta(Ds, U, hidden, R=None, seed=0):
    """weights N(0, 1/fan_in) and biases N(0, 0.3^2) in the flat layout, [R?, n_theta]"""
    rng = np.random.RandomState(seed + 31)
    widths = [Ds] + list(hidden) + [U]
    one = lambda: np.concatenate([np.concatenate([rng.randn(widths[l + 1], widths[l]) / np.sqrt(widths[l]),
                                                  0.3 * rng.randn(widths[l + 1], 1)], 1).ravel()
                                  for l in range(len(widths) - 1)])
    return one() if R is None else np.stack([one() for _ in range(R)])


def _case(E, U, hidden, R=None, squash=True, joint=True, seed=0):
    """-> gp, spec, the oracle's policy dict (restart 0), terms (linear, exp, MULT box; joint EXP_SA and LINEAR_SA)"""
    gp, lin, _, terms = _angle_case(E, [], U, "linear", joint=joint, seed=seed)
    theta = _theta(E, U, hidden, R, seed)
    spec = dict(kind=_lib.POLICY_MLP, Ds=E, U=U, squash=squash, max_action=lin["max_action"], hidden=tuple(hidden),
                theta=theta)
    pol = dict(kind=_lib.POLICY_MLP, squash=squash, maxa=np.asarray(lin["max_action"]), Ds=E, U=U,
               hidden=tuple(hidden), theta=theta if R is None else theta[0])
    return gp, spec, pol, terms


def _draw(E, P, H, seed):
    rng = np.random.RandomState(seed)
    return 0.8 * rng.randn(P, E), rng.randn(P, H, E), rng.randn(P, H, E)


def _make(gp, spec, terms, P, H, mu, sampler="stepwise", R=1, x=None, grad=True):
    if sampler == "consistent" and grad:
        return engine.ConsistentGradPlan(gp, spec, terms, P, H, mult_mu=mu, R=R, exploration=x)
    return engine.ParticlePlan(gp, spec, terms, P, H, mult_mu=mu, grad=grad, R=R, consistent=sampler == "consistent",
                               exploration=x, resample=sampler == "resampled")


def _run(plan, x0, eps, xi, grad=True):
    plan.set_inputs(x0, eps, xi=xi if plan.resample else None)
    g = {k: t.clone() for k, t in plan.launch_grad().items()} if grad else {}
    if not grad:
        plan.launch()
    torch.cuda.synchronize()
    return [t.clone() for t in plan.outputs()], g


SHAPES = {"small": (4, 1), "swimmer": (8, 2)}                  # E, U
PARITY = [  # shape, sampler, hidden, squash
    ("small", "stepwise", (16,), True),
    ("small", "stepwise", (64, 64), False),
    ("small", "consistent", (24, 12), True),
    ("small", "resampled", (64, 64), True),
    ("swimmer", "stepwise", (64, 64), True),
    ("swimmer", "consistent", (32,), True),
    ("swimmer", "resampled", (20, 30), True),
]


@pytest.mark.parametrize("shape,sampler,hidden,squash", PARITY)
def test_oracle_parity(shape, sampler, hidden, squash):
    """the forward against the numpy oracle (the torch oracle's for the refit), value and d value / d theta against the
    torch oracle; every reward kind (linear, exp, MULT box, joint EXP_SA and LINEAR_SA; the refit: no joint terms)"""
    E, U = SHAPES[shape]
    gp, spec, pol, terms = _case(E, U, hidden, squash=squash, joint=sampler != "resampled")
    P, H, mu = 200, 5, 1.5
    x0, eps, xi = _draw(E, P, H, seed=P + H + len(hidden))
    out, g = _run(_make(gp, spec, terms, P, H, mu, sampler), x0, eps, xi)
    out = [t.cpu().numpy() for t in out]
    dyn = _dyn_np(gp)
    own = 0.0
    if sampler == "resampled":
        r = pgo.resampled_rollout(dyn, pol, terms, x0, eps, xi, mu)
        ref_out = [r[k] for k in ("traj", "act", "rew", "risk", "ret")]
        val, ref = r["value"], r["grad"]
    elif sampler == "consistent":
        ref_out = po.consistent_rollout(dyn, pol, terms, x0, eps, mu)
        own = scaled_err(po.consistent_rollout(dyn, pol, terms, x0, eps, mu, swap=True)[0], ref_out[0])
        val, ref = pgo.consistent_value_and_grad(dyn, pol, terms, x0, eps, mu)[:2]
    else:
        ref_out = po.particle_rollout(dyn, pol, terms, x0, eps, mu)
        val, ref = pgo.value_and_grad(dyn, pol, terms, x0, eps, mu)
    ref_out = [np.asarray(r) for r in ref_out]
    errs = [scaled_err(o, r) if r.size and np.abs(r).max() > 0 else float(np.abs(o).max(initial=0.0))
            for o, r in zip(out, ref_out)]
    gt = g["theta"].cpu().numpy().reshape(-1)
    err = scaled_err(gt, np.asarray(ref["theta"]).reshape(-1))
    verr = abs(float(g["value"][0]) - val) / max(abs(val), 1e-300)
    print("MLP %s %s hidden=%s squash=%s: forward %.1e, gradient %.1e of scale, value %.1e (oracle's own %.1e)"
          % (shape, sampler, hidden, squash, max(errs), err, verr, own))
    assert g["theta"].shape == (1, engine.mlp_theta_size(E, U, hidden)) or g["theta"].shape == (gt.size,)
    assert max(errs) <= max(1e-12, 10.0 * own)
    assert err <= max(1e-10, 10.0 * own) and verr <= max(1e-10, 10.0 * own)


def test_central_difference_along_a_theta_direction():
    E, U, hidden = 4, 1, (32, 16)
    gp, spec, _, terms = _case(E, U, hidden)
    P, H, mu = 500, 6, 1.5
    x0, eps, _ = _draw(E, P, H, seed=9)
    _, g = _run(_make(gp, spec, terms, P, H, mu), x0, eps, None)
    val = lambda th: float(engine.particles_rollout(gp, dict(spec, theta=th), terms, x0, eps, mult_mu=mu)[4].mean())
    d = np.random.RandomState(3).randn(spec["theta"].size)
    h = 1e-5
    fd = (val(spec["theta"] + h * d) - val(spec["theta"] - h * d)) / (2 * h)
    gd = float((g["theta"].cpu().numpy().reshape(-1) * d).sum())
    print("MLP directional derivative: central difference %.12e, pathwise %.12e" % (fd, gd))
    assert abs(fd - gd) <= 1e-6 * abs(gd)


@pytest.mark.parametrize("sampler", ["stepwise", "consistent", "resampled"])
def test_restarts_are_their_single_calls_and_replay_bitwise(sampler):
    E, U, R, hidden = 4, 1, 3, (64, 64)
    gp, spec, _, terms = _case(E, U, hidden, R=R, joint=sampler != "resampled")
    P, H, mu = 300, 5, 1.5
    x0, eps, xi = _draw(E, P, H, seed=21)
    plan = _make(gp, spec, terms, P, H, mu, sampler, R=R)
    out, g = _run(plan, x0, eps, xi)
    assert g["theta"].shape == (R, spec["theta"].shape[1]) and g["value"].shape == (R,)
    for r in range(R):
        o1, g1 = _run(_make(gp, dict(spec, theta=spec["theta"][r]), terms, P, H, mu, sampler), x0, eps, xi)
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


@pytest.mark.parametrize("sampler", ["stepwise", "consistent"])
def test_a_particle_does_not_depend_on_P_or_its_row(sampler):
    E, U, hidden = 4, 2, (64, 64)
    gp, spec, _, terms = _case(E, U, hidden)
    P, H = 260, 5
    x0, eps, _ = _draw(E, P, H, seed=5)
    full = engine.particles_rollout(gp, spec, terms, x0, eps, mult_mu=1.5, consistent=sampler == "consistent")
    rows = np.random.RandomState(2).permutation(P)[:37]
    part = engine.particles_rollout(gp, spec, terms, x0[rows], eps[rows], mult_mu=1.5,
                                    consistent=sampler == "consistent")
    idx = torch.as_tensor(rows, device=full[0].device)
    assert all(torch.equal(a[idx], b) for a, b in zip(full, part))


@pytest.mark.parametrize("sampler", ["stepwise", "consistent"])
def test_exploration_at_b0_is_the_call_without_it(sampler):
    E, U, R, hidden = 4, 1, 2, (16, 8)
    gp, spec, _, terms = _case(E, U, hidden, R=R)
    terms = [t for t in terms if t["kind"] != _lib.REWARD_BOX]
    P, H, mu = 150, 4, 0.0
    x0, eps, _ = _draw(E, P, H, seed=8)
    out0, g0 = _run(_make(gp, spec, terms, P, H, mu, sampler, R=R), x0, eps, None)
    out1, g1 = _run(_make(gp, spec, terms, P, H, mu, sampler, R=R, x=0.0), x0, eps, None)
    assert all(torch.equal(a, b) for a, b in zip(out0, out1))
    assert all(torch.equal(g0[k], g1[k]) for k in g0)
    _, g2 = _run(_make(gp, spec, terms, P, H, mu, sampler, R=R, x=0.5), x0, eps, None)
    assert not torch.equal(g2["theta"], g0["theta"])                # b != 0 reaches the MLP's gradient


def _pilco(seed=0):
    np.random.seed(seed)
    rng = np.random.RandomState(seed)
    X = np.hstack([rng.randn(60, 2) * 0.5, rng.uniform(-1, 1, (60, 1))])
    Y = np.stack([0.1 * X[:, 1], 0.1 * (-np.sin(X[:, 0]) + X[:, 2])], 1)
    c = controllers.MlpController(2, 1, hidden=(16, 16), max_action=1.0)
    pilco = PILCO((X, Y), controller=c, horizon=6, reward=rewards.ExponentialReward(2, t=np.array([0.5, 0.0])),
                  m_init=np.zeros((1, 2)), S_init=0.01 * np.eye(2))
    for m in pilco.mgpr.models:
        m.likelihood.variance.assign(1e-3)
    return pilco


@pytest.mark.parametrize("sampler", ["stepwise", "consistent", "resampled"])
def test_optimize_policy_sampled_raises_the_sampled_return(sampler):
    pilco = _pilco()
    kw = dict(consistent=sampler == "consistent", resample=sampler == "resampled")
    v0 = pilco.sample_policy_gradient(pilco.m_init, pilco.S_init, pilco.horizon, num_samples=64, seed=11, **kw).value
    best = pilco.optimize_policy_sampled(maxiter=15, restarts=4, num_samples=64, seed=11, **kw)
    v1 = pilco.sample_policy_gradient(pilco.m_init, pilco.S_init, pilco.horizon, num_samples=64, seed=11, **kw).value
    print("MLP optimize_policy_sampled %s: in-sample value %.6f -> %.6f (re-evaluated %.6f)" % (sampler, v0, best, v1))
    assert best > v0 and abs(v1 - best) <= 1e-9 * max(1.0, abs(best))
    u = np.asarray(pilco.compute_action(np.array([[0.1, -0.2]])))
    assert u.shape == (1, 1) and np.all(np.isfinite(u)) and abs(float(u[0, 0])) <= 1.0
