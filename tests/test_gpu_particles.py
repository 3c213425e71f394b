"""Particle rollout on the device (pilco_particles_rollout through engine.particles_rollout / ParticlePlan and
PILCO.sample_trajectories): parity with the numpy particle oracle given the same x0 and eps (tests/particle_oracle.py),
actions against compute_action, the exact one-step moments of moment matching, bitwise independence of a particle
from its batch, CUDA-graph replay, and the class API."""
import numpy as np
import pytest
import torch

from pilco_b200 import engine, _lib
from particle_cases import _case, _controller_np, _draw, _dyn_np, _linear, _pilco_data
from particle_oracle import moment_check, particle_rollout
from util import make_rollout_problem, scaled_err

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("name", ["metric_rbf", "linear_squash", "linear_nosquash", "fitc", "n1_d16_h0"])
def test_parity_with_particle_oracle(name):
    gp, spec, pol, terms, m0, S0, H, P, mu = _case(name)
    x0, eps = _draw(m0, S0, P, H, seed=P + H)
    out = [t.cpu().numpy() for t in engine.particles_rollout(gp, spec, terms, x0, eps, mult_mu=mu)]
    ref = particle_rollout(_dyn_np(gp), pol, terms, x0, eps, mult_mu=mu)
    Ds, U = spec["Ds"], spec["U"]
    shapes = [(P, H + 1, Ds), (P, H, U), (P, H), (P, H), (P,)]
    errs = []
    for what, o, r, shp in zip(("traj", "act", "reward", "risk", "ret"), out, ref, shapes):
        assert o.shape == shp, what
        errs.append(scaled_err(o, r) if r.size and np.abs(r).max() > 0 else float(np.abs(o).max(initial=0.0)))
    print("particles %s (P=%d, H=%d) vs oracle: traj %.1e act %.1e reward %.1e risk %.1e ret %.1e" % ((name, P, H) + tuple(errs)))
    assert max(errs) <= 1e-9
    assert np.array_equal(out[0][:, 0], x0)
    if not any(t.get("channel", 0) == _lib.CHANNEL_MULT for t in terms):
        assert not out[3].any()


@pytest.mark.parametrize("kind", ["rbf", "linear"])
def test_actions_equal_compute_action(kind):
    from pilco.models import PILCO
    from pilco.controllers import RbfController, LinearController
    np.random.seed(12)
    Ds, U = 3, 2
    X0 = np.random.rand(60, Ds + U)
    Y0 = 0.1 * np.sin(X0).dot(np.random.rand(Ds + U, Ds))
    ctrl = LinearController(Ds, U, max_action=np.array([1.5, 0.5])) if kind == "linear" \
        else RbfController(Ds, U, 9, max_action=0.8)
    pilco = PILCO((X0, Y0), controller=ctrl, horizon=5)
    res = pilco.sample_trajectories(X0[0, :Ds], 0.1 * np.eye(Ds), 5, num_samples=16, seed=3)
    worst = 0.0
    for p in range(0, 16, 3):
        for t in range(5):
            u = np.asarray(pilco.compute_action(res.states[p, t]))[0]
            worst = max(worst, float(np.max(np.abs(res.actions[p, t] - u))))
    print("%s policy: sampled actions vs compute_action: %.1e" % (kind, worst))
    assert worst <= 1e-12


def test_one_step_moments_are_exact():
    """Linear policy, no squash, H = 1: the joint input is Gaussian, so the moment-matching rollout's traj_m[1],
    traj_S[1] and step reward are the exact moments the particles sample."""
    pb = make_rollout_problem(300, 10, 2, 50, 1, seed=13)
    gp = engine.gp_factorize(pb["X"], pb["Y"], pb["ell"], pb["sf2"], pb["sn2"])
    rng = np.random.RandomState(14)
    spec, _ = _linear(0.5 * rng.randn(2, 10), rng.randn(2), np.ones(2), False)
    terms = [dict(kind=_lib.REWARD_EXP, coef=1.0, W=np.eye(10), t=pb["m0"] + 0.3)]
    m0, S0 = pb["m0"], 0.1 * np.eye(10)
    plan = engine.RolloutPlan(gp, spec, terms, m0, S0, 1, R=1)
    tm, tS, _ = plan.forward()
    M1, S1, r0 = tm[0, 1].cpu().numpy(), tS[0, 1].cpu().numpy(), float(plan.step_reward[0, 0])
    P = 1 << 18
    g = torch.Generator(device=engine.device())
    g.manual_seed(15)
    x0 = engine.dev(m0)[None] + torch.randn((P, 10), dtype=engine.F64, device=engine.device(), generator=g) @ \
        engine.dev(np.linalg.cholesky(S0)).T
    eps = torch.randn((P, 1, 10), dtype=engine.F64, device=engine.device(), generator=g)
    traj, _, rew, _, _ = engine.particles_rollout(gp, spec, terms, x0, eps)
    worst = moment_check(traj[:, 1].cpu().numpy(), M1, S1)
    r = rew[:, 0].cpu().numpy()
    z = (r.mean() - r0) / (r.std() / np.sqrt(P))
    print("one-step moments at P=2^18: worst %.2f standard errors (mean, covariance), reward %.2f" % (worst, z))
    assert worst <= 5.0 and abs(z) <= 5.0


def test_particle_is_bitwise_independent_of_its_batch():
    gp, spec, pol, terms, m0, S0, H, _, mu = _case("metric_rbf")
    H = 4
    x0, eps = _draw(m0, S0, 1300, H, seed=16)
    full = engine.particles_rollout(gp, spec, terms, x0, eps, mult_mu=mu)
    part = engine.particles_rollout(gp, spec, terms, x0[:500], eps[:500], mult_mu=mu)
    for a, b in zip(full, part):
        assert torch.equal(a[:500], b)
    perm = np.random.RandomState(17).permutation(1300)
    pm = engine.particles_rollout(gp, spec, terms, x0[perm], eps[perm], mult_mu=mu)
    for a, b in zip(full, pm):
        assert torch.equal(a[perm], b)


def test_graph_replay_is_bitwise_equal_to_eager():
    gp, spec, pol, terms, m0, S0, H, P, mu = _case("metric_rbf")
    x0, eps = _draw(m0, S0, P, H, seed=18)
    plan = engine.ParticlePlan(gp, spec, terms, P, H, mult_mu=mu)
    plan.set_inputs(x0, eps)
    plan.launch()
    eager = [t.clone() for t in plan.outputs()]
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        plan.launch()
    for t in plan.outputs():
        t.zero_()
    g.replay()
    torch.cuda.synchronize()
    for a, b in zip(eager, plan.outputs()):
        assert torch.equal(a, b)



def test_sample_trajectories_class_api():
    from pilco.models import PILCO
    from pilco.controllers import RbfController
    np.random.seed(19)
    X, Y = _pilco_data(19)
    pilco = PILCO((X[:60], Y[:60]), controller=RbfController(3, 1, 10, max_action=1.2), horizon=6)
    m, S = X[0, :3], 0.05 * np.eye(3)
    a = pilco.sample_trajectories(m, S, 6, num_samples=200, seed=5)
    b = pilco.sample_trajectories(m, S, 6, num_samples=200, seed=5)
    c = pilco.sample_trajectories(m, S, 6, num_samples=200, seed=6)
    assert [x.shape for x in a] == [(200, 7, 3), (200, 6, 1), (200, 6), (200, 6), (200,)]
    assert all(np.array_equal(x, y) for x, y in zip(a, b))
    assert not np.array_equal(a.states, c.states)
    assert not a.risks.any() and np.allclose(a.returns, a.rewards.sum(1), rtol=0, atol=1e-12)
    np.random.seed(7); d = pilco.sample_trajectories(m, S, 6, num_samples=50)
    np.random.seed(7); e = pilco.sample_trajectories(m, S, 6, num_samples=50)
    assert np.array_equal(d.states, e.states)
    k = pilco.sample_trajectories(m, np.zeros((3, 3)), 2, num_samples=8, seed=1)   # known start state
    assert np.array_equal(k.states[:, 0], np.broadcast_to(m, (8, 3)))
    h0 = pilco.sample_trajectories(m, S, 0, num_samples=8, seed=1)
    assert h0.states.shape == (8, 1, 3) and h0.actions.shape == (8, 0, 1) and not h0.returns.any()
    with pytest.raises(ValueError):
        pilco.sample_trajectories(m, -np.eye(3), 2, num_samples=8, seed=1)
    # appended data: the rollout follows the MGPR's updated factorisation
    gp0 = pilco.mgpr.device_gp()
    pilco.mgpr.set_data((X, Y))
    assert pilco.mgpr.device_gp() is not gp0 and pilco.mgpr.last_update == "append"
    f = pilco.sample_trajectories(m, S, 6, num_samples=200, seed=5)
    assert not np.array_equal(f.states, a.states) and np.array_equal(f.states[:, 0], a.states[:, 0])
    gp = pilco.mgpr.device_gp()
    g = torch.Generator(device=engine.device()); g.manual_seed(5)
    torch.randn((200, 3), dtype=engine.F64, device=engine.device(), generator=g)
    eps = torch.randn((200, 6, 3), dtype=engine.F64, device=engine.device(), generator=g).cpu().numpy()
    ref =particle_rollout(_dyn_np(gp), _controller_np(pilco.controller), pilco.reward.terms(), f.states[:, 0], eps)
    assert scaled_err(f.states, ref[0]) <= 1e-9



def test_sample_trajectories_smgpr_and_safe_pilco():
    from pilco.models import PILCO
    from pilco.controllers import LinearController
    from safe_pilco_extension.safe_pilco import SafePILCO
    from safe_pilco_extension.rewards_safe import RiskOfCollision
    from pilco.rewards import LinearReward
    np.random.seed(20)
    X, Y = _pilco_data(20, n=300, Ds=4)
    sp = PILCO((X, Y), num_induced_points=40, controller=LinearController(4, 1), horizon=5)
    res = sp.sample_trajectories(X[0, :4], 0.05 * np.eye(4), 5, num_samples=100, seed=2)
    assert res.states.shape == (100, 6, 4) and np.all(np.isfinite(res.states))
    pilco = SafePILCO((X, Y), controller=LinearController(4, 1), horizon=5, reward_add=LinearReward(4, np.ones(4)),
                      reward_mult=RiskOfCollision(4, [0.0, 0.1], [0.6, 0.9]), mu=-4.0)
    res = pilco.sample_trajectories(X[0, :4], 0.05 * np.eye(4), 5, num_samples=300, seed=3)
    assert res.risks.any() and np.all((res.risks == 0.0) | (res.risks == 1.0))
    ref = res.rewards.sum(1) + (-4.0) * (1.0 - np.prod(1.0 - res.risks, axis=1))
    assert np.allclose(res.returns, ref, rtol=0, atol=1e-12)
