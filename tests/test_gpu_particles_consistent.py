"""The consistent particle sampler on the device (pilco_particles_rollout_consistent through engine.particles_rollout /
ParticlePlan and PILCO.sample_trajectories(consistent=True)): parity with the numpy oracle (tests/particle_oracle.py)
given the same x0 and eps, step 0 bitwise the marginal sampler's, a revisited input reproducing its value, bitwise
independence of a particle from P, its row and the chunking, CUDA-graph replay, and the class API."""
import numpy as np
import pytest
import torch

from pilco_b200 import engine, _lib
from particle_cases import _case, _controller_np, _draw, _dyn_np, _pilco_data, _revisit_problem
from particle_oracle import consistent_rollout
from util import scaled_err

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("name", ["metric_rbf", "linear_squash", "linear_nosquash", "fitc", "n1_d16_h0"])
def test_parity_with_consistent_oracle(name):
    gp, spec, pol, terms, m0, S0, H, P, mu = _case(name)
    x0, eps = _draw(m0, S0, P, H, seed=P + H + 1)
    out = [t.cpu().numpy() for t in engine.particles_rollout(gp, spec, terms, x0, eps, mult_mu=mu, consistent=True)]
    ref = consistent_rollout(_dyn_np(gp), pol, terms, x0, eps, mult_mu=mu)
    own = scaled_err(consistent_rollout(_dyn_np(gp), pol, terms, x0, eps, mult_mu=mu, swap=True)[0], ref[0]) if H else 0.0
    Ds, U = spec["Ds"], spec["U"]
    shapes = [(P, H + 1, Ds), (P, H, U), (P, H), (P, H), (P,)]
    errs = []
    for what, o, r, shp in zip(("traj", "act", "reward", "risk", "ret"), out, ref, shapes):
        assert o.shape == shp, what
        errs.append(scaled_err(o, r) if r.size and np.abs(r).max() > 0 else float(np.abs(o).max(initial=0.0)))
    print("consistent particles %s (P=%d, H=%d) vs oracle: traj %.1e act %.1e reward %.1e risk %.1e ret %.1e; "
          "the oracle against itself with its sums reordered: traj %.1e" % ((name, P, H) + tuple(errs) + (own,)))
    # sampling a smooth function at nearby inputs is ill-conditioned (DESIGN.md section 14): the bar is 1e-9 of scale or
    # ten times the sampler's own sensitivity to rounding, whichever is larger
    assert max(errs) <= max(1e-9, 10.0 * own)
    assert np.array_equal(out[0][:, 0], x0)


@pytest.mark.parametrize("name", ["metric_rbf", "linear_squash", "fitc"])
def test_first_step_is_bitwise_the_marginal_samplers(name):
    gp, spec, pol, terms, m0, S0, H, P, mu = _case(name)
    x0, eps = _draw(m0, S0, P, H, seed=3)
    cons = engine.particles_rollout(gp, spec, terms, x0, eps, mult_mu=mu, consistent=True)
    marg = engine.particles_rollout(gp, spec, terms, x0, eps, mult_mu=mu)
    for a, b in zip(cons[:3], marg[:3]):
        assert torch.equal(a[:, :2], b[:, :2])
    assert not torch.equal(cons[0][:, 2:], marg[0][:, 2:])


def test_revisited_input_gives_the_same_value():
    H = 20
    gp, spec, terms, x0, eps = _revisit_problem(H, 1 << 14, seed=21)
    cons = engine.particles_rollout(gp, spec, terms, x0, eps, consistent=True)[0].cpu().numpy()
    marg = engine.particles_rollout(gp, spec, terms, x0, eps)[0].cpu().numpy()
    step = cons[:, 1] - cons[:, 0]
    t = np.arange(H + 1)[None, :, None]
    scale = t * np.abs(step).max(1)[:, None, None]              # per particle: the largest component of its step
    worst = float((np.abs((cons - cons[:, :1]) - t * step[:, None])[:, 1:] / scale[:, 1:]).max())
    ratios = []
    for traj, want in ((cons, H * H), (marg, H)):
        v1, vH = np.var(traj[:, 1] - traj[:, 0], axis=0), np.var(traj[:, H] - traj[:, 0], axis=0)
        r = vH / v1
        se = r * np.sqrt(4.0 / traj.shape[0])                   # the two variance estimates' relative errors
        ratios.append((r, np.abs(r - want) / se))
    print("revisited input: x_t - x_0 = t (x_1 - x_0) within %.1e relative; Var ratio consistent %s (%s se), "
          "marginal %s (%s se)" % (worst, np.round(ratios[0][0], 2), np.round(ratios[0][1], 2),
                                   np.round(ratios[1][0], 2), np.round(ratios[1][1], 2)))
    assert worst <= 1e-6
    assert np.all(ratios[0][1] <= 5.0) and np.all(ratios[1][1] <= 5.0)


def test_particle_is_bitwise_independent_of_batch_row_and_chunking():
    gp, spec, pol, terms, m0, S0, H, _, mu = _case("metric_rbf")
    H = 6
    x0, eps = _draw(m0, S0, 1300, H, seed=22)
    full = engine.particles_rollout(gp, spec, terms, x0, eps, mult_mu=mu, consistent=True)
    part = engine.particles_rollout(gp, spec, terms, x0[:500], eps[:500], mult_mu=mu, consistent=True)
    for a, b in zip(full, part):
        assert torch.equal(a[:500], b)
    perm = np.random.RandomState(23).permutation(1300)
    pm = engine.particles_rollout(gp, spec, terms, x0[perm], eps[perm], mult_mu=mu, consistent=True)
    for a, b in zip(full, pm):
        assert torch.equal(a[perm], b)
    one = engine.consistent_workspace_bytes(gp, spec["Ds"], spec["U"], 1, H)
    budget = engine.consistent_workspace_bytes(gp, spec["Ds"], spec["U"], 333, H)
    assert one > 0 and budget > one
    chunked = engine.particles_rollout(gp, spec, terms, x0, eps, mult_mu=mu, consistent=True, max_ws_bytes=budget)
    for a, b in zip(full, chunked):
        assert torch.equal(a, b)
    with pytest.raises(ValueError, match="max_ws_bytes"):
        engine.particles_rollout(gp, spec, terms, x0, eps, consistent=True, max_ws_bytes=one - 8)


def test_graph_replay_is_bitwise_equal_to_eager():
    gp, spec, pol, terms, m0, S0, H, P, mu = _case("metric_rbf")
    x0, eps = _draw(m0, S0, P, H, seed=24)
    plan = engine.ParticlePlan(gp, spec, terms, P, H, mult_mu=mu, consistent=True)
    plan.set_inputs(x0, eps)
    plan.launch()
    eager = [t.clone() for t in plan.outputs()]
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        plan.launch()
    for t in plan.outputs():
        t.zero_()
    plan.ws.zero_()
    g.replay()
    torch.cuda.synchronize()
    for a, b in zip(eager, plan.outputs()):
        assert torch.equal(a, b)
    with pytest.raises(ValueError, match="gradient"):
        engine.ParticlePlan(gp, spec, terms, P, H, grad=True, consistent=True)


def test_sample_trajectories_consistent_class_api():
    from pilco.models import PILCO
    from pilco.controllers import RbfController
    np.random.seed(25)
    X, Y = _pilco_data(25)
    pilco = PILCO((X[:60], Y[:60]), controller=RbfController(3, 1, 10, max_action=1.2), horizon=6)
    m, S = X[0, :3], 0.05 * np.eye(3)
    a = pilco.sample_trajectories(m, S, 6, num_samples=200, seed=5, consistent=True)
    b = pilco.sample_trajectories(m, S, 6, num_samples=200, seed=5, consistent=True)
    c = pilco.sample_trajectories(m, S, 6, num_samples=200, seed=6, consistent=True)
    marg = pilco.sample_trajectories(m, S, 6, num_samples=200, seed=5)
    assert [x.shape for x in a] == [(200, 7, 3), (200, 6, 1), (200, 6), (200, 6), (200,)]
    assert all(np.array_equal(x, y) for x, y in zip(a, b))
    assert not np.array_equal(a.states, c.states)
    assert np.array_equal(a.states[:, :2], marg.states[:, :2]) and not np.array_equal(a.states, marg.states)
    assert not a.risks.any() and np.allclose(a.returns, a.rewards.sum(1), rtol=0, atol=1e-12)
    h0 = pilco.sample_trajectories(m, S, 0, num_samples=8, seed=1, consistent=True)
    assert h0.states.shape == (8, 1, 3) and h0.actions.shape == (8, 0, 1) and not h0.returns.any()
    # consistent=False is the step-wise sampler, bitwise
    d = pilco.sample_trajectories(m, S, 6, num_samples=200, seed=5, consistent=False)
    assert all(np.array_equal(x, y) for x, y in zip(d, marg))
    # appended data: the sampler follows the MGPR's updated factorisation
    gp0 = pilco.mgpr.device_gp()
    pilco.mgpr.set_data((X, Y))
    assert pilco.mgpr.device_gp() is not gp0 and pilco.mgpr.last_update == "append"
    f = pilco.sample_trajectories(m, S, 6, num_samples=200, seed=5, consistent=True)
    assert not np.array_equal(f.states, a.states) and np.array_equal(f.states[:, 0], a.states[:, 0])
    gp = pilco.mgpr.device_gp()
    g = torch.Generator(device=engine.device()); g.manual_seed(5)
    torch.randn((200, 3), dtype=engine.F64, device=engine.device(), generator=g)
    eps = torch.randn((200, 6, 3), dtype=engine.F64, device=engine.device(), generator=g).cpu().numpy()
    args = (_dyn_np(gp), _controller_np(pilco.controller), pilco.reward.terms(), f.states[:, 0], eps)
    ref, own = consistent_rollout(*args)[0], consistent_rollout(*args, swap=True)[0]
    assert scaled_err(f.states, ref) <= max(1e-9, 10.0 * scaled_err(own, ref))


def test_sample_trajectories_consistent_smgpr_and_safe_pilco():
    from pilco.models import PILCO
    from pilco.controllers import LinearController
    from safe_pilco_extension.safe_pilco import SafePILCO
    from safe_pilco_extension.rewards_safe import RiskOfCollision
    from pilco.rewards import LinearReward
    np.random.seed(26)
    X, Y = _pilco_data(26, n=300, Ds=4)
    sp = PILCO((X, Y), num_induced_points=40, controller=LinearController(4, 1), horizon=5)
    res = sp.sample_trajectories(X[0, :4], 0.05 * np.eye(4), 5, num_samples=100, seed=2, consistent=True)
    assert res.states.shape == (100, 6, 4) and np.all(np.isfinite(res.states))
    pilco = SafePILCO((X, Y), controller=LinearController(4, 1), horizon=5, reward_add=LinearReward(4, np.ones(4)),
                      reward_mult=RiskOfCollision(4, [0.0, 0.1], [0.6, 0.9]), mu=-4.0)
    res = pilco.sample_trajectories(X[0, :4], 0.05 * np.eye(4), 5, num_samples=300, seed=3, consistent=True)
    assert res.risks.any() and np.all((res.risks == 0.0) | (res.risks == 1.0))
    ref = res.rewards.sum(1) + (-4.0) * (1.0 - np.prod(1.0 - res.risks, axis=1))
    assert np.allclose(res.returns, ref, rtol=0, atol=1e-12)
