"""GPU tests of the time-varying linear policy (pilco_rollout_scheduled_*, DESIGN.md section 27) through
engine.RolloutPlan(schedule=True) and the class API: a constant schedule against the stationary call (bitwise forward,
per-step gradients summing to its gradient), the torch oracle (tests/action_reward_oracle.py) on the features the
cascade combines, both reverse sweeps, a central difference, restarts against single calls and graph replay, the
open-loop closed form, and TimeVaryingLinearController with PILCO.optimize_policy / plan / compute_action."""
import os
import sys

import numpy as np
import pytest
import torch

from pilco_b200 import engine, _lib, rewards, controllers
from pilco_b200.models.pilco import PILCO
import action_reward_oracle as aro
from particle_cases import BOX2
from particle_grad_oracle import T
from util import make_gp_problem, scaled_err

pytestmark = pytest.mark.gpu


def _case(Ds=3, U=2, H=6, R=2, dims=(), seed=5, n=50, fitc=False, mi=20):
    Dh = Ds + len(dims)
    X, Y, ell, sf2, sn2 = make_gp_problem(n, Dh + U, Ds, seed=seed)
    Y = 0.1 * Y
    rng = np.random.RandomState(seed + 1)
    Z = X[rng.choice(n, mi, replace=False)] if fitc else None
    gp = engine.fitc_factorize(X, Z, Y, ell, sf2, sn2) if fitc else engine.gp_factorize(X, Y, ell, sf2, sn2)
    B = rng.randn(Ds, Ds)
    return dict(X=X, Y=Y, ell=ell, sf2=sf2, sn2=sn2, Z=Z, gp=gp, Ds=Ds, Dh=Dh, U=U, H=H, R=R, dims=list(dims),
                maxa=0.7 + rng.rand(U), W=0.5 * rng.randn(R, H, U, Dh), b=0.3 * rng.randn(R, H, U), m0=X[0, :Ds],
                S0=0.03 * B @ B.T + 0.02 * np.eye(Ds), v=0.01 + 0.05 * rng.rand(Ds))


def _terms(which, Ds, Dh, U, seed=0):
    rng = np.random.RandomState(seed)
    t = 0.4 * rng.randn(Ds)
    state = rewards.CombinedRewards(Ds, [rewards.ExponentialReward(Ds, W=np.diag(0.5 + rng.rand(Ds)), t=t),
                                         rewards.LinearReward(Ds, rng.randn(Ds))], coefs=[1.0, 0.3]).terms()
    if which == "state":
        return state
    if which == "safe":
        return state + [dict(kind=_lib.REWARD_BOX, coef=1.0, channel=_lib.CHANNEL_MULT, W=BOX2, t=None)]
    combined = rewards.CombinedRewards(Ds, [rewards.ExponentialReward(Ds, t=t), rewards.action_cost(Dh, U)],
                                       coefs=[1.0, 0.2]).terms()
    return combined + [dict(kind=_lib.REWARD_LINEAR_SA, coef=0.3, W=rng.randn(Dh + U), t=None)]


def _spec(P, W, b):
    return dict(kind=_lib.POLICY_LINEAR, Ds=P["Dh"], U=P["U"], squash=True, max_action=P["maxa"], W=W, b=b)


def _plan(P, terms, W, b, schedule=True, grad=False, noise=False, x=None, mu=1.5, H=None, R=None):
    return engine.RolloutPlan(P["gp"], _spec(P, W, b), terms, P["m0"], P["S0"], P["H"] if H is None else H,
                              R=P["R"] if R is None else R, mult_mu=mu, grad=grad, angles=P["dims"] or None,
                              exploration=x, measurement_noise=P["v"] if noise else None, schedule=schedule)


def _outputs(plan):
    out = [plan.traj_m, plan.traj_S, plan.reward, plan.step_reward, plan.step_risk, plan.info]
    return [t.clone() for t in out + ([plan.step_var] if plan.step_var is not None else [])]


CONSTANT = [  # angles, noise, exploration, terms, taped
    ((), False, None, "state", True),
    ((), False, None, "safe", False),
    ((1,), True, 0.4, "joint", True),
    ((0,), False, None, "joint", False),
]


@pytest.mark.parametrize("dims,noise,x,which,taped", CONSTANT)
def test_constant_schedule_is_the_stationary_call(dims, noise, x, which, taped):
    P = _case(dims=dims)
    terms = _terms(which, P["Ds"], P["Dh"], P["U"])
    W0, b0 = P["W"][:, 0], P["b"][:, 0]
    H = P["H"]
    ref = _plan(P, terms, W0, b0, schedule=False, grad=taped, noise=noise, x=x)
    ref.forward()
    gref = {k: v.clone() for k, v in ref.backward().items()}
    Wc = np.repeat(W0[:, None], H, 1)
    bc = np.repeat(b0[:, None], H, 1)
    plan = _plan(P, terms, Wc, bc, grad=taped, noise=noise, x=x)
    plan.forward()
    g = plan.backward()
    torch.cuda.synchronize()
    for a, e in zip(_outputs(plan), _outputs(ref)):
        assert torch.equal(a, e)
    assert g["W"].shape == (P["R"], H, P["U"], P["Dh"]) and g["b"].shape == (P["R"], H, P["U"])
    for k in ("W", "b"):
        s, e = g[k].sum(1), gref[k]
        assert float((s - e).abs().max() / e.abs().max()) <= 1e-13, k
    for k in ("m0", "S0"):
        assert torch.equal(g[k], gref[k]), k


PARITY = [  # angles, noise, exploration b, terms, fitc, taped, centres
    ((), False, None, "state", False, True, 50),
    ((), False, None, "state", False, False, 50),
    ((1,), False, None, "joint", False, True, 50),
    ((), True, None, "state", False, True, 50),
    ((0,), True, 0.5, "joint", False, False, 50),
    ((), False, -0.3, "state", True, True, 80),
    ((), False, None, "safe", False, True, 50),
    ((), False, None, "safe", True, False, 80),
    ((), False, 0.2, "joint", False, False, 1100),
]


@pytest.mark.parametrize("shape", ["metric", "swimmer"])
@pytest.mark.parametrize("dims,noise,x,which,fitc,taped,n", PARITY)
def test_oracle_parity(shape, dims, noise, x, which, fitc, taped, n):
    Ds, U = (3, 2) if shape == "metric" else (6, 2)
    if shape == "swimmer" and (n > 100 or fitc):
        pytest.skip("the swimmer shape runs the exact GP at 50 centres")
    P = _case(Ds=Ds, U=U, H=5, dims=dims, n=n, fitc=fitc)
    terms = _terms(which, P["Ds"], P["Dh"], P["U"])
    mu = 1.5
    plan = _plan(P, terms, P["W"], P["b"], grad=taped, noise=noise, x=x, mu=mu)
    assert (plan.tape is not None) == taped or n > 1024
    plan.forward()
    g = plan.backward()
    torch.cuda.synchronize()
    assert int(plan.info.max()) == 0
    dyn = aro.dynamics(P["X"], P["Y"], P["ell"], P["sf2"], P["sn2"], P["Z"])
    for r in range(P["R"]):
        Wt, bt = T(P["W"][r]).requires_grad_(), T(P["b"][r]).requires_grad_()
        ref = aro.mm_rollout(dyn, aro.step_action(Wt, bt, P["maxa"]), terms, P["m0"], P["S0"], P["H"], mult_mu=mu,
                             angle_dims=P["dims"] or None, v=P["v"] if noise else None, b=x or 0.0)
        tol = 1e-9 if fitc else 1e-10
        assert scaled_err(plan.traj_m[r].cpu().numpy(), ref["traj_m"].detach().numpy()) <= tol
        assert scaled_err(plan.traj_S[r].cpu().numpy(), ref["traj_S"].detach().numpy()) <= tol
        assert abs(float(plan.reward[r]) - float(ref["reward"])) <= tol * max(1.0, abs(float(ref["reward"])))
        gW, gb = torch.autograd.grad(ref["reward"], (Wt, bt))
        gtol = 1e-6 if fitc else 1e-7
        assert scaled_err(g["W"][r].cpu().numpy(), gW.numpy()) <= gtol
        assert scaled_err(g["b"][r].cpu().numpy(), gb.numpy()) <= gtol


def test_central_difference_along_a_schedule_direction():
    P = _case(R=1, H=8)
    terms = _terms("joint", P["Ds"], P["Dh"], P["U"])
    rng = np.random.RandomState(3)
    vW, vb = rng.randn(*P["W"].shape), rng.randn(*P["b"].shape)
    plan = _plan(P, terms, P["W"], P["b"], grad=True)
    plan.forward()
    g = plan.backward()
    gv = float((g["W"].cpu().numpy() * vW).sum() + (g["b"].cpu().numpy() * vb).sum())
    h, f = 1e-5, []
    for s in (1, -1):
        p = _plan(P, terms, P["W"] + s * h * vW, P["b"] + s * h * vb)
        p.forward()
        f.append(float(p.reward[0]))
    fd = (f[0] - f[1]) / (2 * h)
    assert abs(fd - gv) <= 1e-6 * max(1.0, abs(gv)), (fd, gv)


@pytest.mark.parametrize("taped", [True, False])
def test_restarts_are_their_single_calls_and_replay_bitwise(taped):
    P = _case(R=3, dims=(1,))
    terms = _terms("joint", P["Ds"], P["Dh"], P["U"])
    plan = _plan(P, terms, P["W"], P["b"], grad=taped, noise=True)
    plan.forward()
    g = {k: v.clone() for k, v in plan.backward().items()}
    out = _outputs(plan)
    for r in range(3):
        one = _plan(P, terms, P["W"][r], P["b"][r], grad=taped, noise=True, R=1)
        one.forward()
        g1 = one.backward()
        torch.cuda.synchronize()
        for a, e in zip(_outputs(one)[:4], out[:4]):
            assert torch.equal(a[0], e[r])
        for k in ("W", "b", "m0", "S0"):
            assert torch.equal(g1[k][0], g[k][r]), k
    plan.forward()
    plan.backward()
    assert all(torch.equal(a, e) for a, e in zip(_outputs(plan), out))
    plan.capture(backward=True)
    plan.replay()
    torch.cuda.synchronize()
    assert all(torch.equal(a, e) for a, e in zip(_outputs(plan), out))
    assert all(torch.equal(plan.gbuf[k], g[k]) for k in g)


def test_open_loop_one_step_closed_form():
    """H = 1 from a known state under u_0 = maxa sin(b_0): the next mean is the GP's posterior mean at [x0, u0] and a
    joint linear term w'[x0, u0] has d/db_0 = w_u maxa cos(b_0)"""
    P = _case(R=1, H=1)
    Ds, U = P["Ds"], P["U"]
    w = np.random.RandomState(2).randn(Ds + U)
    terms = [dict(kind=_lib.REWARD_LINEAR_SA, coef=1.0, W=w, t=None)]
    b0 = P["b"][0]
    plan = engine.RolloutPlan(P["gp"], _spec(P, np.zeros((1, U, Ds)), b0), terms, P["m0"], np.zeros((Ds, Ds)), 1,
                              schedule=True)
    plan.forward()
    g = plan.backward()
    u = P["maxa"] * np.sin(b0[0])
    xu = np.r_[P["m0"], u]
    K = lambda A, B, e: P["sf2"][e] * np.exp(-0.5 * (((A[:, None] - B[None]) / P["ell"][e]) ** 2).sum(-1))
    mean = np.array([K(xu[None], P["X"], e)[0] @ np.linalg.solve(K(P["X"], P["X"], e) + P["sn2"][e] * np.eye(len(P["X"])),
                                                              P["Y"][:, e]) for e in range(Ds)])
    assert scaled_err(plan.traj_m[0, 1].cpu().numpy(), P["m0"] + mean) <= 1e-9
    assert abs(float(plan.reward[0]) - float(w @ xu)) <= 1e-12 * max(1.0, abs(float(w @ xu)))
    assert scaled_err(g["b"][0, 0].cpu().numpy(), w[Ds:] * P["maxa"] * np.cos(b0[0])) <= 1e-10
    assert bool(torch.isfinite(g["W"]).all())


# ---- class level -------------------------------------------------------------------------------------------------

def _pilco(feedback, H=8, seed=0):
    np.random.seed(seed)
    rng = np.random.RandomState(seed)
    X = np.hstack([rng.randn(60, 2) * 0.5, rng.uniform(-1, 1, (60, 1))])
    Y = np.stack([0.1 * X[:, 1], 0.1 * (-np.sin(X[:, 0]) + X[:, 2])], 1)
    c = controllers.TimeVaryingLinearController(2, 1, H, max_action=1.0, feedback=feedback)
    pilco = PILCO((X, Y), controller=c, horizon=H, reward=rewards.ExponentialReward(2, t=np.array([0.5, 0.0])),
                  m_init=np.zeros((1, 2)), S_init=0.01 * np.eye(2))
    for m in pilco.mgpr.models:
        m.likelihood.variance.assign(1e-3)
    return pilco


@pytest.mark.parametrize("feedback", [True, False])
def test_optimize_policy_raises_the_objective(feedback):
    pilco = _pilco(feedback)
    before = float(-pilco.training_loss().item())
    value, grad = pilco.policy_gradient()
    assert abs(value - before) <= 1e-12 * max(1.0, abs(before)) and grad.shape == pilco.controller.get_flat().shape
    best = pilco.optimize_policy(maxiter=15, restarts=3)
    after = float(-pilco.training_loss().item())
    assert after > before and abs(after - best) <= 1e-9 * max(1.0, abs(best))
    if not feedback:
        assert not np.any(np.asarray(pilco.controller.W))


def test_plan_acts_shifts_and_warm_starts():
    pilco = _pilco(False)
    c = pilco.controller
    m_init, S_init = np.array(pilco.m_init), np.array(pilco.S_init)
    seen = []
    shift = c.shift
    c.shift = lambda: (seen.append(c.get_flat().copy()), shift())
    x = np.array([0.1, -0.2])
    u = np.asarray(pilco.plan(x, maxiter=10, restarts=2))
    assert u.shape == (1, 1) and np.all(np.isfinite(u))
    b = seen[0].reshape(8, 1)
    assert np.allclose(u, np.sin(b[0]), rtol=0, atol=1e-12)          # u_0 = maxa sin(b_0) at a measured state
    assert np.array_equal(np.asarray(c.b), np.concatenate([b[1:], b[-1:]]))
    assert np.array_equal(pilco.m_init, m_init) and np.array_equal(pilco.S_init, S_init)
    r_start = pilco.policy_gradient(x[None], np.zeros((2, 2)))[0]
    pilco.plan(x, maxiter=10, restarts=1)                            # restart 0 is the shifted plan: never worse
    c.set_flat(seen[1])
    assert pilco.policy_gradient(x[None], np.zeros((2, 2)))[0] >= r_start - 1e-12
    rng = np.random.RandomState(1)
    with pytest.raises(TypeError):
        PILCO((rng.randn(10, 3), 0.1 * rng.randn(10, 2)), horizon=4).plan(x)


def test_compute_action_reads_step_t_and_particles_refuse():
    pilco = _pilco(True, H=4)
    c = pilco.controller
    x = np.array([[0.3, -0.1]])
    W, b = np.asarray(c.W), np.asarray(c.b)
    for t in range(4):
        u = np.asarray(pilco.compute_action(x, t=t))
        assert np.allclose(u, np.sin(W[t] @ x[0] + b[t]), rtol=0, atol=1e-12), t
    assert np.allclose(np.asarray(pilco.compute_action(x)), np.sin(W[0] @ x[0] + b[0]), rtol=0, atol=1e-12)
    with pytest.raises(ValueError):
        pilco.predict(pilco.m_init, pilco.S_init, 5)
    for call in (lambda: pilco.sample_trajectories(pilco.m_init, pilco.S_init, 3, num_samples=10),
                 lambda: pilco.sample_reward_moments(pilco.m_init, pilco.S_init, 3, num_samples=10),
                 lambda: pilco.sample_policy_gradient(pilco.m_init, pilco.S_init, 3, num_samples=10),
                 lambda: pilco.optimize_policy_sampled(maxiter=2, num_samples=10)):
        with pytest.raises(ValueError, match="TimeVaryingLinearController"):
            call()


def test_mpc_on_the_example_pendulum_beats_random_actions():
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "examples"))
    import pendulum_mpc_numpy
    random_returns, mpc_returns = pendulum_mpc_numpy.run(episodes=1, T=20, horizon=8, restarts=2, maxiter=8,
                                                         verbose=False)
    assert np.all(np.isfinite(mpc_returns))
    assert np.mean(mpc_returns) > np.mean(random_returns), (mpc_returns, random_returns)
