"""GPU tests of the exploration objective (pilco_rollout_explore_*, DESIGN.md section 21) through engine.RolloutPlan and
the class API: step_var and the objective against the torch oracle (tests/action_reward_oracle.py), the reverse sweep
against autograd (taped and recomputing, with and without angles) and central differences, the bitwise identities
(no exploration, b = 0, batch position, graph replay, sigma_0 = 0) and PILCO(exploration=...)."""
import ctypes

import numpy as np
import pytest
import torch

from pilco_b200 import engine, _lib, rewards
import action_reward_oracle as aro
from particle_cases import BOX2
from particle_grad_oracle import T
from util import make_gp_problem, make_rollout_problem, scaled_err

pytestmark = pytest.mark.gpu


def _case(kind, R, Ds=3, U=2, dims=(), seed=9, n=50, bf=12):
    Dh = Ds + len(dims)
    X, Y, ell, sf2, sn2 = make_gp_problem(n, Dh + U, Ds, seed=seed)
    Y = 0.1 * Y
    rng = np.random.RandomState(seed + 1)
    maxa = 0.7 + rng.rand(U)
    if kind == "linear":
        prm = (0.5 * rng.randn(R, U, Dh), 0.3 * rng.randn(R, U))
        spec = dict(kind=_lib.POLICY_LINEAR, Ds=Dh, U=U, squash=True, max_action=maxa, W=prm[0], b=prm[1])
    else:
        prm = (rng.randn(R, bf, Dh) * 0.5 + 0.5, 0.1 * rng.randn(R, bf, U), 1.0 + 0.1 * rng.randn(R, U, Dh))
        pgp = engine.gp_factorize(*prm, np.ones((R, U)), 1e-4 * np.ones((R, U)), need_iK=False, mode=1)
        spec = dict(kind=_lib.POLICY_RBF, Ds=Dh, U=U, squash=True, max_action=maxa, gp=pgp)
    B = rng.randn(Ds, Ds)
    P = dict(X=X, Y=Y, ell=ell, sf2=sf2, sn2=sn2, maxa=maxa, m0=X[0, :Ds], S0=0.03 * B @ B.T + 0.02 * np.eye(Ds),
             dims=list(dims), kind=kind, Ds=Ds, Dh=Dh, U=U)
    return P, spec, prm


def _terms(which, Ds, Dh, U, seed=0):
    """"state": exponential + linear state terms; "joint": a CombinedRewards with an action cost, plus joint terms and
    MULT terms; "safe": the state terms with a MULT box risk (SafePILCO)"""
    rng = np.random.RandomState(seed)
    t = 0.4 * rng.randn(Ds)
    state = rewards.CombinedRewards(Ds, [rewards.ExponentialReward(Ds, W=np.diag(0.5 + rng.rand(Ds)), t=t),
                                         rewards.LinearReward(Ds, rng.randn(Ds))], coefs=[1.0, 0.3]).terms()
    if which == "state":
        return state
    if which == "safe":
        return state + [dict(kind=_lib.REWARD_BOX, coef=1.0, channel=_lib.CHANNEL_MULT, W=BOX2, t=None)]
    D = Dh + U
    Bj = rng.randn(D, D)
    combined = rewards.CombinedRewards(Ds, [rewards.ExponentialReward(Ds, t=t), rewards.action_cost(Dh, U)],
                                       coefs=[1.0, 0.2]).terms()
    return combined + [dict(kind=_lib.REWARD_EXP_SA, coef=-0.5, W=0.2 * Bj @ Bj.T, t=0.2 * rng.randn(D)),
                       dict(kind=_lib.REWARD_LINEAR_SA, coef=0.3, W=rng.randn(D), t=None),
                       dict(kind=_lib.REWARD_EXP, coef=0.1, channel=_lib.CHANNEL_MULT, W=np.eye(Ds), t=np.zeros(Ds)),
                       dict(kind=_lib.REWARD_LINEAR_SA, coef=0.01, channel=_lib.CHANNEL_MULT, W=rng.randn(D), t=None)]


def _plan(P, spec, terms, H, R, b, mu=1.5, grad=False, m0=None, S0=None):
    gp = engine.gp_factorize(P["X"], P["Y"], P["ell"], P["sf2"], P["sn2"])
    return engine.RolloutPlan(gp, spec, terms, P["m0"] if m0 is None else m0, P["S0"] if S0 is None else S0, H, R=R,
                              mult_mu=mu, grad=grad, angles=P["dims"] or None, exploration=b)


def _oracle(P, prm_r, terms, H, b, mu=1.5, m0=None, S0=None):
    return aro.problem_rollout(P["kind"], prm_r, P["X"], P["Y"], P["ell"], P["sf2"], P["sn2"], P["maxa"], terms,
                               T(P["m0"]) if m0 is None else m0, T(P["S0"]) if S0 is None else S0, H, mult_mu=mu,
                               angle_dims=P["dims"] or None, b=b)


def _check_forward(plan, ref, r, H, tol=1e-10):
    out = dict(step_var=plan.step_var[r, :H], reward=plan.reward[r], step_reward=plan.step_reward[r, :H],
               traj_m=plan.traj_m[r], traj_S=plan.traj_S[r])
    for k, v in out.items():
        o, e = v.cpu().numpy(), ref[k].detach().numpy()
        if e.size:
            assert scaled_err(o, e) <= tol, (k, r, scaled_err(o, e))


FORWARD = [  # policy, R, state dim, U, angles, terms, b
    ("linear", 2, 3, 2, (), "state", 0.5),
    ("rbf", 2, 3, 2, (), "joint", -0.5),
    ("linear", 3, 4, 1, (1,), "joint", 0.5),            # cart-pole-like
    ("rbf", 2, 4, 1, (1,), "state", 0.8),
    ("linear", 2, 3, 2, (), "safe", 0.5),               # SafePILCO: the MULT box term is not in sigma
]


@pytest.mark.parametrize("kind,R,Ds,U,dims,which,b", FORWARD)
def test_forward_matches_oracle(kind, R, Ds, U, dims, which, b):
    H = 6
    P, spec, prm = _case(kind, R, Ds, U, dims)
    terms = _terms(which, Ds, P["Dh"], U)
    plan = _plan(P, spec, terms, H, R, b)
    plan.forward()
    torch.cuda.synchronize()
    assert int(plan.info.max().item()) == 0
    for r in range(R):
        ref = _oracle(P, [T(p[r]) for p in prm], terms, H, b)
        assert float(ref["step_var"].min()) > 1e-8
        _check_forward(plan, ref, r, H)
    if which == "safe":                                 # the same step_var without the risk term, to the bit
        bare = _plan(P, spec, [t for t in terms if t.get("channel", 0) == _lib.CHANNEL_ADD], H, R, b)
        bare.forward()
        assert torch.equal(bare.step_var, plan.step_var)


def test_metric_shape_matches_oracle():
    """N = 300, E = 10, D = 12, RBF policies with 50 centres, R = 32 restarts (the restarts checked: first, middle, last)"""
    H, R, b = 10, 32, 0.5
    pb = make_rollout_problem(300, 10, 2, 50, R, seed=0)
    pgp = engine.gp_factorize(pb["Xc"], pb["Yc"], pb["lc"], np.ones((R, 2)), 1e-4 * np.ones((R, 2)), need_iK=False, mode=1)
    spec = dict(kind=_lib.POLICY_RBF, Ds=10, U=2, squash=True, max_action=pb["maxa"], gp=pgp)
    terms = [dict(kind=_lib.REWARD_EXP, coef=1.0, W=0.5 * np.eye(10), t=pb["m0"])]     # sigma_t^2 ~ 1e-2
    P = dict(pb, dims=[], kind="rbf")
    plan = _plan(P, spec, terms, H, R, b, mu=0.0)
    plan.forward()
    torch.cuda.synchronize()
    for r in (0, 17, R - 1):
        ref = _oracle(P, [T(pb[k][r]) for k in ("Xc", "Yc", "lc")], terms, H, b, mu=0.0)
        _check_forward(plan, ref, r, H)


GRADS = [  # policy, state dim, U, angles, terms, b
    ("linear", 3, 2, (), "joint", 0.5),
    ("rbf", 3, 2, (), "safe", -0.5),
    ("linear", 4, 1, (1,), "state", -0.5),
    ("rbf", 4, 1, (1,), "joint", 0.5),
]


@pytest.mark.parametrize("kind,Ds,U,dims,which,b", GRADS)
def test_gradient_matches_autograd(kind, Ds, U, dims, which, b):
    """policy, gm0 and gS0 gradients of both sweeps against autograd of the oracle (1e-8 of the gradient's scale)"""
    H, R = 5, 2
    P, spec, prm = _case(kind, R, Ds, U, dims, seed=4)
    terms = _terms(which, Ds, P["Dh"], U, seed=1)
    names = ["W", "b"] if kind == "linear" else ["X", "Y", "ell"]
    for taped in (True, False):
        plan = _plan(P, spec, terms, H, R, b, grad=taped)
        assert (plan.tape is not None) == taped
        plan.forward()
        g = {k: v.clone().cpu().numpy() for k, v in plan.backward().items()}
        torch.cuda.synchronize()
        for r in range(R):
            ps = [T(p[r]).requires_grad_() for p in prm]
            m0, S0 = T(P["m0"]).requires_grad_(), T(P["S0"]).requires_grad_()
            ref = _oracle(P, ps, terms, H, b, m0=m0, S0=S0)
            gref = torch.autograd.grad(ref["reward"], ps + [m0, S0])
            for k, gr in zip(names + ["m0", "S0"], gref):
                gr, o = gr.numpy(), g[k][r]
                if k == "S0":
                    gr, o = 0.5 * (gr + gr.T), 0.5 * (o + o.T)
                assert scaled_err(o, gr) <= 1e-8, (taped, k, r, scaled_err(o, gr))


@pytest.mark.parametrize("b", [0.5, -0.5])
def test_gradient_matches_central_differences(b):
    """d reward along a random direction of the linear policy's (W, b): restarts 1 and 2 carry theta +- h v"""
    H, Ds, U, h = 6, 3, 2, 1e-5
    P, spec, prm = _case("linear", 1, Ds, U, seed=13)
    terms = _terms("joint", Ds, Ds, U, seed=2)
    rng = np.random.RandomState(3)
    vW, vb = rng.randn(U, Ds), rng.randn(U)
    W = np.stack([prm[0][0], prm[0][0] + h * vW, prm[0][0] - h * vW])
    bb = np.stack([prm[1][0], prm[1][0] + h * vb, prm[1][0] - h * vb])
    plan = _plan(P, dict(spec, W=W, b=bb), terms, H, 3, b, grad=True)
    plan.forward()
    g = plan.backward()
    torch.cuda.synchronize()
    rew = plan.reward.cpu().numpy()
    fd = (rew[1] - rew[2]) / (2 * h)
    ad = float((g["W"][0].cpu().numpy() * vW).sum() + (g["b"][0].cpu().numpy() * vb).sum())
    assert abs(fd - ad) < 1e-6 * max(1.0, abs(ad)), (fd, ad)


def _outputs(plan, grads):
    out = dict(reward=plan.reward, traj_m=plan.traj_m, traj_S=plan.traj_S, step_reward=plan.step_reward,
               step_risk=plan.step_risk)
    out.update({"g" + k: v for k, v in grads.items()})
    return {k: v.clone() for k, v in out.items()}


@pytest.mark.parametrize("dims,taped", [((), True), ((), False), ((1,), True)])
def test_no_bonus_is_bitwise_the_call_without_exploration(dims, taped):
    """ex == NULL and b = 0 with step_var set: every output and gradient is the call without exploration's"""
    Ds, U, H, R = 4 if dims else 3, 1 if dims else 2, 5, 2
    P, spec, prm = _case("rbf", R, Ds, U, dims, seed=21)
    terms = _terms("joint", Ds, P["Dh"], U, seed=3)
    base = _plan(P, spec, terms, H, R, None, grad=taped)
    base.forward()
    ref = _outputs(base, base.backward())
    # ex == NULL through the exploration entry points, on the same description
    ang = ctypes.byref(base.ang) if base.ang is not None else None
    _lib.check(_lib.lib.pilco_rollout_explore_forward(ctypes.byref(base.ro), ang, None, engine.stream_ptr()), "fwd")
    _lib.check(_lib.lib.pilco_rollout_explore_backward(ctypes.byref(base.ro), ang, None, ctypes.byref(base.grad),
                                                       engine.stream_ptr()), "bwd")
    null = _outputs(base, base.gbuf)
    zero = _plan(P, spec, terms, H, R, 0.0, grad=taped)
    zero.forward()
    got = _outputs(zero, zero.backward())
    torch.cuda.synchronize()
    for k in ref:
        assert torch.equal(ref[k], null[k]) and torch.equal(ref[k], got[k]), k
    assert float(zero.step_var.min()) > 0.0


def test_restart_does_not_follow_batch_size_or_position():
    H, Ds, U, b = 5, 3, 2, 0.5
    P, spec, prm = _case("linear", 5, Ds, U, seed=31)
    terms = _terms("joint", Ds, Ds, U, seed=4)
    big = _plan(P, spec, terms, H, 5, b, grad=True)
    big.forward()
    gbig = {k: v.clone() for k, v in big.backward().items()}
    one = _plan(P, dict(spec, W=prm[0][3:4], b=prm[1][3:4]), terms, H, 1, b, grad=True)
    one.forward()
    gone = one.backward()
    torch.cuda.synchronize()
    assert torch.equal(big.reward[3:4], one.reward) and torch.equal(big.step_var[3:4], one.step_var)
    for k in gone:
        assert torch.equal(gbig[k][3:4], gone[k]), k


def test_graph_replay_matches_eager():
    H, Ds, U, R, b = 5, 4, 1, 2, -0.5
    P, spec, prm = _case("rbf", R, Ds, U, (1,), seed=41)
    terms = _terms("joint", Ds, P["Dh"], U, seed=5)
    plan = _plan(P, spec, terms, H, R, b, grad=True)
    plan.forward()
    eager = _outputs(plan, plan.backward())
    eager["step_var"] = plan.step_var.clone()
    plan.capture(backward=True)
    for t in [plan.reward, plan.step_var] + list(plan.gbuf.values()):
        t.zero_()
    plan.replay()
    torch.cuda.synchronize()
    again = _outputs(plan, plan.gbuf)
    again["step_var"] = plan.step_var.clone()
    for k in eager:
        assert torch.equal(eager[k], again[k]), k


def test_zero_initial_covariance_one_step():
    """S0 = 0, H = 1: sigma_0 = 0, so the reward and its gradient are those at b = 0"""
    Ds, U = 3, 2
    P, spec, prm = _case("linear", 1, Ds, U, seed=51)
    terms = _terms("state", Ds, Ds, U, seed=6)
    out = {}
    for b in (0.0, 0.5):
        plan = _plan(P, spec, terms, 1, 1, b, grad=True, S0=np.zeros((Ds, Ds)))
        plan.forward()
        out[b] = _outputs(plan, plan.backward())
        out[b]["step_var"] = plan.step_var.clone()
    torch.cuda.synchronize()
    assert float(out[0.5]["step_var"].abs().max()) <= aro.VAR_FLOOR
    for k in out[0.0]:
        assert torch.equal(out[0.0][k], out[0.5][k]), k


# ---- class API ---------------------------------------------------------------------------------------------------------
def _pilco(b, joint=True):
    from pilco.models import PILCO
    from pilco.controllers import RbfController
    np.random.seed(0)
    Ds, U = 3, 1
    X0 = np.random.rand(80, Ds + U) * 2.0 - 1.0
    Y0 = 0.1 * np.sin(X0).dot(np.random.rand(Ds + U, Ds))
    parts = [rewards.ExponentialReward(Ds, t=np.array([0.8, 0.8, 0.8])), rewards.LinearReward(Ds, [0.1, -0.2, 0.05])]
    if joint:
        parts.append(rewards.action_cost(Ds, U, [[1.0]]))
    reward = rewards.CombinedRewards(Ds, parts, coefs=[1.0, 0.5, 0.1][:len(parts)])
    ctrl = RbfController(Ds, U, 10, max_action=2.0)
    return PILCO((X0, Y0), controller=ctrl, horizon=10, reward=reward, m_init=np.zeros((1, Ds)),
                 S_init=0.05 * np.eye(Ds), exploration=b)


def test_class_objective_and_gradient():
    p = _pilco(0.5)
    val, grad = p.policy_gradient()
    terms, mu = p.reward_spec()
    plan = engine.RolloutPlan(p.mgpr.device_gp(), p.policy_spec(), terms, p.m_init.reshape(-1), p.S_init, p.horizon,
                              R=1, mult_mu=mu, grad=True, exploration=0.5)
    plan.forward()
    ref = p._flat_grad({k: v[0] for k, v in plan.backward().items()})
    assert val == float(plan.reward[0].item()) and np.array_equal(np.asarray(grad), ref)
    assert float(np.asarray(p.training_loss()).item()) == -val
    assert float(np.asarray(p.compute_reward()).item()) == val
    p.exploration = 0.0                                  # reassigned: the objective without the bonus
    v0, _ = p.policy_gradient()
    m, s = p.predict_reward_moments(p.m_init, p.S_init, p.horizon)
    assert abs(val - v0 - 0.5 * np.sqrt(np.asarray(s)).sum()) < 1e-9 * max(1.0, abs(val))


def test_predict_is_unchanged_by_exploration():
    p = _pilco(0.0)
    ref = [np.array(a) for a in p.predict(p.m_init, p.S_init, p.horizon)]
    for b in (0.7, -0.3):
        p.exploration = b
        got = p.predict(p.m_init, p.S_init, p.horizon)
        assert all(np.array_equal(np.asarray(g), r) for g, r in zip(got, ref))
        M, S = p.propagate(p.m_init, p.S_init)
        assert np.all(np.isfinite(M)) and np.all(np.isfinite(S))


def test_predict_reward_moments_match_compute_reward():
    p = _pilco(0.5, joint=False)
    n = 6
    mean, var = p.predict_reward_moments(p.m_init, p.S_init, n)
    assert mean.shape == (n,) and var.shape == (n,)
    for t in range(n):
        m, s = (p.m_init, p.S_init) if t == 0 else p.predict(p.m_init, p.S_init, t)[:2]
        mu, sr = p.reward.compute_reward(m, s)
        assert abs(mean[t] - float(np.asarray(mu).item())) <= 1e-10 * max(1.0, abs(mean[t]))
        assert abs(var[t] - float(np.asarray(sr).item())) <= 1e-10 * max(1e-3, abs(var[t]))


def test_optimize_policy_with_exploration():
    p = _pilco(0.5)
    start = -float(np.asarray(p.training_loss()).item())
    np.random.seed(1)
    best = p.optimize_policy(maxiter=20, restarts=8)
    end = -float(np.asarray(p.training_loss()).item())
    assert np.isfinite(best) and np.isfinite(end)
    assert end > start and abs(end - best) <= 1e-6 * max(1.0, abs(best))


def test_box_term_with_exploration_is_a_value_error():
    from pilco.models import PILCO
    from pilco.controllers import LinearController
    from safe_pilco_extension.rewards_safe import ObjectiveFunction, SingleConstraint
    X = np.random.RandomState(0).rand(20, 3)
    reward = ObjectiveFunction(rewards.ExponentialReward(2), SingleConstraint(0, high=0.5))
    p = PILCO((X, 0.1 * X[:, :2]), controller=LinearController(2, 1), horizon=4, reward=reward, exploration=0.5)
    with pytest.raises(ValueError, match="box"):
        p.policy_gradient()
    p.exploration = 0.0
    assert np.isfinite(p.policy_gradient()[0])


def test_safe_pilco_exploration():
    """SafePILCO(exploration=b): the bonus of the additive reward's sigma_t, the risk channel unchanged"""
    from safe_pilco_extension.safe_pilco import SafePILCO
    from safe_pilco_extension.rewards_safe import RiskOfCollision
    from pilco.controllers import LinearController
    X = np.random.RandomState(1).rand(30, 5)
    make = lambda b: SafePILCO((X, 0.1 * X[:, :4]), controller=LinearController(4, 1), horizon=4,
                               reward_add=rewards.ExponentialReward(4, t=0.5 * np.ones(4)),
                               reward_mult=RiskOfCollision(4, [0.0, 0.1], [0.6, 0.9]), mu=-4.0, exploration=b)
    p0, p1 = make(0.0), make(0.5)
    p1.controller.set_flat(p0.controller.get_flat())
    v0, v1 = p0.policy_gradient()[0], p1.policy_gradient()[0]
    m, s = p1.predict_reward_moments(p1.m_init, p1.S_init, p1.horizon)
    assert abs(v1 - v0 - 0.5 * np.sqrt(np.asarray(s)).sum()) < 1e-9 * max(1.0, abs(v1))
    assert float(np.asarray(p1.training_loss()).item()) == -v1
