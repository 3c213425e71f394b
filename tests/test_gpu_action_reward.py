"""Reward terms on the joint state-action Gaussian on the device (PILCO_REWARD_EXP_SA / PILCO_REWARD_LINEAR_SA, DESIGN.md
section 18), through the C ABI plans of pilco_b200.engine and through the class API: the moment-matching rollout and
its reverse sweep against the torch oracle and autograd (tests/action_reward_oracle.py), the identity with state terms
when the action block is zero, the particle rollouts and their three gradient estimators against the numpy / autograd
oracles given the same x0 and eps, bitwise independence and graph replay, and policy optimisation with an action cost."""
import numpy as np
import pytest
import torch

from pilco_b200 import engine, _lib, rewards
import action_reward_oracle as aro
import particle_oracle as po
from particle_cases import BOX2, _case, _draw, _dyn_np, _linear, _oracle_pol, _rbf
from particle_grad_oracle import T, score_grad, value_and_grad
from util import make_gp_problem, make_rollout_problem, scaled_err

pytestmark = pytest.mark.gpu


def _joint_terms(Ds, U, seed=0, box=True):
    """state exp / linear / box terms mixed with joint exp / linear terms on both channels"""
    rng = np.random.RandomState(seed)
    D = Ds + U
    B = rng.randn(D, D) / np.sqrt(D)
    Q = np.zeros((D, D)); Q[Ds:, Ds:] = 2.0 * np.eye(U)
    terms = [dict(kind=_lib.REWARD_EXP, coef=1.0, W=np.eye(Ds), t=0.5 * np.ones(Ds)),
             dict(kind=_lib.REWARD_EXP_SA, coef=-0.5, W=B @ B.T, t=0.3 * rng.rand(D)),
             dict(kind=_lib.REWARD_LINEAR, coef=0.3, W=rng.randn(Ds), t=None),
             dict(kind=_lib.REWARD_LINEAR_SA, coef=0.2, W=rng.randn(D), t=None),
             dict(kind=_lib.REWARD_EXP_SA, coef=0.1, channel=_lib.CHANNEL_MULT, W=Q, t=np.zeros(D)),
             dict(kind=_lib.REWARD_LINEAR_SA, coef=0.01, channel=_lib.CHANNEL_MULT, W=rng.randn(D), t=None),
             dict(kind=_lib.REWARD_EXP, coef=0.1, channel=_lib.CHANNEL_MULT, W=2.0 * np.eye(Ds), t=np.zeros(Ds))]
    if box:
        terms.append(dict(kind=_lib.REWARD_BOX, coef=-0.2, W=BOX2, t=None))
    return terms


def _mm_case(kind, R, squash, Ds=3, U=2, n=50, bf=12, seed=9):
    X, Y, ell, sf2, sn2 = make_gp_problem(n, Ds + U, Ds, seed=seed)
    Y = 0.1 * Y
    rng = np.random.RandomState(seed + 1)
    maxa = 0.7 + rng.rand(U)
    if kind == "linear":
        prm = (0.5 * rng.randn(R, U, Ds), 0.3 * rng.randn(R, U))
        spec = dict(kind=_lib.POLICY_LINEAR, Ds=Ds, U=U, squash=squash, max_action=maxa, W=prm[0], b=prm[1])
    else:
        prm = (rng.randn(R, bf, Ds) * 0.5 + 0.5, 0.1 * rng.randn(R, bf, U), 1.0 + 0.1 * rng.randn(R, U, Ds))
        pgp = engine.gp_factorize(*prm, np.ones((R, U)), 1e-4 * np.ones((R, U)), need_iK=False, mode=1)
        spec = dict(kind=_lib.POLICY_RBF, Ds=Ds, U=U, squash=squash, max_action=maxa, gp=pgp)
    return dict(X=X, Y=Y, ell=ell, sf2=sf2, sn2=sn2, maxa=maxa, m0=X[0, :Ds], S0=0.05 * np.eye(Ds)), spec, prm


def _oracle(P, kind, prm_r, terms, H, mu, squash, **kw):
    return aro.problem_rollout(kind, prm_r, P["X"], P["Y"], P["ell"], P["sf2"], P["sn2"], P["maxa"] if squash else None,
                               terms, P["m0"], P["S0"], H, mult_mu=mu, **kw)


def _check_forward(plan, ref, r, H, tol=1e-10):
    out = dict(traj_m=plan.traj_m[r], traj_S=plan.traj_S[r], step_reward=plan.step_reward[r, :H],
               step_risk=plan.step_risk[r, :H], reward=plan.reward[r])
    for k, v in out.items():
        o, e = v.cpu().numpy(), ref[k].detach().numpy()
        if e.size:
            assert scaled_err(o, e) <= tol, (k, scaled_err(o, e))


@pytest.mark.parametrize("kind,R,squash,H", [("linear", 1, True, 4), ("linear", 5, False, 4), ("rbf", 1, False, 4),
                                             ("rbf", 5, True, 4), ("linear", 1, True, 0), ("rbf", 1, True, 1)])
def test_forward_and_backward_match_oracle(kind, R, squash, H):
    """reward, step_reward, step_risk, traj_m, traj_S vs the torch oracle (1e-10 of scale) and pilco_rollout_backward vs
    autograd (1e-7 of the gradient's scale, gm0 / gS0 included), taped and recomputing paths agreeing to round-off"""
    P, spec, prm = _mm_case(kind, R, squash)
    terms, mu = _joint_terms(3, 2, seed=R), 1.5
    grads = {}
    for taped in (True, False):
        plan = engine.RolloutPlan(engine.gp_factorize(P["X"], P["Y"], P["ell"], P["sf2"], P["sn2"]), spec, terms,
                                  P["m0"], P["S0"], H, R=R, mult_mu=mu, grad=taped)
        assert (plan.tape is not None) == (taped and H > 0)
        plan.forward()
        assert int(plan.info.max().item()) == 0
        grads[taped] = {k: v.clone().cpu().numpy() for k, v in plan.backward().items()}
    names = ["W", "b"] if kind == "linear" else ["X", "Y", "ell"]
    for k in names + ["m0", "S0"]:
        a, b = grads[True][k], grads[False][k]
        assert np.abs(a - b).max() <= 1e-8 * max(np.abs(b).max(), 1e-300), k
    for r in range(R):
        ps = [T(p[r]).requires_grad_() for p in prm]
        m0, S0 = T(P["m0"]).requires_grad_(), T(P["S0"]).requires_grad_()
        ref = _oracle(dict(P, m0=m0, S0=S0), kind, ps, terms, H, mu, squash)
        _check_forward(plan, ref, r, H)
        if H == 0:
            assert not any(np.any(grads[True][k][r]) for k in names)
            continue
        gref = torch.autograd.grad(ref["reward"], ps + [m0, S0])
        for k, g in zip(names + ["m0", "S0"], gref):
            g, o = g.numpy(), grads[True][k][r]
            if k == "S0":                                           # the symmetric part is what is defined
                g, o = 0.5 * (g + g.T), 0.5 * (o + o.T)
            err = scaled_err(o, g)
            assert err <= 1e-7, "%s r=%d: %g" % (k, r, err)


def test_smgpr_d16_and_long_horizon():
    """a FITC dynamics model at D = 16 (Ds = 14, U = 2) and H = 40 steps at the metric shape, forward vs the oracle"""
    from oracle import torch_port as tp
    pb = make_rollout_problem(400, 14, 2, 10, 1, seed=4)
    Z = np.random.RandomState(5).rand(60, 16)
    gp = engine.fitc_factorize(pb["X"], Z, pb["Y"], pb["ell"], pb["sf2"], pb["sn2"])
    spec, _ = _rbf(pb["Xc"][0], pb["Yc"][0], pb["lc"][0], pb["maxa"])
    terms = _joint_terms(14, 2, seed=3, box=False)
    plan = engine.RolloutPlan(gp, spec, terms, pb["m0"], pb["S0"], 3, R=1, mult_mu=0.7)
    plan.forward()
    fact = tp.fitc_factorizations(T(pb["X"]), T(Z), T(pb["Y"]), T(pb["ell"]), T(pb["sf2"]), T(pb["sn2"]))
    P = dict(pb, maxa=pb["maxa"])
    ref = _oracle(P, "rbf", [T(pb[k][0]) for k in ("Xc", "Yc", "lc")], terms, 3, 0.7, True, fact=fact, Z=Z)
    _check_forward(plan, ref, 0, 3, tol=1e-7)
    pb = make_rollout_problem(300, 10, 2, 50, 1, seed=0)
    gp = engine.gp_factorize(pb["X"], pb["Y"], pb["ell"], pb["sf2"], pb["sn2"])
    spec, _ = _rbf(pb["Xc"][0], pb["Yc"][0], pb["lc"][0], pb["maxa"])
    terms = _joint_terms(10, 2, seed=6)
    plan = engine.RolloutPlan(gp, spec, terms, pb["m0"], pb["S0"], 40, R=1, mult_mu=0.7)
    plan.forward()
    ref = _oracle(pb, "rbf", [T(pb[k][0]) for k in ("Xc", "Yc", "lc")], terms, 40, 0.7, True)
    _check_forward(plan, ref, 0, 40, tol=1e-9)


def test_zero_action_block_equals_state_terms_on_device():
    P, spec, _ = _mm_case("rbf", 2, True)
    rng = np.random.RandomState(2)
    B = rng.randn(3, 3)
    Ws, ts, wl = B @ B.T, rng.rand(3), rng.randn(3)
    Wj = np.zeros((5, 5)); Wj[:3, :3] = Ws
    state = [dict(kind=_lib.REWARD_EXP, coef=0.7, W=Ws, t=ts), dict(kind=_lib.REWARD_LINEAR, coef=0.3, W=wl, t=None)]
    joint = [dict(kind=_lib.REWARD_EXP_SA, coef=0.7, W=Wj, t=np.append(ts, [0.9, -0.4])),
             dict(kind=_lib.REWARD_LINEAR_SA, coef=0.3, W=np.append(wl, [0.0, 0.0]), t=None)]
    gp = engine.gp_factorize(P["X"], P["Y"], P["ell"], P["sf2"], P["sn2"])
    out = []
    for terms in (state, joint):
        plan = engine.RolloutPlan(gp, spec, terms, P["m0"], P["S0"], 6, R=2, grad=True)
        plan.forward()
        g = plan.backward()
        out.append((plan.traj_m.clone(), plan.traj_S.clone(), plan.reward.cpu().numpy().copy(),
                    {k: v.cpu().numpy().copy() for k, v in g.items()}))
    (ma, Sa, ra, ga), (mb, Sb, rb, gb) = out
    assert torch.equal(ma, mb) and torch.equal(Sa, Sb)
    assert np.abs(ra - rb).max() <= 1e-14 * np.abs(ra).max()
    for k in ga:
        assert np.abs(ga[k] - gb[k]).max() <= 1e-11 * np.abs(ga[k]).max(), k
    x0, eps = _draw(P["m0"], P["S0"], 64, 6, seed=1)
    spec1, _ = _rbf(spec["gp"].X[0].cpu().numpy(), spec["gp"].Y[0].cpu().numpy(), spec["gp"].ell[0].cpu().numpy(), P["maxa"])
    pa, pb_ = (engine.particles_rollout(gp, spec1, t, x0, eps) for t in (state, joint))
    assert torch.equal(pa[0], pb_[0]) and torch.equal(pa[1], pb_[1])
    assert (pa[4] - pb_[4]).abs().max().item() <= 1e-14 * pa[4].abs().max().item()


def _particle_case(name):
    gp, spec, pol, _, m0, S0, H, P, mu = _case(name)
    terms = _joint_terms(spec["Ds"], spec["U"], seed=H)
    return gp, spec, pol, terms, m0, S0, min(H, 10), min(P, 300), mu


@pytest.mark.parametrize("consistent", [False, True])
@pytest.mark.parametrize("name", ["metric_rbf", "linear_nosquash"])
def test_particle_values_match_oracle(name, consistent):
    gp, spec, pol, terms, m0, S0, H, P, mu = _particle_case(name)
    x0, eps = _draw(m0, S0, P, H, seed=P + H)
    out = [t.cpu().numpy() for t in engine.particles_rollout(gp, spec, terms, x0, eps, mult_mu=mu, consistent=consistent)]
    if consistent:
        # the function-sample chain has its own oracle for the states; the reward terms are checked at the device's points
        traj, act = out[0], out[1]
        rew, risk = po.path_rewards(terms, traj, act)
        ref = (traj, act, rew, risk, po.particle_return(terms, rew, risk, mu))
        step0 = engine.particles_rollout(gp, spec, terms, x0, eps, mult_mu=mu)
        assert np.array_equal(step0[2][:, 0].cpu().numpy(), out[2][:, 0])           # step 0 is the marginal sampler's
    else:
        ref = po.particle_rollout(_dyn_np(gp), pol, terms, x0, eps, mult_mu=mu)
    for what, o, r in zip(("traj", "act", "reward", "risk", "ret"), out, ref):
        assert scaled_err(o, r) <= 1e-9, (what, scaled_err(o, r))


def _grad(gp, spec, terms, x0, eps, mu, estimator="pathwise", consistent=False, R=1):
    if consistent:
        plan = engine.ConsistentGradPlan(gp, spec, terms, x0.shape[0], eps.shape[1], mult_mu=mu, R=R)
    else:
        plan = engine.ParticlePlan(gp, spec, terms, x0.shape[0], eps.shape[1], mult_mu=mu, grad=True, R=R, estimator=estimator)
    plan.set_inputs(x0, eps)
    g = plan.launch_grad()
    return plan, {k: v.cpu().numpy().copy() for k, v in g.items()}


@pytest.mark.parametrize("name", ["metric_rbf", "linear_squash", "linear_nosquash", "fitc"])
def test_pathwise_gradient_matches_autograd(name):
    gp, spec, pol, terms, m0, S0, H, P, mu = _particle_case(name)
    terms = [t for t in terms if t["kind"] != _lib.REWARD_BOX]
    x0, eps = _draw(m0, S0, P, H, seed=P + H + 1)
    plan, g = _grad(gp, spec, terms, x0, eps, mu)
    v, ref = value_and_grad(_dyn_np(gp), _oracle_pol(spec, pol), terms, x0, eps, mu)
    scale = max(float(np.abs(r).max()) for r in ref.values())
    err = max(float(np.abs(g[k] - ref[k]).max()) for k in ref) / scale
    assert err <= (1e-6 if name == "fitc" else 1e-8), err
    assert abs(float(g["value"][0]) - v) <= 1e-9 * abs(v)
    fwd = engine.particles_rollout(gp, spec, terms, x0, eps, mult_mu=mu)
    for a, b in zip(plan.outputs(), fwd):
        assert torch.equal(a, b)
    # H = 1: the only step is the last one, which has no transition but still an action cost
    _, g1 = _grad(gp, spec, terms, x0, eps[:, :1], mu)
    _, r1 = value_and_grad(_dyn_np(gp), _oracle_pol(spec, pol), terms, x0, eps[:, :1], mu)
    s1 = max(float(np.abs(r).max()) for r in r1.values())
    assert s1 > 0 and max(float(np.abs(g1[k] - r1[k]).max()) for k in r1) <= 1e-8 * s1


def test_consistent_gradient_directional_difference():
    """the consistent rollout's pathwise gradient with joint terms against a central difference of its own value"""
    gp, spec, pol, terms, m0, S0, H, P, mu = _particle_case("linear_squash")
    terms = [t for t in terms if t["kind"] != _lib.REWARD_BOX]
    H, P = 5, 64
    x0, eps = _draw(m0, S0, P, H, seed=11)
    _, g = _grad(gp, spec, terms, x0, eps, mu, consistent=True)
    rng = np.random.RandomState(12)
    dW, db = rng.randn(*g["W"].shape), rng.randn(*g["b"].shape)
    h = 1e-5
    val = lambda s: _grad(gp, dict(spec, W=spec["W"] + s * h * dW, b=spec["b"] + s * h * db), terms, x0, eps, mu,
                          consistent=True)[1]["value"][0]
    fd, gv = (val(1) - val(-1)) / (2 * h), float((g["W"] * dW).sum() + (g["b"] * db).sum())
    assert abs(fd - gv) <= 1e-6 * abs(gv), (fd, gv)


@pytest.mark.parametrize("name", ["metric_rbf", "linear_squash"])
def test_score_gradient_matches_oracle_and_direct_term(name):
    gp, spec, pol, terms, m0, S0, H, P, mu = _particle_case(name)
    x0, eps = _draw(m0, S0, P, H, seed=5)
    plan, g = _grad(gp, spec, terms, x0, eps, mu, estimator="score")
    traj = plan.traj.cpu().numpy()
    dyn, opol = _dyn_np(gp), _oracle_pol(spec, pol)
    ref = score_grad(dyn, opol, terms, traj, eps, mu)
    scale = max(float(np.abs(r).max()) for r in ref.values())
    assert max(float(np.abs(g[k] - ref[k]).max()) for k in ref) <= 1e-6 * scale
    # the direct term alone: H = 1 has no transition with a reward after it, so the whole gradient is the direct term
    _, g1 = _grad(gp, spec, terms, x0, eps[:, :1], mu, estimator="score")
    d1 = score_grad(dyn, opol, terms, traj[:, :2], eps[:, :1], mu, transitions=False)
    s1 = max(float(np.abs(r).max()) for r in d1.values())
    assert s1 > 0 and max(float(np.abs(g1[k] - d1[k]).max()) for k in d1) <= 1e-9 * s1
    pw = _grad(gp, spec, terms, x0, eps, mu)[0]
    assert torch.equal(plan.ret, pw.ret) and torch.equal(plan.rew_buf, pw.rew_buf)


def test_score_estimator_agrees_with_pathwise_in_expectation():
    """smooth terms (no box): the mean of the score gradient over independent seeds is within 5 standard errors of the
    pathwise one's"""
    X, Y, ell, sf2, sn2 = make_gp_problem(100, 5, 4, seed=6)
    gp = engine.gp_factorize(X, 0.1 * Y, ell, 0.1 * sf2, 1e-3 * np.ones(4))
    rng = np.random.RandomState(7)
    spec, _ = _linear(0.5 * rng.randn(1, 4), rng.randn(1), np.array([1.3]), True)
    terms = [dict(kind=_lib.REWARD_EXP, coef=1.0, W=np.eye(4), t=0.5 * np.ones(4)),
             dict(kind=_lib.REWARD_EXP_SA, coef=1.0, W=np.diag([0, 0, 0, 0, 2.0]), t=np.zeros(5))]
    m0, S0, H, P = X[0, :4], 0.05 * np.eye(4), 4, 4096
    sc, pw = [], []
    for seed in range(24):
        x0, eps = _draw(m0, S0, P, H, seed=100 + seed)
        sc.append(np.concatenate([_grad(gp, spec, terms, x0, eps, 0.0, estimator="score")[1][k].ravel() for k in ("W", "b")]))
        pw.append(np.concatenate([_grad(gp, spec, terms, x0, eps, 0.0)[1][k].ravel() for k in ("W", "b")]))
    sc, pw = np.array(sc), np.array(pw)
    se = np.sqrt(sc.var(0, ddof=1) / len(sc) + pw.var(0, ddof=1) / len(pw))
    z = np.abs(sc.mean(0) - pw.mean(0)) / se
    assert z.max() <= 5.0, z


def test_bitwise_independence_and_graph_replay():
    gp, spec, pol, terms, m0, S0, H, P, mu = _particle_case("metric_rbf")
    terms = [t for t in terms if t["kind"] != _lib.REWARD_BOX]
    x0, eps = _draw(m0, S0, P, H, seed=9)
    full = engine.particles_rollout(gp, spec, terms, x0, eps, mult_mu=mu)
    perm = np.random.RandomState(1).permutation(P)[:97]
    part = engine.particles_rollout(gp, spec, terms, x0[perm], eps[perm], mult_mu=mu)
    for a, b in zip(full, part):
        assert torch.equal(a[torch.as_tensor(perm, device=a.device)], b)
    # R policies at once: restart r's results are those of the single-policy call, for every estimator
    pb = make_rollout_problem(300, 10, 2, 50, 3, seed=5)
    pgp = engine.gp_factorize(pb["Xc"], pb["Yc"], pb["lc"], np.ones((3, 2)), 1e-4 * np.ones((3, 2)), need_iK=False, mode=1)
    bspec = dict(spec, gp=pgp)
    for est, cons in (("pathwise", False), ("score", False), ("pathwise", True)):
        x0s, epss = x0[:64], eps[:64, :5]
        bplan, bg = _grad(gp, bspec, terms, x0s, epss, mu, estimator=est, consistent=cons, R=3)
        s1, _ = _rbf(pb["Xc"][1], pb["Yc"][1], pb["lc"][1], pb["maxa"])
        splan, sg = _grad(gp, s1, terms, x0s, epss, mu, estimator=est, consistent=cons)
        assert torch.equal(bplan.ret[1], splan.ret.reshape(-1)), (est, cons)
        for k in ("X", "Y", "ell"):
            assert np.array_equal(bg[k][1], sg[k].reshape(bg[k][1].shape)), (est, cons, k)
        assert bg["value"][1] == sg["value"][0]
    # graph replay: bitwise the eager results
    for est in ("pathwise", "score"):
        plan, g = _grad(gp, spec, terms, x0, eps, mu, estimator=est)
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            plan.launch_grad()
        for v in plan.gbuf.values():
            v.zero_()
        graph.replay()
        torch.cuda.synchronize()
        for k in g:
            assert np.array_equal(plan.gbuf[k].cpu().numpy(), g[k]), (est, k)
    P_, spec_, _ = _mm_case("rbf", 2, True)
    rp = engine.RolloutPlan(engine.gp_factorize(P_["X"], P_["Y"], P_["ell"], P_["sf2"], P_["sn2"]), spec_,
                            _joint_terms(3, 2), P_["m0"], P_["S0"], 5, R=2, mult_mu=1.0, grad=True)
    rp.forward()
    eager = {k: v.clone() for k, v in rp.backward().items()}
    reward = rp.reward.clone()
    rp.capture(backward=True)
    rp.replay()
    torch.cuda.synchronize()
    assert torch.equal(rp.reward, reward) and all(torch.equal(rp.gbuf[k], eager[k]) for k in eager)


def test_plan_rejects_wrong_shapes_before_device_work():
    P, spec, _ = _mm_case("linear", 1, True)
    gp = engine.gp_factorize(P["X"], P["Y"], P["ell"], P["sf2"], P["sn2"])
    bad = [rewards.ExponentialStateActionReward(3, 1).terms(),                   # control_dim does not match the policy
           [dict(kind=_lib.REWARD_EXP_SA, coef=1.0, W=np.eye(3), t=np.zeros(3))],   # W is [Ds,Ds], not [D,D]
           [dict(kind=_lib.REWARD_LINEAR_SA, coef=1.0, W=np.ones(3), t=None)]]
    for terms in bad:
        with pytest.raises(ValueError):
            engine.RolloutPlan(gp, spec, terms, P["m0"], P["S0"], 3)
        with pytest.raises(ValueError):
            engine.ParticlePlan(gp, spec, terms, 8, 3)


def _pendulum_like(cost):
    from pilco.models import PILCO
    from pilco.controllers import RbfController
    from pilco.rewards import ExponentialReward, CombinedRewards, action_cost
    np.random.seed(0)
    Ds, U = 3, 1
    X0 = np.random.rand(80, Ds + U) * 2.0 - 1.0
    A = np.random.rand(Ds + U, Ds)
    Y0 = 0.1 * np.sin(X0).dot(A)
    base = ExponentialReward(Ds, t=np.array([0.8, 0.8, 0.8]))
    reward = CombinedRewards(Ds, [base, action_cost(Ds, U, [[1.0]])], coefs=[1.0, cost]) if cost else base
    ctrl = RbfController(Ds, U, 10, max_action=2.0)
    p = PILCO((X0, Y0), controller=ctrl, horizon=10, reward=reward, m_init=np.zeros((1, Ds)), S_init=0.05 * np.eye(Ds))
    return p


def _mean_abs_u(p):
    res = p.sample_trajectories(p.m_init, p.S_init, p.horizon, num_samples=512, seed=3)
    return float(np.abs(np.asarray(res.actions)).mean())


@pytest.mark.parametrize("sampled", [False, True])
def test_action_cost_lowers_control_effort(sampled):
    """optimize_policy / optimize_policy_sampled with an action cost run, stay finite and end with a smaller mean |u|
    along the sampled trajectories than the same run without the cost"""
    us = []
    for cost in (0.0, 2.0):
        p = _pendulum_like(cost)
        np.random.seed(1)
        v = p.optimize_policy_sampled(maxiter=25, num_samples=256, seed=2) if sampled else p.optimize_policy(maxiter=25)
        assert np.isfinite(v)
        m, S, r = p.predict(p.m_init, p.S_init, p.horizon)
        assert np.all(np.isfinite(m)) and np.all(np.isfinite(S)) and np.isfinite(r).all()
        r = float(np.asarray(r).reshape(-1)[0])
        r2, g = p.policy_gradient()
        assert abs(r2 - r) <= 1e-9 * max(1.0, abs(r2)) and np.all(np.isfinite(g))
        assert float(np.asarray(p.compute_reward()).reshape(-1)[0]) == pytest.approx(r, rel=1e-12)
        for est in ("pathwise", "score"):
            assert np.all(np.isfinite(p.sample_policy_gradient(p.m_init, p.S_init, 5, num_samples=64, seed=1, estimator=est).grad))
        assert np.all(np.isfinite(p.sample_policy_gradient(p.m_init, p.S_init, 5, num_samples=32, seed=1, consistent=True).grad))
        assert np.all(np.isfinite(p.sample_trajectories(p.m_init, p.S_init, 5, num_samples=32, seed=1, consistent=True).returns))
        us.append(_mean_abs_u(p))
    print("mean |u| without / with the action cost (%s): %.4f / %.4f" % ("sampled" if sampled else "moment matching", us[0], us[1]))
    assert us[1] < us[0]


def test_safe_pilco_takes_a_joint_reward_add():
    from pilco_b200.safe import SafePILCO, SingleConstraint
    from pilco.rewards import ExponentialReward, CombinedRewards, action_cost
    np.random.seed(0)
    X0 = np.random.rand(40, 3)
    Y0 = 0.1 * np.sin(X0).dot(np.random.rand(3, 2))
    add = CombinedRewards(2, [ExponentialReward(2), action_cost(2, 1)], coefs=[1.0, 0.3])
    p = SafePILCO((X0, Y0), horizon=5, reward_add=add, reward_mult=SingleConstraint(0, high=0.9), mu=-2.0)
    kinds = [t["kind"] for t in p.reward_spec()[0]]
    assert kinds == [_lib.REWARD_EXP, _lib.REWARD_EXP_SA, _lib.REWARD_BOX]
    r = p.predict(p.m_init, p.S_init, 5)[2]
    assert np.isfinite(r).all()
    assert np.all(np.isfinite(p.policy_gradient()[1]))
