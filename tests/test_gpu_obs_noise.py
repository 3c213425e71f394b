"""GPU tests of measurement noise at the policy's input (pilco_rollout_noisy_*, DESIGN.md section 22) through
engine.RolloutPlan and the class API: trajectory, rewards and step_var against the torch oracle
(tests/action_reward_oracle.py), the reverse sweep against autograd (taped and recomputing) and central differences, the
identities (nz == NULL, v = 0, batch position, graph replay) and PILCO(measurement_noise=...)."""
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


def _case(kind, R, Ds=3, U=2, dims=(), seed=9, n=50, bf=12, squash=True):
    Dh = Ds + len(dims)
    X, Y, ell, sf2, sn2 = make_gp_problem(n, Dh + U, Ds, seed=seed)
    Y = 0.1 * Y
    rng = np.random.RandomState(seed + 1)
    maxa = 0.7 + rng.rand(U)
    if kind == "linear":
        prm = (0.5 * rng.randn(R, U, Dh), 0.3 * rng.randn(R, U))
        spec = dict(kind=_lib.POLICY_LINEAR, Ds=Dh, U=U, squash=squash, max_action=maxa, W=prm[0], b=prm[1])
    else:
        prm = (rng.randn(R, bf, Dh) * 0.5 + 0.5, 0.1 * rng.randn(R, bf, U), 1.0 + 0.1 * rng.randn(R, U, Dh))
        pgp = engine.gp_factorize(*prm, np.ones((R, U)), 1e-4 * np.ones((R, U)), need_iK=False, mode=1)
        spec = dict(kind=_lib.POLICY_RBF, Ds=Dh, U=U, squash=squash, max_action=maxa, gp=pgp)
    B = rng.randn(Ds, Ds)
    P = dict(X=X, Y=Y, ell=ell, sf2=sf2, sn2=sn2, maxa=maxa if squash else None, m0=X[0, :Ds],
             S0=0.03 * B @ B.T + 0.02 * np.eye(Ds), v=0.01 + 0.05 * rng.rand(Ds), dims=list(dims), kind=kind, Ds=Ds,
             Dh=Dh, U=U)
    return P, spec, prm


def _terms(which, Ds, Dh, U, seed=0):
    """"state": exponential + linear state terms; "joint": an action cost (EXP_SA) and joint terms; "safe": the state
    terms with a MULT box risk (SafePILCO)"""
    rng = np.random.RandomState(seed)
    t = 0.4 * rng.randn(Ds)
    state = rewards.CombinedRewards(Ds, [rewards.ExponentialReward(Ds, W=np.diag(0.5 + rng.rand(Ds)), t=t),
                                         rewards.LinearReward(Ds, rng.randn(Ds))], coefs=[1.0, 0.3]).terms()
    if which == "state":
        return state
    if which == "safe":
        return state + [dict(kind=_lib.REWARD_BOX, coef=1.0, channel=_lib.CHANNEL_MULT, W=BOX2, t=None)]
    D = Dh + U
    combined = rewards.CombinedRewards(Ds, [rewards.ExponentialReward(Ds, t=t), rewards.action_cost(Dh, U)],
                                       coefs=[1.0, 0.2]).terms()
    return combined + [dict(kind=_lib.REWARD_LINEAR_SA, coef=0.3, W=rng.randn(D), t=None)]


def _plan(P, spec, terms, H, R, v, b=None, mu=1.5, grad=False, m0=None, S0=None):
    gp = engine.gp_factorize(P["X"], P["Y"], P["ell"], P["sf2"], P["sn2"])
    return engine.RolloutPlan(gp, spec, terms, P["m0"] if m0 is None else m0, P["S0"] if S0 is None else S0, H, R=R,
                              mult_mu=mu, grad=grad, angles=P["dims"] or None, exploration=b, measurement_noise=v)


def _oracle(P, prm_r, terms, H, v, b=0.0, mu=1.5, m0=None, S0=None):
    return aro.problem_rollout(P["kind"], prm_r, P["X"], P["Y"], P["ell"], P["sf2"], P["sn2"], P["maxa"], terms,
                               T(P["m0"]) if m0 is None else m0, T(P["S0"]) if S0 is None else S0, H, mult_mu=mu,
                               angle_dims=P["dims"] or None, v=v, b=b)


def _check_forward(plan, ref, r, H, tol=1e-10):
    out = dict(reward=plan.reward[r], step_reward=plan.step_reward[r, :H], traj_m=plan.traj_m[r], traj_S=plan.traj_S[r])
    if plan.step_var is not None:
        out["step_var"] = plan.step_var[r, :H]
    for k, v in out.items():
        o, e = v.cpu().numpy(), ref[k].detach().numpy()
        if e.size:
            assert scaled_err(o, e) <= tol, (k, r, scaled_err(o, e))


FORWARD = [  # policy, R, state dim, U, angles, terms, squash, b
    ("linear", 2, 3, 2, (), "state", True, None),
    ("linear", 2, 3, 2, (), "joint", False, None),
    ("rbf", 2, 3, 2, (), "joint", True, None),
    ("rbf", 2, 3, 1, (), "state", False, None),
    ("linear", 3, 4, 1, (1,), "joint", True, None),          # cart-pole-like
    ("rbf", 2, 4, 1, (1,), "state", True, None),
    ("linear", 2, 4, 1, (0, 2), "state", True, None),        # two angles
    ("rbf", 2, 4, 1, (1, 3), "joint", True, None),
    ("linear", 2, 3, 2, (), "safe", True, None),             # SafePILCO's MULT box
    ("rbf", 2, 4, 1, (1,), "joint", True, 0.5),              # with the exploration bonus
    ("linear", 2, 3, 2, (), "state", True, 0.5),
]


@pytest.mark.parametrize("kind,R,Ds,U,dims,which,squash,b", FORWARD)
def test_forward_matches_oracle(kind, R, Ds, U, dims, which, squash, b):
    H = 6
    P, spec, prm = _case(kind, R, Ds, U, dims, squash=squash)
    terms = _terms(which, Ds, P["Dh"], U)
    plan = _plan(P, spec, terms, H, R, P["v"], b=b)
    plan.forward()
    torch.cuda.synchronize()
    assert int(plan.info.max().item()) == 0
    for r in range(R):
        ref = _oracle(P, [T(p[r]) for p in prm], terms, H, P["v"], b=b or 0.0)
        _check_forward(plan, ref, r, H)
        bare = _oracle(P, [T(p[r]) for p in prm], terms, H, np.zeros(Ds), b=b or 0.0)
        assert float((ref["traj_S"][1:] - bare["traj_S"][1:]).abs().max()) > 1e-6       # the noise is visible


def test_metric_shape_matches_oracle():
    """N = 300, E = 10, D = 12, RBF policies with 50 centres, R = 32 restarts (first, middle, last checked)"""
    H, R = 10, 32
    pb = make_rollout_problem(300, 10, 2, 50, R, seed=0)
    pgp = engine.gp_factorize(pb["Xc"], pb["Yc"], pb["lc"], np.ones((R, 2)), 1e-4 * np.ones((R, 2)), need_iK=False, mode=1)
    spec = dict(kind=_lib.POLICY_RBF, Ds=10, U=2, squash=True, max_action=pb["maxa"], gp=pgp)
    terms = [dict(kind=_lib.REWARD_EXP, coef=1.0, W=0.5 * np.eye(10), t=pb["m0"])]
    v = 0.01 * np.linspace(0.5, 1.5, 10)
    P = dict(pb, dims=[], kind="rbf")
    plan = _plan(P, spec, terms, H, R, v, mu=0.0)
    plan.forward()
    torch.cuda.synchronize()
    for r in (0, 17, R - 1):
        ref = _oracle(P, [T(pb[k][r]) for k in ("Xc", "Yc", "lc")], terms, H, v, mu=0.0)
        _check_forward(plan, ref, r, H)


GRADS = [  # policy, state dim, U, angles, terms, squash, b
    ("linear", 3, 2, (), "joint", True, None),
    ("linear", 3, 2, (), "state", False, None),
    ("rbf", 3, 2, (), "safe", True, None),
    ("linear", 4, 1, (1,), "state", True, 0.5),
    ("rbf", 4, 1, (1,), "joint", True, None),
    ("rbf", 4, 1, (0, 2), "state", True, -0.5),
]


@pytest.mark.parametrize("kind,Ds,U,dims,which,squash,b", GRADS)
def test_gradient_matches_autograd(kind, Ds, U, dims, which, squash, b):
    """policy, gm0 and gS0 gradients of both sweeps against autograd of the oracle (1e-8 of the gradient's scale)"""
    H, R = 5, 2
    P, spec, prm = _case(kind, R, Ds, U, dims, seed=4, squash=squash)
    terms = _terms(which, Ds, P["Dh"], U, seed=1)
    names = ["W", "b"] if kind == "linear" else ["X", "Y", "ell"]
    for taped in (True, False):
        plan = _plan(P, spec, terms, H, R, P["v"], b=b, grad=taped)
        assert (plan.tape is not None) == taped
        plan.forward()
        g = {k: v.clone().cpu().numpy() for k, v in plan.backward().items()}
        torch.cuda.synchronize()
        for r in range(R):
            ps = [T(p[r]).requires_grad_() for p in prm]
            m0, S0 = T(P["m0"]).requires_grad_(), T(P["S0"]).requires_grad_()
            ref = _oracle(P, ps, terms, H, P["v"], b=b or 0.0, m0=m0, S0=S0)
            gref = torch.autograd.grad(ref["reward"], ps + [m0, S0])
            for k, gr in zip(names + ["m0", "S0"], gref):
                gr, o = gr.numpy(), g[k][r]
                if k == "S0":
                    gr, o = 0.5 * (gr + gr.T), 0.5 * (o + o.T)
                assert scaled_err(o, gr) <= 1e-8, (taped, k, r, scaled_err(o, gr))


def test_gradient_matches_central_differences():
    """d reward along a random direction of the linear policy's (W, b): restarts 1 and 2 carry theta +- h v"""
    H, Ds, U, h = 6, 4, 1, 1e-5
    P, spec, prm = _case("linear", 1, Ds, U, (1,), seed=13)
    terms = _terms("joint", Ds, P["Dh"], U, seed=2)
    rng = np.random.RandomState(3)
    vW, vb = rng.randn(U, P["Dh"]), rng.randn(U)
    W = np.stack([prm[0][0], prm[0][0] + h * vW, prm[0][0] - h * vW])
    bb = np.stack([prm[1][0], prm[1][0] + h * vb, prm[1][0] - h * vb])
    plan = _plan(P, dict(spec, W=W, b=bb), terms, H, 3, P["v"], grad=True)
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
    if plan.step_var is not None:
        out["step_var"] = plan.step_var
    out.update({"g" + k: v for k, v in grads.items()})
    return {k: v.clone() for k, v in out.items()}


@pytest.mark.parametrize("dims,b,taped", [((), None, True), ((), 0.5, False), ((1,), 0.5, True)])
def test_null_noise_is_bitwise_the_explore_call(dims, b, taped):
    """nz == NULL through the noisy entry points is the pilco_rollout_explore_* call on the same description"""
    Ds, U, H, R = 4 if dims else 3, 1 if dims else 2, 5, 2
    P, spec, prm = _case("rbf", R, Ds, U, dims, seed=21)
    terms = _terms("joint", Ds, P["Dh"], U, seed=3)
    base = _plan(P, spec, terms, H, R, None, b=b, grad=taped)
    base.forward()
    ref = _outputs(base, base.backward())
    ang = ctypes.byref(base.ang) if base.ang is not None else None
    ex = ctypes.byref(base.ex) if base.ex is not None else None
    _lib.check(_lib.lib.pilco_rollout_noisy_forward(ctypes.byref(base.ro), ang, ex, None, engine.stream_ptr()), "fwd")
    _lib.check(_lib.lib.pilco_rollout_noisy_backward(ctypes.byref(base.ro), ang, ex, None, ctypes.byref(base.grad),
                                                     engine.stream_ptr()), "bwd")
    got = _outputs(base, base.gbuf)
    torch.cuda.synchronize()
    for k in ref:
        assert torch.equal(ref[k], got[k]), k


@pytest.mark.parametrize("kind,dims,taped", [("linear", (), True), ("rbf", (), False), ("rbf", (1,), True)])
def test_zero_noise_matches_the_noiseless_call(kind, dims, taped):
    """v = 0 runs the noisy kernels; forward and gradients agree with the call without noise to 1e-12 of scale"""
    Ds, U, H, R = 4 if dims else 3, 1 if dims else 2, 6, 2
    P, spec, prm = _case(kind, R, Ds, U, dims, seed=25)
    terms = _terms("joint", Ds, P["Dh"], U, seed=7)
    out = []
    for v in (None, np.zeros(Ds)):
        plan = _plan(P, spec, terms, H, R, v, grad=taped)
        plan.forward()
        out.append(_outputs(plan, plan.backward()))
    torch.cuda.synchronize()
    for k in out[0]:
        a, e = out[1][k].cpu().numpy(), out[0][k].cpu().numpy()
        if k == "gS0":
            a, e = 0.5 * (a + a.swapaxes(-1, -2)), 0.5 * (e + e.swapaxes(-1, -2))
        assert scaled_err(a, e) <= 1e-12, (k, scaled_err(a, e))


def test_restart_does_not_follow_batch_size_or_position():
    H, Ds, U = 5, 3, 2
    P, spec, prm = _case("linear", 5, Ds, U, seed=31)
    terms = _terms("joint", Ds, Ds, U, seed=4)
    big = _plan(P, spec, terms, H, 5, P["v"], b=0.5, grad=True)
    big.forward()
    gbig = {k: v.clone() for k, v in big.backward().items()}
    for r in range(5):
        one = _plan(P, dict(spec, W=prm[0][r:r + 1], b=prm[1][r:r + 1]), terms, H, 1, P["v"], b=0.5, grad=True)
        one.forward()
        gone = one.backward()
        torch.cuda.synchronize()
        assert torch.equal(big.reward[r:r + 1], one.reward) and torch.equal(big.traj_S[r:r + 1], one.traj_S)
        assert torch.equal(big.step_var[r:r + 1], one.step_var)
        for k in gone:
            assert torch.equal(gbig[k][r:r + 1], gone[k]), (k, r)


def test_graph_replay_matches_eager():
    H, Ds, U, R = 5, 4, 1, 2
    P, spec, prm = _case("rbf", R, Ds, U, (1,), seed=41)
    terms = _terms("joint", Ds, P["Dh"], U, seed=5)
    plan = _plan(P, spec, terms, H, R, P["v"], b=-0.5, grad=True)
    plan.forward()
    eager = _outputs(plan, plan.backward())
    plan.capture(backward=True)
    for t in [plan.reward, plan.traj_S, plan.step_var] + list(plan.gbuf.values()):
        t.zero_()
    plan.replay()
    torch.cuda.synchronize()
    again = _outputs(plan, plan.gbuf)
    for k in eager:
        assert torch.equal(eager[k], again[k]), k


# ---- class API ---------------------------------------------------------------------------------------------------------
def _pilco(noise, ctrl="rbf", safe=False):
    from pilco.models import PILCO
    from pilco.controllers import LinearController, RbfController
    np.random.seed(0)
    Ds, U = 3, 1
    X0 = np.random.rand(80, Ds + U) * 2.0 - 1.0
    Y0 = 0.1 * np.sin(X0).dot(np.random.rand(Ds + U, Ds))
    reward = rewards.CombinedRewards(Ds, [rewards.ExponentialReward(Ds, t=np.array([0.8, 0.8, 0.8])),
                                          rewards.action_cost(Ds, U, [[1.0]])], coefs=[1.0, 0.1])
    c = RbfController(Ds, U, 10, max_action=2.0) if ctrl == "rbf" else LinearController(Ds, U, max_action=2.0)
    if safe:
        from safe_pilco_extension.safe_pilco import SafePILCO
        from safe_pilco_extension.rewards_safe import RiskOfCollision
        return SafePILCO((X0, Y0), controller=c, horizon=8, reward_add=rewards.ExponentialReward(Ds, t=0.5 * np.ones(Ds)),
                         reward_mult=RiskOfCollision(Ds, [0.0, 0.1], [0.6, 0.9]), mu=-4.0, m_init=np.zeros((1, Ds)),
                         S_init=0.05 * np.eye(Ds), measurement_noise=noise)
    return PILCO((X0, Y0), controller=c, horizon=8, reward=reward, m_init=np.zeros((1, Ds)), S_init=0.05 * np.eye(Ds),
                 measurement_noise=noise)


def test_class_none_is_bitwise_today():
    p, q = _pilco(None), _pilco(None)
    q.measurement_noise = None
    ref = [np.array(a) for a in p.predict(p.m_init, p.S_init, 8)]
    plan = p._single_plan(p.m_init, p.S_init, 8, grad=True)
    assert plan.nz is None
    got = q.predict(q.m_init, q.S_init, 8)
    assert all(np.array_equal(np.asarray(g), r) for g, r in zip(got, ref))


def test_class_model_equals_explicit_array_and_follows_the_model():
    p = _pilco("model")
    v = np.asarray(p.mgpr.noise, dtype=np.float64) / 2.0
    q = _pilco(v)
    a, b = p.predict(p.m_init, p.S_init, 8), q.predict(q.m_init, q.S_init, 8)
    assert all(np.array_equal(np.asarray(x), np.asarray(y)) for x, y in zip(a, b))
    assert np.array_equal(np.asarray(p.policy_gradient()[1]), np.asarray(q.policy_gradient()[1]))
    bare = _pilco(None).predict(p.m_init, p.S_init, 8)
    assert not np.array_equal(np.asarray(bare[1]), np.asarray(a[1]))
    for m in p.mgpr.models:                              # a new noise level: "model" reads it again (cache key)
        m.likelihood.variance.assign(np.asarray(m.likelihood.variance) * 4.0)
    c = p.predict(p.m_init, p.S_init, 8)
    assert not np.array_equal(np.asarray(c[1]), np.asarray(a[1]))


def test_class_predict_equals_repeated_propagate():
    p = _pilco(np.array([0.02, 0.01, 0.03]))
    m, s = p.m_init, p.S_init
    for _ in range(4):
        m, s = p.propagate(m, s)
    M, S, _ = p.predict(p.m_init, p.S_init, 4)
    assert np.max(np.abs(np.asarray(M) - np.asarray(m))) <= 1e-12 and np.max(np.abs(np.asarray(S) - np.asarray(s))) <= 1e-12


@pytest.mark.parametrize("ctrl", ["linear", "rbf"])
def test_class_policy_gradient_matches_central_differences(ctrl):
    p = _pilco(np.array([0.02, 0.01, 0.03]), ctrl=ctrl)
    val, grad = p.policy_gradient()
    assert abs(val + float(np.asarray(p.training_loss()).item())) <= 1e-12 * max(1.0, abs(val))
    flat = p.controller.get_flat().copy()
    d = np.random.RandomState(2).randn(flat.size)
    h, vals = 1e-5, []
    for sgn in (1.0, -1.0):
        p.controller.set_flat(flat + sgn * h * d)
        vals.append(p.policy_gradient()[0])
    p.controller.set_flat(flat)
    fd = (vals[0] - vals[1]) / (2 * h)
    ad = float(np.dot(np.asarray(grad), d))
    assert abs(fd - ad) < 1e-6 * max(1.0, abs(ad)), (fd, ad)


def test_class_optimize_policy_raises_the_noisy_objective():
    p = _pilco("model", safe=True)
    start = -float(np.asarray(p.training_loss()).item())
    np.random.seed(1)
    best = p.optimize_policy(maxiter=20, restarts=8)
    end = -float(np.asarray(p.training_loss()).item())
    assert np.isfinite(best) and np.isfinite(end)
    assert end > start and abs(end - best) <= 1e-6 * max(1.0, abs(best))


def test_class_particle_methods_raise():
    p = _pilco(np.array([0.02, 0.01, 0.03]))
    for call in (lambda: p.sample_trajectories(p.m_init, p.S_init, 3, num_samples=16),
                 lambda: p.sample_policy_gradient(p.m_init, p.S_init, 3, num_samples=16),
                 lambda: p.optimize_policy_sampled(maxiter=2, num_samples=16)):
        with pytest.raises(ValueError, match="measurement_noise"):
            call()
    with pytest.raises(ValueError, match="measurement_noise"):
        _pilco(np.array([0.1, -0.1, 0.1]))
