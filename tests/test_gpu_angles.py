"""GPU tests of the moment-matching rollout with angular state dimensions (pilco_trig_moments,
pilco_rollout_angles_forward / _backward through engine.RolloutPlan(angles=...)): the feature map's moments against
the host build of the same formulas, the cascade against the torch statement in tests/action_reward_oracle.py, the
reverse sweep against torch autograd (taped and recomputing), periodicity in the angles, and CUDA-graph replay."""
import numpy as np
import pytest
import torch

from pilco_b200 import _lib
import action_reward_oracle as aro
from util import TRIG_CASES, host_moments, make_gp_problem, scaled_err, trig_harness

pytestmark = pytest.mark.gpu
T = lambda a: torch.tensor(np.asarray(a), dtype=torch.float64)


def test_trig_moments_match_host_build(tmp_path):
    from pilco_b200 import engine
    lib = trig_harness(str(tmp_path / "trig_harness.so"))
    for name, m, s, dims in TRIG_CASES:
        M, S, C = engine.trig_moments(m[None], s[None], dims)
        hM, hS, hC = host_moments(lib, m, s, dims)
        for got, ref in ((M[0], hM), (S[0], hS), (C[0], hC)):
            assert np.max(np.abs(got.cpu().numpy() - ref)) < 1e-14, name


def _problem(Ds, dims, U, kind, R, seed=0, singular=False, joint=False):
    from pilco_b200 import engine, _lib
    A = len(dims)
    Dh, D = Ds + A, Ds + A + U
    n, bf = 60, 12
    X, Y, ell, sf2, sn2 = make_gp_problem(n, D, Ds, seed=seed)
    Y = 0.05 * Y
    gp = engine.gp_factorize(X, Y, ell, sf2, sn2)
    rng = np.random.RandomState(seed + 1)
    maxa = 1.5 * np.ones(U)
    if kind == "linear":
        W, b = 0.3 * rng.randn(R, U, Dh), 0.1 * rng.randn(R, U)
        spec = dict(kind=_lib.POLICY_LINEAR, Ds=Dh, U=U, squash=True, max_action=maxa, W=W, b=b)
        pol = dict(W=W, b=b)
    else:
        Xc, Yc, lc = rng.randn(R, bf, Dh) * 0.5, 0.3 * rng.randn(R, bf, U), 1.0 + 0.1 * rng.randn(R, U, Dh)
        pgp = engine.gp_factorize(Xc, Yc, lc, np.ones((R, U)), 1e-4 * np.ones((R, U)), need_iK=False, mode=1)
        spec = dict(kind=_lib.POLICY_RBF, Ds=Dh, U=U, squash=True, max_action=maxa, gp=pgp)
        pol = dict(X=Xc, Y=Yc, ell=lc)
    Wr = np.diag(rng.rand(Ds) + 0.5)
    for a in dims:                                   # no state term reads an angle (periodicity test)
        Wr[a, a] = 0.0
    tr = 0.2 * rng.randn(Ds)
    terms = [dict(kind=_lib.REWARD_EXP, coef=1.0, W=Wr, t=tr)]
    Wj = tj = None
    if joint:
        B = rng.randn(D, D)
        Wj, tj = 0.1 * B @ B.T, 0.3 * rng.randn(D)
        terms.append(dict(kind=_lib.REWARD_EXP_SA, coef=-0.5, W=Wj, t=tj))
    m0 = rng.rand(Ds)
    if singular:
        v = rng.randn(Ds)
        S0 = 0.05 * np.outer(v, v)
    else:
        B = rng.randn(Ds, Ds)
        S0 = 0.02 * B @ B.T
    return dict(gp=gp, spec=spec, pol=pol, terms=terms, X=X, Y=Y, ell=ell, sf2=sf2, sn2=sn2, maxa=maxa, Wr=Wr, tr=tr,
                Wj=Wj, tj=tj, m0=m0, S0=S0, Ds=Ds, dims=dims, U=U, kind=kind, R=R)


def _oracle(P, r, H, params=None, m0=None, S0=None):
    """torch cascade of restart r; params: torch leaves of the policy (else built from P).  -> (trajectory means
    [H+1,Ds], covariances [H+1,Ds,Ds], total reward)"""
    if params is None:
        params = [T(P["pol"][k][r]) for k in (("W", "b") if P["kind"] == "linear" else ("X", "Y", "ell"))]
    terms = [dict(kind=_lib.REWARD_EXP, coef=1.0, W=P["Wr"], t=P["tr"])]
    if P["Wj"] is not None:
        terms.append(dict(kind=_lib.REWARD_EXP_SA, coef=-0.5, W=P["Wj"], t=P["tj"]))
    out = aro.problem_rollout(P["kind"], params, P["X"], P["Y"], P["ell"], P["sf2"], P["sn2"], P["maxa"], terms,
                              T(P["m0"])[None] if m0 is None else m0, T(P["S0"]) if S0 is None else S0, H,
                              angle_dims=P["dims"])
    return out["traj_m"], out["traj_S"], out["reward"]


SHAPES = [  # Ds, dims, U, policy, R, singular S0, joint term
    (4, [1], 1, "linear", 1, False, False),          # cart-pole-like
    (4, [1], 1, "rbf", 32, False, True),
    (4, [1], 1, "linear", 32, False, True),
    (6, [1, 2], 1, "rbf", 1, False, False),          # double pendulum
    (8, [0, 1, 2, 3, 4, 5, 6], 1, "linear", 2, False, False),   # Dh + U = 16
    (3, [2, 0, 1], 1, "rbf", 2, False, False),       # every dimension an angle
    (4, [3], 2, "linear", 2, True, False),           # singular S0
]


@pytest.mark.parametrize("Ds,dims,U,kind,R,singular,joint", SHAPES)
def test_forward_matches_oracle(Ds, dims, U, kind, R, singular, joint):
    from pilco_b200 import engine
    H = 6
    P = _problem(Ds, dims, U, kind, R, seed=Ds + 10 * U, singular=singular, joint=joint)
    plan = engine.RolloutPlan(P["gp"], P["spec"], P["terms"], P["m0"], P["S0"], H, R=R, angles=dims)
    tm, tS, rew = plan.forward()
    torch.cuda.synchronize()
    assert int(plan.info.max().item()) == 0
    for r in sorted({0, R - 1}):
        om, oS, tot = _oracle(P, r, H)
        assert scaled_err(tm[r].cpu().numpy(), om.numpy()) < 1e-9
        assert scaled_err(tS[r].cpu().numpy(), oS.numpy()) < 1e-9
        assert abs(float(rew[r]) - float(tot)) < 1e-9 * max(1.0, abs(float(tot)))


@pytest.mark.parametrize("kind", ["linear", "rbf"])
def test_periodicity(kind):
    """m0 + 2 pi e_a: the same rewards, and trajectory means that differ by 2 pi in dimension a only"""
    from pilco_b200 import engine
    H, dims = 6, [1, 3]
    P = _problem(5, dims, 1, kind, 2, seed=4)
    out = []
    for shift in (0.0, 2 * np.pi):
        m0 = P["m0"].copy()
        m0[3] += shift
        plan = engine.RolloutPlan(P["gp"], P["spec"], P["terms"], m0, P["S0"], H, R=2, angles=dims)
        tm, tS, rew = plan.forward()
        torch.cuda.synchronize()
        out.append((tm.cpu().numpy().copy(), tS.cpu().numpy().copy(), rew.cpu().numpy().copy(),
                    plan.step_reward.cpu().numpy().copy()))
    (m_a, S_a, r_a, sr_a), (m_b, S_b, r_b, sr_b) = out
    assert np.max(np.abs(r_a - r_b)) <= 1e-12 * np.max(np.abs(r_a))
    assert np.max(np.abs(sr_a - sr_b)) <= 1e-12 * np.max(np.abs(sr_a))
    d = m_b - m_a
    assert np.max(np.abs(d[..., 3] - 2 * np.pi)) <= 1e-12 * np.max(np.abs(m_b))
    assert np.max(np.abs(np.delete(d, 3, axis=-1))) <= 1e-12 * np.max(np.abs(m_a))
    assert scaled_err(S_b, S_a) < 1e-12


@pytest.mark.parametrize("Ds,dims,U,kind,R,singular,joint", SHAPES + [(4, [0, 2], 1, "rbf", 2, False, True)])
def test_backward_matches_autograd(Ds, dims, U, kind, R, singular, joint):
    """taped and recomputing reverse sweeps agree; policy gradient, gm0 and the (symmetric) gS0 against autograd"""
    from pilco_b200 import engine
    H = 5
    P = _problem(Ds, dims, U, kind, R, seed=Ds + 10 * U + 1, singular=singular, joint=joint)
    grads = {}
    for taped in (True, False):
        plan = engine.RolloutPlan(P["gp"], P["spec"], P["terms"], P["m0"], P["S0"], H, R=R, grad=taped, angles=dims)
        assert (plan.tape is not None) == taped
        plan.forward()
        g = plan.backward()
        torch.cuda.synchronize()
        assert int(plan.info.max().item()) == 0
        grads[taped] = {k: v.cpu().numpy().copy() for k, v in g.items()}
    for k in grads[True]:
        assert scaled_err(grads[False][k], grads[True][k]) < 1e-12, k
    assert np.array_equal(grads[True]["S0"], np.swapaxes(grads[True]["S0"], 1, 2))
    names = ("W", "b") if kind == "linear" else ("X", "Y", "ell")
    for r in sorted({0, R - 1}):
        params = [T(P["pol"][k][r]).requires_grad_() for k in names]
        m0, S0 = T(P["m0"])[None].requires_grad_(), T(P["S0"]).requires_grad_()
        _, _, tot = _oracle(P, r, H, params=params, m0=m0, S0=S0)
        ref = torch.autograd.grad(tot, params + [m0, S0])
        for k, rg in zip(names + ("m0", "S0"), ref):
            rg = rg.numpy()
            if k == "S0":
                rg = 0.5 * (rg + rg.T)
            got = grads[True][k][r]
            assert scaled_err(got, rg.reshape(got.shape)) < 1e-8, (k, r)


def test_backward_matches_central_differences():
    """d reward / d W by central differences of the device forward itself (linear policy)"""
    from pilco_b200 import engine
    H, dims = 5, [1]
    P = _problem(3, dims, 1, "linear", 1, seed=33)
    plan = engine.RolloutPlan(P["gp"], P["spec"], P["terms"], P["m0"], P["S0"], H, R=1, grad=True, angles=dims)
    plan.forward()
    g = plan.backward()["W"][0].cpu().numpy().copy()
    h = 1e-6
    W = P["spec"]["W"]
    for (u, k) in [(0, 0), (0, 2), (0, 3)]:
        vals = []
        for sgn in (1, -1):
            W2 = W.copy()
            W2[0, u, k] += sgn * h
            spec = dict(P["spec"], W=W2)
            p2 = engine.RolloutPlan(P["gp"], spec, P["terms"], P["m0"], P["S0"], H, R=1, angles=dims)
            vals.append(float(p2.forward()[2][0]))
        fd = (vals[0] - vals[1]) / (2 * h)
        assert abs(fd - g[u, k]) < 1e-6 * max(1.0, np.max(np.abs(g))), (u, k, fd, g[u, k])


def test_graph_replay_matches_eager():
    from pilco_b200 import engine
    H, dims = 5, [1]
    P = _problem(4, dims, 1, "rbf", 4, seed=5, joint=True)
    plan = engine.RolloutPlan(P["gp"], P["spec"], P["terms"], P["m0"], P["S0"], H, R=4, grad=True, angles=dims)
    plan.forward()
    g = plan.backward()
    torch.cuda.synchronize()
    eager = [plan.reward.cpu().numpy().copy(), plan.traj_S.cpu().numpy().copy()] + [g[k].cpu().numpy().copy() for k in g]
    plan.capture(backward=True)
    plan.replay()
    torch.cuda.synchronize()
    again = [plan.reward.cpu().numpy(), plan.traj_S.cpu().numpy()] + [plan.gbuf[k].cpu().numpy() for k in plan.gbuf]
    for a, b in zip(eager, again):
        assert np.array_equal(a, b)


def test_no_angles_forwards_to_the_plain_rollout():
    """angles=[] is the rollout without angles, bit for bit"""
    from pilco_b200 import engine, _lib
    import ctypes as C
    P = _problem(4, [], 1, "linear", 2, seed=8)
    a = engine.RolloutPlan(P["gp"], P["spec"], P["terms"], P["m0"], P["S0"], 5, R=2)
    ra = a.forward()[2].cpu().numpy().copy()
    empty = _lib.Angles()
    rc = _lib.lib.pilco_rollout_angles_forward(C.byref(a.ro), C.byref(empty), engine.stream_ptr())
    assert rc == 0
    torch.cuda.synchronize()
    assert np.array_equal(a.reward.cpu().numpy(), ra)
