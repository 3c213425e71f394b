"""Reward terms on the joint state-action Gaussian (PILCO_REWARD_EXP_SA / PILCO_REWARD_LINEAR_SA, DESIGN.md section 18),
checked WITHOUT a GPU: the header and ctypes constants with unchanged struct layouts, argument validation of the C ABI,
the moment-matching and particle oracles against Monte Carlo, central differences and the state-term identity, the
Python classes, and the SASS of the kernels the feature added or touched."""
import ctypes as C
import os
import re

import numpy as np
import pytest
import torch

from pilco_b200 import _lib, rewards
from pilco_b200._lib import lib
import action_reward_oracle as aro
import particle_oracle as po
from abi_fakes import ERR_NULL, ERR_UNSUP, ERR_WS, FAKE, _particles, _rollout
from particle_grad_oracle import T, score_grad, value_and_grad
from util import CUOBJDUMP, ROOT, make_gp_problem, sass


def test_header_constants_and_unchanged_layouts():
    hdr = open(os.path.join(ROOT, "include", "pilco_b200.h")).read()
    for name, val in (("PILCO_REWARD_EXP", 0), ("PILCO_REWARD_LINEAR", 1), ("PILCO_REWARD_BOX", 2),
                      ("PILCO_REWARD_EXP_SA", 3), ("PILCO_REWARD_LINEAR_SA", 4)):
        assert re.search(r"#define\s+%s\s+%d\b" % (name, val), hdr), name
    assert (_lib.REWARD_EXP_SA, _lib.REWARD_LINEAR_SA) == (3, 4)
    # new kinds only: no struct grew (the sizes the ABI has had since version 3)
    assert (C.sizeof(_lib.RewardTerm), C.sizeof(_lib.Rollout), C.sizeof(_lib.Particles)) == (32, 640, 600)
    assert lib.pilco_version() == _lib.ABI_VERSION


def test_rollout_validation_of_joint_kinds():
    fwd = lambda ro: lib.pilco_rollout_forward(C.byref(ro), None)
    for kind in (_lib.REWARD_EXP_SA, _lib.REWARD_LINEAR_SA):
        for ch in (_lib.CHANNEL_ADD, _lib.CHANNEL_MULT):
            assert fwd(_rollout(reward_kind=kind, channel=ch)) == ERR_WS       # accepted: reaches the size check
    assert fwd(_rollout(reward_kind=5)) == ERR_UNSUP
    ro = _rollout(reward_kind=_lib.REWARD_EXP_SA); ro.rewards[0].t = None
    assert fwd(ro) == ERR_NULL
    ro = _rollout(reward_kind=_lib.REWARD_LINEAR_SA); ro.rewards[0].t = None     # the linear kind has no target
    assert fwd(ro) == ERR_WS
    ro = _rollout(reward_kind=_lib.REWARD_LINEAR_SA); ro.rewards[0].W = None
    assert fwd(ro) == ERR_NULL
    # the backward workspace grows only when a joint term is present: [H,2,R,D] + [H,2,R,D,D] doubles
    base = lib.pilco_rollout_bwd_workspace_bytes(C.byref(_rollout()))
    assert lib.pilco_rollout_bwd_workspace_bytes(C.byref(_rollout(reward_kind=_lib.REWARD_LINEAR))) == base
    R, H, D = 2, 5, 4
    assert lib.pilco_rollout_bwd_workspace_bytes(C.byref(_rollout(reward_kind=_lib.REWARD_EXP_SA))) \
        == base + 8 * H * 2 * R * (D + D * D)
    assert lib.pilco_rollout_workspace_bytes(C.byref(_rollout(reward_kind=_lib.REWARD_EXP_SA))) \
        == lib.pilco_rollout_workspace_bytes(C.byref(_rollout()))


def test_particles_validation_of_joint_kinds():
    run = lambda pr: lib.pilco_particles_rollout(C.byref(pr), None)
    ok = run(_particles())                                                       # a valid description's status
    for kind in (_lib.REWARD_EXP_SA, _lib.REWARD_LINEAR_SA):
        assert run(_particles(reward_kind=kind)) == ok
        assert run(_particles(reward_kind=kind, channel=_lib.CHANNEL_MULT)) == ok
    assert run(_particles(reward_kind=5)) == ERR_UNSUP
    pr = _particles(reward_kind=_lib.REWARD_EXP_SA); pr.rewards[0].t = None
    assert run(pr) == ERR_NULL
    # the score gradient keeps x~_bar of one more step for the joint terms' direct term; the others are unchanged
    a, b = _particles(), _particles(reward_kind=_lib.REWARD_EXP_SA)
    for f in (lib.pilco_particles_workspace_bytes, lib.pilco_particles_grad_workspace_bytes):
        assert f(C.byref(a)) == f(C.byref(b)) > 0
    sa, sb = (lib.pilco_particles_score_grad_workspace_bytes(C.byref(p), 2) for p in (a, b))
    assert sb == sa + 8 * 2 * a.P * a.dyn.D


def _mc(term, m, s, n=400000, seed=0):
    z = np.random.RandomState(seed).multivariate_normal(m.reshape(-1), s, size=n)
    v = po.point_value(term, z[:, :2], z[:, 2:])
    return v.mean(), v.std() / np.sqrt(n)


def test_joint_closed_form_against_monte_carlo():
    rng = np.random.RandomState(1)
    A = rng.randn(3, 3)
    m, s = rng.rand(1, 3), 0.3 * A @ A.T + 0.05 * np.eye(3)
    B = rng.randn(3, 3)
    for term in (dict(kind=_lib.REWARD_EXP_SA, W=B @ B.T + 0.2 * np.eye(3), t=rng.rand(3)),
                 dict(kind=_lib.REWARD_LINEAR_SA, W=rng.randn(3), t=None)):
        closed = float(aro.term_moment(term, T(m), T(s)))
        mean, se = _mc(term, m, s)
        assert abs(closed - mean) < 5 * se, (term["kind"], closed, mean, se)
    # the class evaluates the same closed form on joint moments, on the host for the linear one
    lin = rewards.LinearStateActionReward(2, 1, [1.0, -2.0, 0.5])
    mu, var = lin.compute_reward(m, s)
    w = np.array([1.0, -2.0, 0.5])
    assert np.allclose(mu, m @ w) and np.allclose(var, w @ s @ w) and mu.shape == var.shape == (1, 1)


def _small_problem(seed=3):
    Ds, U, n = 2, 1, 25
    X, Y, ell, sf2, sn2 = make_gp_problem(n, Ds + U, Ds, seed=seed)
    rng = np.random.RandomState(seed)
    B = rng.randn(3, 3)
    terms = [dict(kind=_lib.REWARD_EXP, coef=1.0, W=np.eye(Ds), t=0.2 * np.ones(Ds)),
             dict(kind=_lib.REWARD_EXP_SA, coef=-0.4, W=B @ B.T, t=0.1 * rng.rand(3)),
             dict(kind=_lib.REWARD_LINEAR_SA, coef=0.2, W=rng.randn(3), t=None),
             dict(kind=_lib.REWARD_EXP_SA, coef=0.1, channel=_lib.CHANNEL_MULT, W=np.diag([0.0, 0.0, 2.0]), t=np.zeros(3))]
    return dict(X=X, Y=0.1 * Y, ell=ell, sf2=sf2, sn2=sn2, maxa=np.array([1.2]), m0=X[0, :Ds], S0=0.05 * np.eye(Ds),
                W=0.5 * rng.randn(U, Ds), b=0.1 * rng.randn(U)), terms


def _mm_value(P, terms, W, b, H=3, mu=1.5):
    return aro.problem_rollout("linear", (W, b), P["X"], P["Y"], P["ell"], P["sf2"], P["sn2"], P["maxa"], terms,
                               P["m0"], P["S0"], H, mult_mu=mu)


def test_moment_oracle_gradient_against_central_differences():
    P, terms = _small_problem()
    W, b = T(P["W"]).requires_grad_(), T(P["b"]).requires_grad_()
    gW, gb = torch.autograd.grad(_mm_value(P, terms, W, b)["reward"], [W, b])
    h = 1e-6
    for (i, j) in ((0, 0), (0, 1)):
        d = np.zeros_like(P["W"]); d[i, j] = h
        fd = (float(_mm_value(P, terms, T(P["W"] + d), T(P["b"]))["reward"])
              - float(_mm_value(P, terms, T(P["W"] - d), T(P["b"]))["reward"])) / (2 * h)
        assert abs(fd - float(gW[i, j])) <= 1e-6 * max(1.0, abs(fd))
    fd = (float(_mm_value(P, terms, T(P["W"]), T(P["b"] + h))["reward"])
          - float(_mm_value(P, terms, T(P["W"]), T(P["b"] - h))["reward"])) / (2 * h)
    assert abs(fd - float(gb[0])) <= 1e-6 * max(1.0, abs(fd))
    # an action cost must pull on the policy: the joint terms' share of the gradient is not zero
    g0 = torch.autograd.grad(_mm_value(P, terms[:1], W, b)["reward"], [W])[0]
    assert float((gW - g0).abs().max()) > 1e-3


def test_zero_action_block_is_the_state_term():
    P, _ = _small_problem()
    rng = np.random.RandomState(5)
    B = rng.randn(2, 2)
    Ws, ts, wl = B @ B.T, rng.rand(2), rng.randn(2)
    Wj = np.zeros((3, 3)); Wj[:2, :2] = Ws
    state = [dict(kind=_lib.REWARD_EXP, coef=0.7, W=Ws, t=ts), dict(kind=_lib.REWARD_LINEAR, coef=0.3, W=wl, t=None)]
    joint = [dict(kind=_lib.REWARD_EXP_SA, coef=0.7, W=Wj, t=np.append(ts, 0.9)),
             dict(kind=_lib.REWARD_LINEAR_SA, coef=0.3, W=np.append(wl, 0.0), t=None)]
    a, b = (_mm_value(P, t, T(P["W"]), T(P["b"])) for t in (state, joint))
    assert torch.allclose(a["step_reward"], b["step_reward"], rtol=1e-12, atol=0)
    x, u = rng.rand(7, 2), rng.randn(7, 1)
    for s, j in zip(state, joint):
        assert np.allclose(po.point_value(s, x, u), po.point_value(j, x, u), rtol=1e-14, atol=0)


def test_particle_oracles_agree_and_score_direct_term():
    """numpy rollout = torch rollout's value; the pathwise autograd gradient against central differences; the score
    oracle's direct term alone is the gradient of the joint terms at fixed states (linear term: closed form)"""
    P, terms = _small_problem(7)
    from oracle import python_port as pp
    iK, beta = pp.calculate_factorizations(P["X"], P["Y"], P["ell"], P["sf2"], P["sn2"])
    dyn = dict(C=P["X"], ell=P["ell"], sf2=P["sf2"], iK=iK, beta=beta)
    pol = dict(kind=_lib.POLICY_LINEAR, squash=True, maxa=P["maxa"], W=P["W"], b=P["b"])
    rng = np.random.RandomState(8)
    x0, eps = P["m0"][None] + 0.2 * rng.randn(40, 2), rng.randn(40, 4, 2)
    ret = po.particle_rollout(dyn, pol, terms, x0, eps, mult_mu=1.5)[4]
    v, g = value_and_grad(dyn, pol, terms, x0, eps, mult_mu=1.5)
    assert abs(v - ret.mean()) <= 1e-13 * max(1.0, abs(v))
    h = 1e-6
    d = np.zeros_like(P["W"]); d[0, 1] = h
    vp = po.particle_rollout(dyn, dict(pol, W=P["W"] + d), terms, x0, eps, mult_mu=1.5)[4].mean()
    vm = po.particle_rollout(dyn, dict(pol, W=P["W"] - d), terms, x0, eps, mult_mu=1.5)[4].mean()
    assert abs((vp - vm) / (2 * h) - g["W"][0, 1]) <= 1e-6 * max(1.0, abs(g["W"][0, 1]))
    # direct term of a lone linear action term, unsquashed policy: d/db mean_p sum_t c w_u = c w_u H
    traj = po.particle_rollout(dyn, dict(pol, squash=False), terms, x0, eps)[0]
    lone = [dict(kind=_lib.REWARD_LINEAR_SA, coef=0.3, W=np.array([0.0, 0.0, 2.0]), t=None)]
    nosq = dict(pol, squash=False)
    gd = score_grad(dyn, nosq, lone, traj, eps, transitions=False)
    assert abs(gd["b"][0] - 0.3 * 2.0 * 4) <= 1e-12
    assert np.allclose(gd["W"][0], 0.6 * traj[:, :4].sum(1).mean(0), rtol=1e-12)
    assert not any(np.any(v) for v in score_grad(dyn, nosq, lone, traj, eps, direct=False, transitions=False).values())


def test_reward_classes_and_term_specs():
    Ds, U = 3, 2
    e = rewards.ExponentialStateActionReward(Ds, U)
    assert np.array_equal(e.W.numpy(), np.eye(5)) and np.array_equal(e.t.numpy(), np.zeros((1, 5)))
    (t,) = e.terms(0.5, _lib.CHANNEL_MULT)
    assert (t["kind"], t["coef"], t["channel"], t["W"].shape, t["t"].shape) == (_lib.REWARD_EXP_SA, 0.5, 1, (5, 5), (5,))
    (t,) = rewards.LinearStateActionReward(Ds, U, np.arange(5.0)).terms()
    assert t["kind"] == _lib.REWARD_LINEAR_SA and t["W"].shape == (5,) and t["t"] is None
    Q = np.array([[2.0, 0.1], [0.1, 1.0]])
    c = rewards.action_cost(Ds, U, Q)
    assert isinstance(c, rewards.ExponentialStateActionReward)
    W = c.W.numpy()
    assert np.array_equal(W[Ds:, Ds:], Q) and not W[:Ds].any() and not W[:, :Ds].any() and not c.t.numpy().any()
    comb = rewards.CombinedRewards(Ds, [rewards.ExponentialReward(Ds), c], coefs=[1.0, 0.1])
    assert [x["kind"] for x in comb.terms()] == [_lib.REWARD_EXP, _lib.REWARD_EXP_SA]
    assert [x["coef"] for x in comb.terms()] == [1.0, 0.1]
    # a reward on the action cannot be evaluated on state moments alone
    with pytest.raises(ValueError, match="joint moments"):
        rewards.CombinedRewards(Ds, [c, rewards.ExponentialReward(Ds)]).compute_reward(np.zeros((1, Ds)), np.eye(Ds))
    with pytest.raises(ValueError, match="joint moments"):
        rewards.LinearStateActionReward(Ds, U, np.ones(5)).compute_reward(np.zeros((1, Ds)), np.eye(Ds))
    import pilco.rewards as alias
    for name in ("ExponentialStateActionReward", "LinearStateActionReward", "action_cost"):
        assert getattr(alias, name) is getattr(rewards, name)
    c.W.assign(2.0 * W)
    assert np.array_equal(c.terms()[0]["W"], 2.0 * W)


def test_reward_key_follows_joint_parameters():
    from pilco.models import PILCO
    rng = np.random.RandomState(0)
    X = rng.rand(20, 3)
    c = rewards.action_cost(2, 1, [[1.0]])
    p = PILCO((X, 0.1 * rng.rand(20, 2)), reward=rewards.CombinedRewards(2, [rewards.ExponentialReward(2), c], [1.0, 0.2]))
    k0 = p._reward_key()
    assert p._reward_key() == k0
    c.W.assign(3.0 * c.W.numpy())
    k1 = p._reward_key()
    c.t.assign(0.1 * np.ones((1, 3)))
    assert len({k0, k1, p._reward_key()}) == 3


@pytest.mark.skipif(not os.path.exists(CUOBJDUMP), reason="cuobjdump not available")
def test_sass_of_joint_reward_kernels():
    """The joint terms' particle kernels keep everything in registers, and so do the state kernels they run beside
    (which the joint terms did not enter).  The moment-matching state reward kernels hold the box risk's per-dimension
    derivative arrays in local memory, as before; of the joint terms' own kernels only rb_reward_joint_kernel touches
    local memory: three registers saved around the LU solve, as rb_reward_kernel saves two."""
    local = lambda text: len(re.findall(r"\b(?:STL|LDL)\b", text))
    for pat in ("pt_joint_kernel", "pj_grad_kernel", "ps_zbar_kernel", "pt_step_kernel", "pg_step_kernel"):
        fn = sass(pat)
        assert len(fn) == 1, pat
        assert all(local(t) == 0 for t in fn.values()), pat
    for pat, bound in (("ro_reward_kernel", 24), ("rb_reward_kernel", 64), ("rb_post_kernel", 8),
                       ("ro_reward_joint_kernel", 0), ("rb_reward_joint_kernel", 16)):
        fn = sass(pat)
        assert len(fn) == 1 and all(local(t) <= bound for t in fn.values()), (pat, [local(t) for t in fn.values()])
    for text in sass("pt_joint_kernel|pj_grad_kernel").values():
        assert "DFMA" in text
