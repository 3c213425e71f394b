"""CPU tests of the score-function gradient of the particle return (pilco_particles_rollout_score_grad,
engine.ParticlePlan(estimator="score"), PILCO.sample_policy_gradient(estimator="score")): the torch oracle
(tests/particle_grad_oracle.py) against the moment-matching gradient where moment matching is exact and against the
pathwise oracle, the workspace size, argument validation of the C entry point (rejecting calls only, with the status
codes of pilco_particles_rollout_batch_grad), the SASS of the new kernels, and the rejected estimator arguments."""
import ctypes as C
import os
import re

import numpy as np
import pytest
import torch

from pilco_b200 import _lib, engine
from pilco_b200._lib import lib
from abi_fakes import ERR_DIM, ERR_WS, PT_MAX_P, _batched, _grad, _particles, _score_grad_cases
from particle_cases import _problem
from particle_oracle import particle_rollout
from particle_grad_oracle import score_grad, value_and_grad
from util import CUOBJDUMP, sass_named

F64 = torch.float64


def _linear_case(seed):
    """linear unsquashed policy, one linear reward, H = 2: E[return] = w'm0 + w'(m0 + E[mu(x~_0)]), which moment
    matching gets exactly"""
    dyn, rng = _problem(seed)
    W, b = 0.6 * rng.randn(1, 3), 0.2 * rng.randn(1)
    pol = dict(kind=_lib.POLICY_LINEAR, squash=False, maxa=np.ones(1), W=W, b=b)
    terms = [dict(kind=_lib.REWARD_LINEAR, coef=1.0, W=rng.randn(3), t=None)]
    m0, S0 = 0.5 + 0.1 * rng.randn(3), 0.04 * np.eye(3)
    return dyn, pol, terms, m0, S0


def _mm_grad(dyn, pol, terms, m0, S0):
    """d/d(W, b) of w' E[mu(x~_0)] for x~_0 = [x0, W x0 + b], x0 ~ N(m0, S0): the expectation of the SE posterior mean
    under a Gaussian input in closed form (PILCO's mean prediction), through torch autograd"""
    t = lambda a: torch.as_tensor(np.asarray(a, dtype=np.float64))
    W, b = t(pol["W"]).clone().requires_grad_(), t(pol["b"]).clone().requires_grad_()
    m0_, S0_ = t(m0), t(S0)
    Ds = m0_.shape[0]
    F = torch.cat([torch.eye(Ds, dtype=F64), W], 0)
    m, S = torch.cat([m0_, W @ m0_ + b]), F @ S0_ @ F.T
    C_, ell, sf2, beta, wr = t(dyn["C"]), t(dyn["ell"]), t(dyn["sf2"]), t(dyn["beta"]), t(terms[0]["W"])
    tot = torch.zeros((), dtype=F64)
    for e in range(ell.shape[0]):
        lam = torch.diag(ell[e] ** 2)
        d = C_ - m[None]
        q = sf2[e] / torch.sqrt(torch.det(S @ torch.linalg.inv(lam) + torch.eye(S.shape[0], dtype=F64))) \
            * torch.exp(-0.5 * (d @ torch.linalg.inv(S + lam) * d).sum(1))
        tot = tot + wr[e] * (q @ beta[e])
    gW, gb = torch.autograd.grad(tot, [W, b])
    return {"W": gW.numpy(), "b": gb.numpy()}


def _draws(dyn, pol, terms, m0, S0, P, K, baseline):
    """K independent score-oracle estimates (and pathwise-oracle estimates) over P particles each"""
    score, path = {"W": [], "b": []}, {"W": [], "b": []}
    F = np.linalg.cholesky(S0)
    for k in range(K):
        rng = np.random.RandomState(1000 + k)
        x0, eps = m0[None] + rng.randn(P, 3) @ F.T, rng.randn(P, 2, 3)
        traj = particle_rollout(dyn, pol, terms, x0, eps)[0]
        g = score_grad(dyn, pol, terms, traj, eps, baseline=baseline)
        gp = value_and_grad(dyn, pol, terms, x0, eps)[1]
        for key in score:
            score[key].append(g[key])
            path[key].append(gp[key])
    return {k: np.stack(v) for k, v in score.items()}, {k: np.stack(v) for k, v in path.items()}


def test_score_oracle_mean_is_the_moment_matching_gradient():
    dyn, pol, terms, m0, S0 = _linear_case(41)
    ref = _mm_grad(dyn, pol, terms, m0, S0)
    score, _ = _draws(dyn, pol, terms, m0, S0, 4000, 24, baseline=False)
    worst = 0.0
    for k, r in ref.items():
        a = score[k]
        worst = max(worst, float(np.max(np.abs(a.mean(0) - r) / (a.std(0, ddof=1) / np.sqrt(a.shape[0])))))
    print("score oracle (no baseline, 24 x 4000 particles) vs moment matching: worst %.2f standard errors" % worst)
    assert worst <= 5.0


def test_score_oracle_with_baseline_agrees_with_pathwise_oracle():
    dyn, pol, terms, m0, S0 = _linear_case(42)
    score, path = _draws(dyn, pol, terms, m0, S0, 4000, 24, baseline=True)
    worst = 0.0
    for k in score:
        d = score[k] - path[k]                                  # paired: the same particles
        worst = max(worst, float(np.max(np.abs(d.mean(0)) / (d.std(0, ddof=1) / np.sqrt(d.shape[0])))))
    print("score oracle (leave-one-out baseline) vs pathwise oracle, paired over 24 x 4000 particles: "
          "worst %.2f standard errors" % worst)
    assert worst <= 5.0


def _layout_bytes(P, H, Ds, U, D, n, bf, R):
    """x~ [H,T,D], mean [T,Ds], var [H,T,Ds], G [H-1,T], the sums [R,H], gmean and gvar [H-1,T,Ds], the VJP output
    [H-1,T,D], z_bar [T,H,U], the RBF sums [R,U,bf,Ds] x 2 and [R,U,bf] x 2, then one predict / VJP workspace for the
    predict at T = R P and the VJP of the largest group of whole steps (at most 65535 * 32 rows)"""
    T, Hm = R * P, max(H - 1, 0)
    even = lambda k: (k + 1) & ~1
    doubles = sum(even(k) for k in (H * T * D, T * Ds, H * T * Ds, Hm * T, R * H, Hm * T * Ds, Hm * T * Ds, Hm * T * D,
                                    T * H * U, R * U * bf * Ds, R * U * bf * Ds, R * U * bf, R * U * bf))
    grp = max(min(Hm, PT_MAX_P // T), 1)
    pred = lib.pilco_gp_predict_workspace_bytes(n, D, Ds, T, 0)
    vjp = lib.pilco_gp_predict_vjp_workspace_bytes(n, D, Ds, grp * T)
    return 8 * doubles + max(pred, vjp)


def _ws(pr, R):
    return lib.pilco_particles_score_grad_workspace_bytes(C.byref(pr) if pr is not None else None, R)


def test_score_grad_workspace_bytes():
    assert _ws(None, 1) == 0
    for R in (0, -2, 65536):
        assert _ws(_batched(), R) == 0, R
    assert _ws(_batched(P=1000), PT_MAX_P // 1000 + 1) == 0
    for P, H in ((0, 5), (PT_MAX_P + 1, 5), (10, -1)):
        assert _ws(_batched(P=P, H=H), 1) == 0, (P, H)
    assert _ws(_particles(P=PT_MAX_P, H=(1 << 31) - 1), 1) == 0            # past 2^31 - 1 per-(step, particle) CTAs
    for kind, bf in ((_lib.POLICY_LINEAR, 0), (_lib.POLICY_RBF, 20)):
        for H in (0, 1, 2, 5):
            pr = _batched(kind, P=1000, H=H)
            prev = 0
            for R in (1, 2, 7, 32):
                assert _ws(pr, R) == _layout_bytes(1000, H, 3, 1, 4, 50, bf, R), (kind, H, R)
                assert _ws(pr, R) > prev
                prev = _ws(pr, R)
        assert _ws(pr, 1) > lib.pilco_particles_grad_workspace_bytes(C.byref(_particles(kind, P=1000, H=5)))
    # steps grouped under the VJP's row limit: 60000 rows per step, 34 steps per call
    pr = _particles(P=60000, H=40)
    assert _ws(pr, 1) == _layout_bytes(60000, 40, 3, 1, 4, 50, 0, 1)
    assert _ws(_batched(P=4096, H=40), 500) < 8 * 500 * 4096 * (40 * (4 + 3 + 3 + 3 + 1 + 1 + 4) + 64)


def _run(pr, R, g):
    return lib.pilco_particles_rollout_score_grad(C.byref(pr) if pr is not None else None, R,
                                                  C.byref(g) if g is not None else None, None)


def _batch_run(pr, R, g):
    return lib.pilco_particles_rollout_batch_grad(C.byref(pr) if pr is not None else None, R,
                                                  C.byref(g) if g is not None else None, None)


def test_score_grad_argument_validation():
    for i, (pr, R, g, want) in enumerate(_score_grad_cases()):
        assert _run(pr, R, g) == want, i
        assert _batch_run(pr, R, g) == want, i                             # the batched pathwise entry point's codes
    for kind in (_lib.POLICY_LINEAR, _lib.POLICY_RBF):                      # a workspace short of the score layout's
        pr = _batched(kind)
        need = _ws(pr, 3)
        g = _grad(); g.ws_bytes = need - 8
        assert need > 0 and _run(pr, 3, g) == ERR_WS
    pr = _particles(P=PT_MAX_P, H=(1 << 31) - 1)
    g = _grad(); g.ws_bytes = (1 << 64) - 1
    assert _run(pr, 1, g) == ERR_DIM


@pytest.mark.skipif(not os.path.exists(CUOBJDUMP), reason="cuobjdump not available")
def test_score_kernels_sass():
    names = ["ps_togo_kernel", "ps_base_kernel", "ps_cot_kernel", "ps_zbar_kernel"]
    sass = sass_named(names)
    assert set(sass) == set(names)
    for k, text in sass.items():                                # no spills, no local memory (MAXD = 16 registers)
        assert not re.search(r"\b(STL|LDL)\b", text), k
    assert "BAR" in sass["ps_base_kernel"]


def test_estimator_arguments_are_rejected_before_any_allocation(monkeypatch):
    from pilco.models import PILCO
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)
    with pytest.raises(ValueError, match="consistent"):
        engine.ParticlePlan(None, None, None, 10, 3, grad=True, consistent=True, estimator="score")
    with pytest.raises(ValueError, match="consistent"):
        engine.ParticlePlan(None, None, None, 10, 3, consistent=True, estimator="score")
    for bad in ("reinforce", None, "Score"):
        with pytest.raises(ValueError, match="estimator"):
            engine.ParticlePlan(None, None, None, 10, 3, grad=True, estimator=bad)
    X = np.random.RandomState(0).rand(20, 3); Y = 0.1 * X[:, :2]
    pilco = PILCO((X, Y))
    with pytest.raises(ValueError, match="consistent"):
        pilco.sample_policy_gradient(X[0, :2], 0.1 * np.eye(2), 3, num_samples=10, seed=0, consistent=True,
                                     estimator="score")
    with pytest.raises(ValueError, match="estimator"):
        pilco.sample_policy_gradient(X[0, :2], 0.1 * np.eye(2), 3, num_samples=10, seed=0, estimator="lr")
    with pytest.raises(RuntimeError, match="CUDA device"):                  # a valid call needs the GPU
        pilco.sample_policy_gradient(X[0, :2], 0.1 * np.eye(2), 3, num_samples=10, seed=0, estimator="score")
