"""CPU tests of the consistent particle sampler (pilco_particles_rollout_consistent, engine.particles_rollout(...,
consistent=True), PILCO.sample_trajectories(..., consistent=True)): argument validation of the C entry point (rejecting
calls only), the exact workspace layout with its 0 for unsupported sizes and size_t overflow, the SASS of the new
kernels, the failure without a GPU, and the numpy oracle (tests/particle_oracle.py) against a joint draw."""
import ctypes as C
import os
import re

import numpy as np
import pytest
import torch

from pilco_b200 import _lib
from pilco_b200._lib import lib
from abi_fakes import ERR_ALIGN, ERR_DIM, ERR_NULL, ERR_UNSUP, ERR_WS, FAKE, PT_MAX_P, _particles
from particle_cases import _problem
from particle_oracle import FunctionSample, consistent_rollout, joint_draw, particle_rollout
from util import CUOBJDUMP, sass_named


def _run(pr):
    return lib.pilco_particles_rollout_consistent(C.byref(pr) if pr is not None else None, None)


def _ws(pr):
    return lib.pilco_particles_consistent_workspace_bytes(C.byref(pr) if pr is not None else None)


def test_consistent_argument_validation():
    assert _run(None) == ERR_NULL
    assert _run(_particles()) == ERR_WS                                     # valid description, no workspace
    for kind in (_lib.POLICY_LINEAR, _lib.POLICY_RBF):
        for rk in (_lib.REWARD_EXP, _lib.REWARD_LINEAR, _lib.REWARD_BOX):
            for ch in (_lib.CHANNEL_ADD, _lib.CHANNEL_MULT):
                assert _run(_particles(kind, rk, ch)) == ERR_WS, (kind, rk, ch)
    assert _run(_particles(H=0)) == ERR_WS
    for P, H in ((0, 5), (PT_MAX_P + 1, 5), (10, -1)):
        assert _run(_particles(P=P, H=H)) == ERR_DIM, (P, H)
    for field in ("x0", "eps", "traj", "act", "step_reward", "step_risk", "ret", "ws"):
        pr = _particles(); setattr(pr, field, None)
        assert _run(pr) == ERR_NULL, field
    pr = _particles(); pr.dyn.beta = None
    assert _run(pr) == ERR_NULL
    pr = _particles(); pr.pol.max_action = None
    assert _run(pr) == ERR_NULL
    pr = _particles(); pr.rewards[0].t = None
    assert _run(pr) == ERR_NULL
    for field, value in (("mode", 1), ("iK", None), ("X_bs", 200)):
        pr = _particles(); setattr(pr.dyn, field, value)
        assert _run(pr) == ERR_UNSUP, field
    pr = _particles(); pr.pol.W_bs = 3                                      # batched policies: the gradient path only
    assert _run(pr) == ERR_UNSUP
    pr = _particles(_lib.POLICY_RBF); pr.pol.rbf.beta_bs = 20
    assert _run(pr) == ERR_UNSUP
    pr = _particles(_lib.POLICY_RBF); pr.pol.rbf.mode = 0
    assert _run(pr) == ERR_UNSUP
    assert _run(_particles(kind=7)) == ERR_UNSUP
    assert _run(_particles(reward_kind=9)) == ERR_UNSUP
    assert _run(_particles(channel=5)) == ERR_UNSUP
    pr = _particles(); pr.pol.U = 2
    assert _run(pr) == ERR_DIM
    pr = _particles(); pr.dyn.E = 4
    assert _run(pr) == ERR_DIM
    pr = _particles(); pr.dyn.ldk = 32
    assert _run(pr) == ERR_DIM
    for nr in (0, 9):
        pr = _particles(); pr.n_rewards = nr
        assert _run(pr) == ERR_DIM
    pr = _particles(); pr.dyn.iK = FAKE + 8
    assert _run(pr) == ERR_ALIGN
    pr = _particles(); pr.dyn.ldk = 65
    assert _run(pr) == ERR_ALIGN
    pr = _particles(); pr.ws = FAKE + 8; pr.ws_bytes = 1 << 40
    assert _run(pr) == ERR_ALIGN
    pr = _particles(P=PT_MAX_P, H=(1 << 31) - 1); pr.ws_bytes = (1 << 64) - 1  # the workspace size overflows size_t
    assert _run(pr) == ERR_DIM
    for H in (0, 1, 5):
        pr = _particles(H=H)
        need = _ws(pr)
        pr.ws_bytes = need - 8
        assert need > 0 and _run(pr) == ERR_WS, H
        assert need == lib.pilco_particles_consistent_workspace_bytes(C.byref(pr))


def _layout_bytes(P, H, Ds, D, n):
    """x~ of every step [H,P,D]; mu, var, the step closure's mean and var [P,Ds]; W_t [E,P,np]; the K* history
    [H,E,P,np]; the packed factor rows [H(H+1)/2,E,P]; then pilco_gp_predict's workspace at T = P"""
    even = lambda k: (k + 1) & ~1
    np_ = lib.pilco_pad_n(n)
    doubles = sum(even(k) for k in (H * P * D, P * Ds, P * Ds, P * Ds, P * Ds, Ds * P * np_, H * Ds * P * np_,
                                    H * (H + 1) // 2 * Ds * P))
    return 8 * doubles + lib.pilco_gp_predict_workspace_bytes(n, D, Ds, P, 0)


def test_consistent_workspace_bytes():
    assert _ws(None) == 0
    for P, H in ((0, 5), (PT_MAX_P + 1, 5), (10, -1)):
        assert _ws(_particles(P=P, H=H)) == 0, (P, H)
    pr = _particles(); pr.dyn.D = 17; pr.pol.U = 14
    assert _ws(pr) == 0
    for P, H in ((1, 0), (1000, 5), (777, 1), (4096, 40), (PT_MAX_P, 3)):
        assert _ws(_particles(P=P, H=H)) == _layout_bytes(P, H, 3, 4, 50), (P, H)
    # the metric shape (n = 300, D = 12, E = 10, P = 4096, H = 40): the K* history alone is 4.2 GB
    pr = _particles(P=4096, H=40)
    pr.dyn.n, pr.dyn.D, pr.dyn.E, pr.pol.Ds, pr.pol.U = 300, 12, 10, 10, 2
    assert _ws(pr) == _layout_bytes(4096, 40, 10, 12, 300) and _ws(pr) > 40 * 10 * 4096 * 320 * 8
    # size_t overflow: 0, not a wrapped size
    for P, H in ((PT_MAX_P, (1 << 31) - 1), (PT_MAX_P, 1 << 30), (1 << 20, (1 << 31) - 1)):
        assert _ws(_particles(P=P, H=H)) == 0, (P, H)
    pr = _particles(P=PT_MAX_P, H=1 << 16); pr.dyn.n = (1 << 31) - 64
    assert _ws(pr) == 0


@pytest.mark.skipif(not os.path.exists(CUOBJDUMP), reason="cuobjdump not available")
def test_consistent_kernels_sass():
    names = ["fs_predict_kernel", "fs_cond_kernel"]
    sass = sass_named(names)
    assert set(sass) == set(names)
    for k, text in sass.items():
        assert not re.search(r"\b(STL|LDL)\b", text), k
    assert "DMMA.16x8x16" in sass["fs_predict_kernel"] and "UBLKCP" in sass["fs_predict_kernel"]
    for forbidden in ("gp_predict_kernel", "gp_predict_vjp_kernel", "pt_step_kernel", "pg_step_kernel",
                      "pg_param_kernel", "pg_rbf_finish_kernel"):
        assert not any(forbidden in k for k in names)


def test_consistent_sampling_fails_loudly_without_gpu(monkeypatch):
    from pilco.models import PILCO
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)
    X = np.random.RandomState(0).rand(20, 3); Y = 0.1 * X[:, :2]
    pilco = PILCO((X, Y))
    with pytest.raises(RuntimeError, match="CUDA device"):
        pilco.sample_trajectories(X[0, :2], 0.1 * np.eye(2), 3, num_samples=10, seed=0, consistent=True)


def test_oracle_sequential_draw_equals_joint_draw():
    """Over a fixed, well-separated input sequence the sequential conditioning is the Cholesky factor of the joint
    posterior covariance: f = mu + chol(K_post) eps."""
    dyn, rng = _problem(5, n=30, Ds=3, U=1)
    T, P = 7, 4
    Xs = rng.rand(P, T, 4) * 3.0
    eps = rng.randn(P, T, 3)
    worst = 0.0
    for p in range(P):
        fs = FunctionSample(dyn, 1)
        seq = np.stack([fs.step(Xs[p, t:t + 1], eps[p, t:t + 1])[0] for t in range(T)])
        ref = joint_draw(dyn, Xs[p], eps[p])
        worst = max(worst, float(np.max(np.abs(seq - ref)) / np.max(np.abs(ref))))
    print("sequential vs joint draw over fixed inputs: %.1e of scale" % worst)
    assert worst < 1e-12


def test_oracle_revisited_input_reproduces_its_value():
    dyn, rng = _problem(6, n=30, Ds=3, U=1)
    P = 5
    A, B = rng.rand(P, 4), rng.rand(P, 4)
    fs = FunctionSample(dyn, P)
    fa = fs.step(A, rng.randn(P, 3))
    fs.step(B, rng.randn(P, 3))
    fa2 = fs.step(A, rng.randn(P, 3))                   # the degenerate pivot: no new randomness
    assert np.max(np.abs(fa2 - fa)) <= 1e-6 * np.max(np.abs(fa))     # sqrt of d2 in the rounding noise: ~1e-9
    assert np.all(fs.piv[2] == 0.0) and np.all(fs.piv[0] > 0.0)


def test_oracle_first_step_is_the_marginal_samplers():
    dyn, rng = _problem(7, n=25, Ds=3, U=1)
    P, H = 30, 4
    pol = dict(kind=_lib.POLICY_LINEAR, squash=True, maxa=np.array([1.1]), W=0.7 * rng.randn(1, 3), b=rng.randn(1))
    terms = [dict(kind=_lib.REWARD_EXP, coef=1.0, W=np.eye(3), t=0.4 * np.ones(3))]
    x0, eps = 0.5 + 0.2 * rng.randn(P, 3), rng.randn(P, H, 3)
    cons = consistent_rollout(dyn, pol, terms, x0, eps)
    marg = particle_rollout(dyn, pol, terms, x0, eps)
    assert np.allclose(cons[0][:, :2], marg[0][:, :2], rtol=0, atol=1e-14) and np.array_equal(cons[1][:, :1], marg[1][:, :1])
    assert not np.allclose(cons[0][:, 2:], marg[0][:, 2:])
