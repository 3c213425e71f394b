"""CPU tests of the consistent sampler's pathwise gradient (pilco_particles_rollout_consistent_grad,
engine.ConsistentGradPlan, PILCO.sample_policy_gradient / optimize_policy_sampled(..., consistent=True)): the torch
autograd oracle (tests/consistent_grad_oracle.py) against central differences of the numpy consistent sampler, the
explicit reverse steps against autograd, the oracle against the step-wise one at H <= 2, argument validation of the C
entry point (rejecting calls only), the exact workspace layout with its 0 on overflow, the SASS, and the failures
without a GPU or with box terms."""
import ctypes as C
import hashlib
import json
import os
import re

import numpy as np
import pytest
import torch

from pilco_b200 import _lib
from pilco_b200._lib import lib
from consistent_grad_oracle import fixed_inputs_objective, reverse_steps, value_and_grad
from consistent_oracle import consistent_rollout
from particle_grad_oracle import rbf_pol_np, value_and_grad as stepwise_value_and_grad
from test_particles_host import ERR_ALIGN, ERR_DIM, ERR_NULL, ERR_UNSUP, ERR_WS, FAKE, ROOT, _particles
from test_particles_grad_host import CUOBJDUMP, _grad, _problem, _sass, _terms
from test_particles_opt_host import _batched, _linear_pilco, _safe_pilco

PT_MAX_P = 65535 * 32


def _fd(dyn, pol, keys, rebuild, terms, x0, eps, mu, h=1e-6):
    """autograd gradient against central differences of the numpy sampler's mean return, every parameter"""
    v, g, ratio = value_and_grad(dyn, pol, terms, x0, eps, mu)
    worst, scale = 0.0, max(np.abs(gv).max() for gv in g.values())
    for k, src in keys.items():
        base = np.asarray(pol[src], dtype=np.float64)
        for idx in np.ndindex(base.shape):
            vals = []
            for s in (1.0, -1.0):
                p = base.copy(); p[idx] += s * h
                vals.append(consistent_rollout(dyn, rebuild(src, p), terms, x0, eps, mu)[4].mean())
            worst = max(worst, abs((vals[0] - vals[1]) / (2 * h) - g[k][idx]) / scale)
    dv = abs(v - consistent_rollout(dyn, rebuild(None, None), terms, x0, eps, mu)[4].mean())
    return worst, dv, ratio


def test_autograd_oracle_matches_finite_differences_linear():
    dyn, rng = _problem(11)
    Ds, U, P, H = 3, 1, 30, 5
    W, b, maxa = 0.7 * rng.randn(U, Ds), rng.randn(U), np.array([1.2])
    x0, eps = 0.5 + 0.2 * rng.randn(P, Ds), rng.randn(P, H, Ds)
    pol = dict(kind=_lib.POLICY_LINEAR, squash=True, maxa=maxa, W=W, b=b)

    def rebuild(src, p):
        q = dict(pol)
        if src:
            q[src] = p
        return q
    worst, dv, ratio = _fd(dyn, pol, {"W": "W", "b": "b"}, rebuild, _terms(Ds), x0, eps, -2.0)
    print("consistent linear: autograd vs central differences %.1e of scale, value %.1e; smallest pivot "
          "d2 / (tau sf2) = %.1e" % (worst, dv, ratio))
    assert ratio >= 1e3 and worst < 1e-6 and dv < 1e-13


def test_autograd_oracle_matches_finite_differences_rbf():
    dyn, rng = _problem(12)
    Ds, U, bf, P, H = 3, 1, 6, 20, 4
    prm = dict(Xc=rng.rand(bf, Ds), Yc=0.5 * rng.randn(bf, U), ell=0.6 + 0.3 * rng.rand(U, Ds))
    maxa = np.array([0.9])

    def rebuild(src, p):
        q = dict(prm)
        if src:
            q[src] = p
        return rbf_pol_np(q["Xc"], q["Yc"], q["ell"], maxa)
    x0, eps = 0.5 + 0.2 * rng.randn(P, Ds), rng.randn(P, H, Ds)
    pol = dict(kind=_lib.POLICY_RBF, squash=True, maxa=maxa, sf2=np.ones(U), sn2=1e-4 * np.ones(U), **prm)
    worst, dv, ratio = _fd(dyn, pol, {"X": "Xc", "Y": "Yc", "ell": "ell"}, rebuild, _terms(Ds), x0, eps, 1.5)
    print("consistent rbf: autograd vs central differences %.1e of scale, value %.1e; smallest pivot "
          "d2 / (tau sf2) = %.1e" % (worst, dv, ratio))
    assert ratio >= 1e3 and worst < 1e-6 and dv < 1e-13


@pytest.mark.parametrize("revisit", [False, True])
def test_reverse_steps_equal_autograd(revisit):
    """DESIGN.md section 15's steps 1-6 written out in numpy against autograd of the draw at fixed inputs; a revisited
    input has a degenerate pivot, whose own noise the tau rule holds constant"""
    dyn, rng = _problem(13, n=30, Ds=3, U=1)
    T = 8
    Xs = rng.rand(T, 4) * 2.0
    if revisit:
        Xs[5] = Xs[2]
    eps, mb, vb = rng.randn(T, 3), rng.randn(T, 3), rng.randn(T, 3)
    x = torch.tensor(Xs, requires_grad=True)
    ref = torch.autograd.grad(fixed_inputs_objective(dyn, x, eps, mb, vb), x)[0].numpy()
    got = reverse_steps(dyn, Xs, eps, mb, vb)
    err = float(np.abs(got - ref).max() / np.abs(ref).max())
    print("reverse steps 1-6 vs autograd (revisited input: %s): %.1e relative" % (revisit, err))
    assert err < 1e-12


@pytest.mark.parametrize("H", [0, 1, 2])
def test_short_horizons_equal_the_stepwise_gradient(H):
    """at H <= 2 the rewarded states x_0, x_1 depend on step 0 only, which is the marginal sampler's step"""
    dyn, rng = _problem(14)
    P, Ds = 25, 3
    pol = dict(kind=_lib.POLICY_LINEAR, squash=True, maxa=np.array([1.1]), W=0.6 * rng.randn(1, Ds), b=rng.randn(1))
    x0, eps = 0.5 + 0.2 * rng.randn(P, Ds), rng.randn(P, H, Ds)
    v, g, _ = value_and_grad(dyn, pol, _terms(Ds), x0, eps, -1.0)
    v1, g1 = stepwise_value_and_grad(dyn, pol, _terms(Ds), x0, eps, -1.0)
    assert abs(v - v1) <= 1e-15 * max(abs(v1), 1.0)
    for k in g1:
        assert np.allclose(g[k], g1[k], rtol=1e-14, atol=1e-16), k


def _run(pr, R, g):
    return lib.pilco_particles_rollout_consistent_grad(C.byref(pr) if pr is not None else None, R,
                                                       C.byref(g) if g is not None else None, None)


def _ws(pr, R):
    return lib.pilco_particles_consistent_grad_workspace_bytes(C.byref(pr) if pr is not None else None, R)


def test_consistent_grad_argument_validation():
    assert _run(None, 1, _grad()) == ERR_NULL
    assert _run(_particles(), 1, None) == ERR_NULL
    assert _run(_particles(), 1, _grad()) == ERR_WS                         # valid description, no workspace
    for kind in (_lib.POLICY_LINEAR, _lib.POLICY_RBF):
        for rk in (_lib.REWARD_EXP, _lib.REWARD_LINEAR, _lib.REWARD_BOX):
            for ch in (_lib.CHANNEL_ADD, _lib.CHANNEL_MULT):
                assert _run(_batched(kind, reward_kind=rk, channel=ch), 3, _grad()) == ERR_WS, (kind, rk, ch)
        assert _run(_particles(kind), 3, _grad()) == ERR_WS                 # stride 0: one policy shared by all
    assert _run(_particles(H=0), 1, _grad()) == ERR_WS
    pr = _particles(); pr.ws = None                                         # the forward's workspace is not used
    assert _run(pr, 1, _grad()) == ERR_WS
    # R bounds
    for R in (0, -1, 65536):
        assert _run(_batched(), R, _grad()) == ERR_DIM, R
    assert _run(_batched(P=1000), PT_MAX_P // 1000, _grad()) == ERR_WS
    assert _run(_batched(P=1000), PT_MAX_P // 1000 + 1, _grad()) == ERR_DIM
    # negative strides
    for field in ("W_bs", "b_bs"):
        pr = _batched(); setattr(pr.pol, field, -3)
        assert _run(pr, 3, _grad()) == ERR_DIM, field
    for field in ("X_bs", "ell_bs", "sf2_bs", "beta_bs"):
        pr = _batched(_lib.POLICY_RBF); setattr(pr.pol.rbf, field, -1)
        assert _run(pr, 3, _grad()) == ERR_DIM, field
        pr = _batched(); setattr(pr.dyn, field, 7)
        assert _run(pr, 3, _grad()) == ERR_UNSUP, field
    for P, H in ((0, 5), (PT_MAX_P + 1, 5), (10, -1)):
        assert _run(_particles(P=P, H=H), 1, _grad()) == ERR_DIM, (P, H)
    for field in ("x0", "eps", "traj", "act", "step_reward", "step_risk", "ret"):
        pr = _batched(); setattr(pr, field, None)
        assert _run(pr, 3, _grad()) == ERR_NULL, field
    pr = _particles(); pr.dyn.iK = None
    assert _run(pr, 1, _grad()) == ERR_UNSUP
    pr = _particles(_lib.POLICY_RBF); pr.pol.rbf.mode = 0
    assert _run(pr, 1, _grad()) == ERR_UNSUP
    assert _run(_particles(kind=7), 1, _grad()) == ERR_UNSUP
    pr = _particles(); pr.dyn.E = 4
    assert _run(pr, 1, _grad()) == ERR_DIM
    pr = _particles(); pr.dyn.iK = FAKE + 8
    assert _run(pr, 1, _grad()) == ERR_ALIGN
    for field in ("value", "ws", "gW", "gb"):
        g = _grad(); setattr(g, field, None)
        assert _run(_batched(), 3, g) == ERR_NULL, field
    for field in ("gXc", "gYc", "gell", "pol_L"):
        g = _grad(); setattr(g, field, None)
        assert _run(_batched(_lib.POLICY_RBF), 3, g) == ERR_NULL, field
    g = _grad(); g.ws = FAKE + 8; g.ws_bytes = 1 << 40                      # misaligned workspace
    assert _run(_batched(), 3, g) == ERR_ALIGN
    pr = _particles(P=PT_MAX_P, H=(1 << 31) - 1)                            # the workspace size overflows size_t
    g = _grad(); g.ws_bytes = (1 << 64) - 1
    assert _run(pr, 1, g) == ERR_DIM
    for kind in (_lib.POLICY_LINEAR, _lib.POLICY_RBF):                      # a short workspace
        for H in (0, 1, 5):
            pr = _batched(kind, H=H)
            need = _ws(pr, 3)
            g = _grad(); g.ws_bytes = need - 8
            assert need > 0 and _run(pr, 3, g) == ERR_WS, (kind, H)


def _layout_bytes(P, H, Ds, U, D, n, bf, R):
    """the consistent forward's workspace at T = R P (x~ [H,T,D]; mu, var, mean', var' [T,Ds]; W [E,T,np]; the K*
    history [H,E,T,np]; the packed rows [H(H+1)/2,E,T]; a predict workspace at T), then the var' history [H,T,Ds], the
    packed cotangent rows [H(H+1)/2,E,T], the direct sums [E,T,D], x_bar and var_bar [T,Ds], the VJP output [T,D],
    z_bar [T,H,U], the RBF sums [R,U,bf,Ds] x 2 and [R,U,bf] x 2, then a VJP workspace at T"""
    T = R * P
    even = lambda k: (k + 1) & ~1
    np_ = lib.pilco_pad_n(n)
    fwd = sum(even(k) for k in (H * T * D, T * Ds, T * Ds, T * Ds, T * Ds, Ds * T * np_, H * Ds * T * np_,
                                H * (H + 1) // 2 * Ds * T))
    bwd = sum(even(k) for k in (H * T * Ds, H * (H + 1) // 2 * Ds * T, Ds * T * D, T * Ds, T * Ds, T * D, T * H * U,
                                R * U * bf * Ds, R * U * bf * Ds, R * U * bf, R * U * bf))
    return (8 * fwd + lib.pilco_gp_predict_workspace_bytes(n, D, Ds, T, 0) + 8 * bwd
            + lib.pilco_gp_predict_vjp_workspace_bytes(n, D, Ds, T))


def test_consistent_grad_workspace_bytes():
    assert _ws(None, 1) == 0
    for R in (0, -2, 65536):
        assert _ws(_batched(), R) == 0, R
    assert _ws(_batched(P=1000), PT_MAX_P // 1000 + 1) == 0
    for P, H in ((0, 5), (PT_MAX_P + 1, 5), (10, -1)):
        assert _ws(_particles(P=P, H=H), 1) == 0, (P, H)
    for kind, bf in ((_lib.POLICY_LINEAR, 0), (_lib.POLICY_RBF, 20)):
        for P, H, R in ((1, 0, 1), (1000, 5, 1), (777, 1, 3), (300, 7, 16)):
            assert _ws(_batched(kind, P=P, H=H), R) == _layout_bytes(P, H, 3, 1, 4, 50, bf, R), (kind, P, H, R)
    # R = 1: the consistent forward's workspace is part of it
    pr = _particles(P=4096, H=40)
    assert _ws(pr, 1) > lib.pilco_particles_consistent_workspace_bytes(C.byref(pr))
    # the metric shape (n = 300, D = 12, E = 10, H = 40): 1024 particles x 16 restarts need 19.5 GB, of which the K*
    # history is 16.8 GB and the packed factor and cotangent rows 2.1 GB
    pr = _particles(P=1024, H=40)
    pr.dyn.n, pr.dyn.D, pr.dyn.E, pr.pol.Ds, pr.pol.U = 300, 12, 10, 10, 2
    assert _ws(pr, 16) == _layout_bytes(1024, 40, 10, 2, 12, 300, 0, 16) and 19e9 < _ws(pr, 16) < 20e9
    # size_t overflow: 0, not a wrapped size
    for P, H, R in ((PT_MAX_P, (1 << 31) - 1, 1), (1 << 10, 1 << 30, 2), (1 << 20, (1 << 31) - 1, 2)):
        assert _ws(_particles(P=P, H=H), R) == 0, (P, H, R)


SASS_GOLDEN = os.path.join(ROOT, "tests", "golden", "consistent_grad_sass.json")


@pytest.mark.skipif(not os.path.exists(CUOBJDUMP), reason="cuobjdump not available")
def test_consistent_grad_kernels_sass():
    names = ["fs_cond_bwd_kernel", "fs_predict_vjp_kernel", "fs_cond_kernel", "pg_step_kernel", "pg_param_kernel",
             "pg_rbf_finish_kernel", "gp_predict_vjp_kernel", "fs_predict_kernel"]
    sass = _sass(names)
    assert set(sass) == set(names)
    for k, text in sass.items():
        assert not re.search(r"\b(STL|LDL)\b", text), k
    assert "DMMA.16x8x16" in sass["fs_predict_vjp_kernel"] and "UBLKCP" in sass["fs_predict_vjp_kernel"]
    # the predict VJP and the consistent forward's predict are separate copies, untouched by their new sibling
    with open(SASS_GOLDEN) as f:
        golden = json.load(f)
    for k, h in golden.items():
        assert hashlib.sha256(sass[k].encode()).hexdigest() == h, k


def test_consistent_gradient_fails_loudly_without_gpu(monkeypatch):
    from pilco_b200 import policy_opt
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)
    pilco, X = _linear_pilco()
    with pytest.raises(RuntimeError, match="CUDA device"):
        pilco.sample_policy_gradient(X[0, :2], 0.1 * np.eye(2), 3, num_samples=10, seed=0, consistent=True)
    flat = pilco.controller.get_flat().copy()
    with pytest.raises(RuntimeError, match="CUDA device"):
        pilco.optimize_policy_sampled(maxiter=2, restarts=2, num_samples=10, seed=0, consistent=True)
    assert np.array_equal(pilco.controller.get_flat(), flat)
    with pytest.raises(RuntimeError, match="CUDA device"):
        policy_opt.ParticleEvaluator(pilco, 2, np.zeros((10, 2)), np.zeros((10, 4, 2)), consistent=True)


def test_consistent_optimisation_rejects_box_terms():
    from pilco_b200 import policy_opt
    sp = _safe_pilco()
    with pytest.raises(ValueError, match="box"):
        sp.optimize_policy_sampled(maxiter=2, restarts=2, num_samples=10, seed=0, consistent=True)
    with pytest.raises(ValueError, match="box"):
        policy_opt.ParticleEvaluator(sp, 2, np.zeros((10, 4)), np.zeros((10, 4, 4)), consistent=True)
