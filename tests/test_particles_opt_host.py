"""CPU tests of policy optimisation on the sampled return (pilco_particles_rollout_batch_grad,
policy_opt.ParticleEvaluator, PILCO.optimize_policy_sampled): argument validation of the batched entry point
(rejecting calls only), its workspace size, the SASS of the kernels it runs, and the failures without a GPU or with
an objective it cannot optimise."""
import ctypes as C
import os
import re

import numpy as np
import pytest
import torch

from pilco_b200 import _lib
from pilco_b200._lib import lib
from abi_fakes import ERR_ALIGN, ERR_DIM, ERR_NULL, ERR_UNSUP, ERR_WS, FAKE, PT_MAX_P, _batched, _grad, _particles
from particle_cases import _linear_pilco, _safe_pilco
from util import CUOBJDUMP, sass_named


def _run(pr, R, g):
    return lib.pilco_particles_rollout_batch_grad(C.byref(pr) if pr is not None else None, R,
                                                  C.byref(g) if g is not None else None, None)


def test_batch_grad_argument_validation():
    assert _run(None, 3, _grad()) == ERR_NULL
    assert _run(_batched(), 3, None) == ERR_NULL
    for kind in (_lib.POLICY_LINEAR, _lib.POLICY_RBF):
        for rk in (_lib.REWARD_EXP, _lib.REWARD_LINEAR, _lib.REWARD_BOX):
            for ch in (_lib.CHANNEL_ADD, _lib.CHANNEL_MULT):
                assert _run(_batched(kind, reward_kind=rk, channel=ch), 3, _grad()) == ERR_WS, (kind, rk, ch)
        assert _run(_particles(kind), 3, _grad()) == ERR_WS                 # stride 0: one policy shared by all
    # R: at least one, at most 65535 CTA rows, and R P predict points within the predict kernel's limit
    for R in (0, -1, 65536):
        assert _run(_batched(), R, _grad()) == ERR_DIM, R
    P = 1000
    assert _run(_batched(P=P), PT_MAX_P // P, _grad()) == ERR_WS
    assert _run(_batched(P=P), PT_MAX_P // P + 1, _grad()) == ERR_DIM
    assert _run(_batched(P=1), 65535, _grad()) == ERR_WS
    # negative strides
    for field in ("W_bs", "b_bs"):
        pr = _batched(); setattr(pr.pol, field, -3)
        assert _run(pr, 3, _grad()) == ERR_DIM, field
    for field in ("X_bs", "ell_bs", "sf2_bs", "beta_bs"):
        pr = _batched(_lib.POLICY_RBF); setattr(pr.pol.rbf, field, -1)
        assert _run(pr, 3, _grad()) == ERR_DIM, field
    # batched dynamics
    for field in ("X_bs", "ell_bs", "sf2_bs", "beta_bs"):
        pr = _batched(); setattr(pr.dyn, field, 7)
        assert _run(pr, 3, _grad()) == ERR_UNSUP, field
    # everything the unbatched entry point checks
    for P, H in ((0, 5), (PT_MAX_P + 1, 5), (10, -1)):
        assert _run(_batched(P=P, H=H), 1, _grad()) == ERR_DIM, (P, H)
    for field in ("x0", "eps", "traj", "act", "step_reward", "step_risk", "ret"):
        pr = _batched(); setattr(pr, field, None)
        assert _run(pr, 3, _grad()) == ERR_NULL, field
    pr = _batched(_lib.POLICY_RBF); pr.pol.rbf.mode = 0
    assert _run(pr, 3, _grad()) == ERR_UNSUP
    pr = _batched(); pr.dyn.iK = FAKE + 8
    assert _run(pr, 3, _grad()) == ERR_ALIGN
    for field in ("value", "ws", "gW", "gb"):
        g = _grad(); setattr(g, field, None)
        assert _run(_batched(), 3, g) == ERR_NULL, field
    for field in ("gXc", "gYc", "gell", "pol_L"):
        g = _grad(); setattr(g, field, None)
        assert _run(_batched(_lib.POLICY_RBF), 3, g) == ERR_NULL, field
    g = _grad(); g.ws = FAKE + 8; g.ws_bytes = 1 << 40
    assert _run(_batched(), 3, g) == ERR_ALIGN
    for kind in (_lib.POLICY_LINEAR, _lib.POLICY_RBF):
        pr = _batched(kind)
        need = lib.pilco_particles_batch_grad_workspace_bytes(C.byref(pr), 3)
        g = _grad(); g.ws_bytes = need - 8
        assert need > 0 and _run(pr, 3, g) == ERR_WS


def test_unbatched_entry_points_still_reject_batched_policies():
    for kind in (_lib.POLICY_LINEAR, _lib.POLICY_RBF):
        pr = _batched(kind)
        assert lib.pilco_particles_rollout(C.byref(pr), None) == ERR_UNSUP
        assert lib.pilco_particles_rollout_grad(C.byref(pr), C.byref(_grad()), None) == ERR_UNSUP


def _layout_bytes(P, H, Ds, U, D, n, bf, R):
    """the workspace layout: x~ [H,RP,D], mean [RP,Ds], var [H,RP,Ds], gx, gvar [RP,Ds], VJP out [RP,D],
    z_bar [RP,H,U], the RBF sums [R,U,bf,Ds] x 2 and [R,U,bf] x 2, then one predict / VJP workspace at T = R P"""
    T = R * P
    even = lambda k: (k + 1) & ~1
    doubles = sum(even(k) for k in (H * T * D, T * Ds, H * T * Ds, T * Ds, T * Ds, T * D, T * H * U,
                                    R * U * bf * Ds, R * U * bf * Ds, R * U * bf, R * U * bf))
    pred = lib.pilco_gp_predict_workspace_bytes(n, D, Ds, T, 0)
    vjp = lib.pilco_gp_predict_vjp_workspace_bytes(n, D, Ds, T)
    return 8 * doubles + max(pred, vjp)


def test_batch_grad_workspace_bytes():
    f = lambda pr, R: lib.pilco_particles_batch_grad_workspace_bytes(C.byref(pr) if pr is not None else None, R)
    assert f(None, 3) == 0
    for R in (0, -2, 65536):
        assert f(_batched(), R) == 0, R
    assert f(_batched(P=1000), PT_MAX_P // 1000 + 1) == 0
    for P, H in ((0, 5), (PT_MAX_P + 1, 5), (10, -1)):
        assert f(_batched(P=P, H=H), 1) == 0
    for kind, bf in ((_lib.POLICY_LINEAR, 0), (_lib.POLICY_RBF, 20)):
        pr = _batched(kind, P=1000, H=5)
        assert f(pr, 1) == lib.pilco_particles_grad_workspace_bytes(C.byref(pr))       # R = 1: the unbatched call's
        for R in (1, 2, 7, 32):
            assert f(pr, R) == _layout_bytes(1000, 5, 3, 1, 4, 50, bf, R), (kind, R)
        assert f(pr, 32) > 30 * f(pr, 1)
    assert f(_batched(P=4096, H=40), 500) < 8 * 500 * 4096 * (40 * (4 + 3 + 1) + 64)  # no [., n] intermediate


@pytest.mark.skipif(not os.path.exists(CUOBJDUMP), reason="cuobjdump not available")
def test_batched_kernels_sass():
    names = ["pt_step_kernel", "pg_step_kernel", "pg_param_kernel", "pg_rbf_finish_kernel", "rbf_factor_bwd_kernel",
             "gp_predict_kernel", "gp_predict_vjp_kernel"]
    sass = sass_named(names)
    assert set(sass) == set(names)
    for k, text in sass.items():
        assert not re.search(r"\b(STL|LDL)\b", text), k
    for k in ("gp_predict_kernel", "gp_predict_vjp_kernel"):
        assert "DMMA.16x8x16" in sass[k] and "UBLKCP" in sass[k], k


def test_sampled_optimisation_fails_loudly_without_gpu(monkeypatch):
    from pilco_b200 import policy_opt
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)
    pilco, X = _linear_pilco()
    flat = pilco.controller.get_flat().copy()
    with pytest.raises(RuntimeError, match="CUDA device"):
        pilco.optimize_policy_sampled(maxiter=2, restarts=2, num_samples=10, seed=0)
    assert np.array_equal(pilco.controller.get_flat(), flat)
    assert all(p.trainable for m in pilco.mgpr.models for p in (m.kernel.lengthscales, m.kernel.variance))
    with pytest.raises(RuntimeError, match="CUDA device"):
        policy_opt.ParticleEvaluator(pilco, 2, np.zeros((10, 2)), np.zeros((10, 4, 2)))


def test_sampled_optimisation_rejects_box_terms_and_no_samples():
    from pilco_b200 import policy_opt
    sp = _safe_pilco()
    with pytest.raises(ValueError, match="box"):
        sp.optimize_policy_sampled(maxiter=2, restarts=2, num_samples=10, seed=0)
    with pytest.raises(ValueError, match="box"):
        policy_opt.ParticleEvaluator(sp, 2, np.zeros((10, 4)), np.zeros((10, 4, 4)))
    pilco, _ = _linear_pilco()
    for S in (0, -5):
        with pytest.raises(ValueError, match="num_samples"):
            pilco.optimize_policy_sampled(num_samples=S)
