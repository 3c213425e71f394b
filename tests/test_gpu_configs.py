"""GPU parity tests at the full BASELINE.json config shapes (SURVEY.md section 8d): complete H-step rollouts through the
C ABI against committed expected values (tests/golden/configs.npz, made by tests/golden/make_config_golden.py
with the numpy port of the reference's Python path), plus size-independent properties over the whole restart
batch: finite moments, info == 0, positive semi-definite state covariances, and independence of a restart's
result from its position in the batch (bitwise).  fp64; tolerances beside each assertion."""
import os

import numpy as np
import pytest
import torch

from util import scaled_err, make_rollout_problem

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "configs.npz")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# name -> (N, Ds, U, bf, H, R, seed, restarts with expected values)   [same table as make_config_golden.py]
CONFIGS = {
    "inverted_pendulum": (300, 4, 1, 10, 40, 1, 11, (0,)),
    "inv_double_pendulum": (400, 6, 1, 40, 40, 32, 12, (0, 31)),
    "swimmer": (500, 8, 2, 40, 50, 32, 13, (0, 31)),
    "metric": (300, 10, 2, 50, 40, 32, 14, (0, 31)),
}


def _plan(P, gp, rows, H):
    from pilco_b200 import engine, _lib
    Ds, U = P["m0"].shape[0], P["Yc"].shape[2]
    R = len(rows)
    pgp = engine.gp_factorize(P["Xc"][rows], P["Yc"][rows], P["lc"][rows], np.ones((R, U)), 1e-4 * np.ones((R, U)),
                              need_iK=False, mode=1)
    spec = dict(kind=_lib.POLICY_RBF, Ds=Ds, U=U, squash=True, max_action=P["maxa"], gp=pgp)
    terms = [dict(kind=_lib.REWARD_EXP, coef=1.0, W=P["W"], t=P["t"])]
    return engine.RolloutPlan(gp, spec, terms, P["m0"], P["S0"], H, R=R)


def _check_batch(name, P, gp, H, R, check, gold, tolM, tolS, tolR):
    plan = _plan(P, gp, list(range(R)), H)
    tm, tS, rew = plan.forward()
    torch.cuda.synchronize()
    assert int(plan.info.max().item()) == 0
    tm, tS, rew = tm.cpu().numpy(), tS.cpu().numpy(), rew.cpu().numpy()
    assert np.isfinite(tm).all() and np.isfinite(tS).all() and np.isfinite(rew).all()
    eig = np.linalg.eigvalsh(0.5 * (tS + np.swapaxes(tS, -1, -2)))
    assert eig.min() > -1e-10, "state covariance lost positive semi-definiteness (min eig %g)" % eig.min()
    for r in check:
        eM = scaled_err(tm[r, -1], gold["%s_r%d_M" % (name, r)][0])
        eS = scaled_err(tS[r, -1], gold["%s_r%d_S" % (name, r)])
        eR = abs(float(rew[r]) - float(gold["%s_r%d_reward" % (name, r)][0, 0]))
        assert eM < tolM and eS < tolS and eR < tolR, (name, r, eM, eS, eR)
    if R > 1:                                  # a restart's rollout must not depend on its batch position
        solo = _plan(P, gp, [check[-1]], H)
        sm, sS, sr = solo.forward()
        torch.cuda.synchronize()
        assert np.array_equal(sm.cpu().numpy()[0], tm[check[-1]]) and np.array_equal(sS.cpu().numpy()[0], tS[check[-1]])
        assert float(sr[0]) == float(rew[check[-1]])


@pytest.mark.parametrize("name", list(CONFIGS))
def test_config_rollout_matches_expected(name):
    from pilco_b200 import engine
    N, Ds, U, bf, H, R, seed, check = CONFIGS[name]
    gold = np.load(GOLD)
    P = make_rollout_problem(N, Ds, U, bf, R, seed=seed)
    gp = engine.gp_factorize(P["X"], P["Y"], P["ell"], P["sf2"], P["sn2"])
    assert int(gp.info.max().item()) == 0
    # 40-50 step cascades compound per-step rounding
    _check_batch(name, P, gp, H, R, check, gold, tolM=1e-10, tolS=1e-10, tolR=1e-10)


def test_config_sparse_rollout_matches_expected():
    """BASELINE config 4 (SMGPR, smgpr.py:24-52): FITC factorisation at N=2000, M=200, E=10, D=12 and the 40-step
    cascade over the inducing points.  FITC is ill-conditioned (|iK| up to ~1e4, SURVEY.md section 8a5); the reference's own
    bar for the sparse path is rtol 1e-4 (tests/test_sparse_predictions.py:55-57)."""
    from pilco_b200 import engine
    gold = np.load(GOLD)
    N, M, Ds, U, bf, H, R, seed = 2000, 200, 10, 2, 50, 40, 2, 15
    P = make_rollout_problem(N, Ds, U, bf, R, seed=seed)
    Z = np.random.RandomState(seed + 100).rand(M, Ds + U)
    gp = engine.fitc_factorize(P["X"], Z, P["Y"], P["ell"], P["sf2"], P["sn2"])
    assert int(gp.info.max().item()) == 0
    beta = gp.beta.cpu().numpy()
    iK = gp.iK.cpu().numpy()[:, :M, :M]
    probe = np.random.RandomState(1).randn(M, 3)
    e_beta = scaled_err(beta, gold["sparse_beta"])
    e_iK = scaled_err(iK @ probe, gold["sparse_iK_probe"])
    assert e_beta < 1e-9 and e_iK < 1e-9, (e_beta, e_iK)
    assert abs(np.abs(iK).max() / float(gold["sparse_iK_absmax"]) - 1.0) < 1e-4
    _check_batch("sparse", P, gp, H, R, (0, 1), gold, tolM=1e-9, tolS=1e-9, tolR=1e-9)
