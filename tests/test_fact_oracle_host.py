"""CPU checks of the factorisation test infrastructure: the extended-precision oracle (tests/fact_oracle.py) against
the fp64 ports of the reference path at benign inputs, against a 40-digit mpmath evaluation in every hard regime, its
complex-step derivative against the closed-form gradient; and the case matrix of tests/fact_cases.py -- every size
cell and every regime is reached."""
import numpy as np
import pytest
import torch

import fact_cases as fc
import fact_oracle as fo

pytestmark = pytest.mark.skipif(not fo.HAVE_EXTENDED, reason=fo.NEED_EXTENDED)


def test_oracle_matches_the_fp64_ports_at_benign_inputs():
    from oracle import python_port as pp
    from pilco_b200 import gp_training as gt
    X, Y, ell, sf2, sn2 = (a[0] for a in fc.make("benign", 60, 3, 2))
    iK, beta = pp.calculate_factorizations(X, Y, ell, sf2, sn2)
    T = lambda a: torch.tensor(np.asarray(a, dtype=np.float64), requires_grad=True)
    for e in range(2):
        f = fo.gp_factor(X, Y[:, e], ell[e], sf2[e], sn2[e])
        sc = fo.gp_scales(f, X, ell[e])
        assert fo.max_ratio(iK[e] - f["iK"].astype(np.float64), sc["iK"]) < 4
        assert fo.beta_backward(f["K"], beta[e], Y[:, e]) < 4 * fo.EPS64
        assert fo.max_ratio(np.abs(f["L"] @ f["L"].T - f["K"]).astype(np.float64), sc["LL"]) < 1e-3
        o = fo.gp_nlml(X, Y[:, e], ell[e], sf2[e], sn2[e])
        te, ts, tn = T(ell[e]), T(sf2[e]), T(sn2[e])
        loss = gt.gpr_loss(torch.tensor(X), torch.tensor(Y[:, e]), te, ts, tn)
        g = torch.autograd.grad(loss, (te, ts, tn))
        assert abs(float(loss) - float(o["nlml"])) < 16 * fo.EPS64 * o["c_nlml"]
        g_ref = np.r_[g[0].numpy(), float(g[1]), float(g[2])]
        assert np.all(np.abs(g_ref - o["grad"].astype(np.float64)) < 16 * fo.EPS64 * o["c_grad"])


def test_fitc_oracle_matches_the_fp64_ports_at_benign_inputs():
    from oracle import python_port as pp
    from oracle import fitc_staged
    from pilco_b200 import gp_training as gt
    X, Y, Z, ell, sf2, sn2 = fc.make_fitc("benign", 80, 12, 3, 2)
    iK, beta = pp.fitc_factorizations(X, Z, Y, ell, sf2, sn2)
    for e in range(2):
        o = fo.fitc_factor(X, Z, Y[:, e], ell[e], sf2[e], sn2[e])
        assert fo.max_ratio(iK[e] - o["iK"].astype(np.float64), o["c_iK"]) < 4
        assert fo.max_ratio(beta[e] - o["beta"].astype(np.float64), o["c_beta"]) < 4
        val, c = fo.fitc_bound(X, Y[:, e], Z, ell[e], sf2[e], sn2[e])
        f64, grad = fitc_staged.fitc_nlml(X, Y[:, e], Z, ell[e], sf2[e], sn2[e])
        assert abs(f64 - float(val)) < 16 * fo.EPS64 * c
        rng = np.random.RandomState(e)
        v_ell, v_sf2, v_sn2, v_Z = rng.randn(3), rng.randn(), rng.randn() * 1e-2, 0.1 * rng.randn(12, 3)
        d = float(fo.fitc_bound_cs(X, Y[:, e], Z, ell[e], sf2[e], sn2[e], v_ell, v_sf2, v_sn2, v_Z))
        terms = np.r_[v_ell * grad["ell"], v_sf2 * grad["sf2"], v_sn2 * grad["sn2"], (v_Z * grad["Z"]).ravel()]
        assert abs(terms.sum() - d) < 1e-9 * np.abs(terms).sum()
        T = lambda a: torch.tensor(np.asarray(a, dtype=np.float64), requires_grad=True)
        tZ, te, ts, tn = T(Z), T(ell[e]), T(sf2[e]), T(sn2[e])
        loss = gt.fitc_loss(torch.tensor(X), torch.tensor(Y[:, e]), tZ, te, ts, tn)
        g = torch.autograd.grad(loss, (te, ts, tn, tZ))
        assert abs(float(loss) - float(val)) < 16 * fo.EPS64 * c
        terms = np.r_[v_ell * g[0].numpy(), v_sf2 * float(g[1]), v_sn2 * float(g[2]), (v_Z * g[3].numpy()).ravel()]
        assert abs(terms.sum() - d) < 1e-9 * np.abs(terms).sum()


def _mp_factor(X, y, ell, sf2, sn2):
    """iK, beta, log det at 40 digits (mpmath's own Cholesky and inverse)"""
    import mpmath as mp
    mp.mp.dps = 40
    n, D = X.shape
    K = mp.matrix(n, n)
    for i in range(n):
        for j in range(n):
            d2 = sum(((mp.mpf(float(X[i, d])) - mp.mpf(float(X[j, d]))) / mp.mpf(float(ell[d]))) ** 2 for d in range(D))
            K[i, j] = mp.mpf(float(sf2)) * mp.exp(-d2 / 2) + (mp.mpf(float(sn2)) if i == j else 0)
    L = mp.cholesky(K)
    iK = mp.inverse(K)
    beta = iK * mp.matrix([mp.mpf(float(v)) for v in y])
    ld = lambda x: fo.LD(float(x)) + fo.LD(float(x - float(x)))          # to longdouble as a sum of two doubles
    return (np.array([[ld(iK[i, j]) for j in range(n)] for i in range(n)]), np.array([ld(beta[i]) for i in range(n)]),
            ld(2 * sum(mp.log(L[i, i]) for i in range(n))))


@pytest.mark.parametrize("regime", fc.HARD)
def test_oracle_matches_mpmath_in_every_hard_regime(regime):
    X, Y, ell, sf2, sn2 = (a[0] for a in fc.make(regime, 12, 4, 1))
    f = fo.gp_factor(X, Y[:, 0], ell[0], sf2[0], sn2[0])
    iK, beta, logdet = _mp_factor(X, Y[:, 0], ell[0], sf2[0], sn2[0])
    sc = fo.gp_scales(f, X, ell[0])
    # the oracle's error in eps64 units of the condition scale: longdouble leaves it ~2e3 times below a fp64 kernel's
    assert fo.max_ratio(f["iK"] - iK, sc["iK"]) < 5e-2
    cb = np.abs(f["iK"].astype(np.float64)) @ (sc["LL"] @ np.abs(f["beta"].astype(np.float64)))
    assert fo.max_ratio(f["beta"] - beta, cb) < 5e-2
    assert abs(float(f["logdet"] - logdet)) < 5e-2 * fo.EPS64 * float((np.abs(f["iK"].astype(np.float64)) * sc["LL"]).sum())


@pytest.mark.parametrize("regime", ("benign",) + fc.HARD)
def test_complex_step_equals_the_closed_form_gradient(regime):
    X, Y, ell, sf2, sn2 = (a[0] for a in fc.make(regime, 40, 3, 1))
    o = fo.gp_nlml(X, Y[:, 0], ell[0], sf2[0], sn2[0])
    for seed in range(3):
        v = np.random.RandomState(seed).randn(5) * np.r_[ell[0], sf2[0], sn2[0]]
        d = fo.gp_nlml_cs(X, Y[:, 0], ell[0], sf2[0], sn2[0], v)
        assert abs(float(d - v @ o["grad"])) <= 1e-2 * fo.EPS64 * float(np.abs(v) @ o["c_grad"])


def test_case_matrix_is_covered():
    assert fc.REQUIRED_CELLS <= fc.covered(), sorted(fc.REQUIRED_CELLS - fc.covered())
    assert {c[0] for c in fc.FACT_CASES} == set(fc.REGIMES)
    # every hard regime at a multi-CTA size too, the training objective at n >= 512, FITC with clustered inducing points
    assert {c[0] for c in fc.FACT_CASES if c[1] >= fc.CHOL_MULTI_N} >= {"noise_floor", "episodes4", "episodes6",
                                                                        "long_ell", "short_ell", "ard_mixed", "scales_hi"}
    assert any(c[1] >= fc.CHOL_MULTI_N for c in fc.NLML_CASES)
    assert any(c[0] == "fitc_clustered" for c in fc.FITC_CASES)


def test_regimes_are_as_conditioned_as_stated():
    """the hard regimes are hard: cond(K + sn2 I) at n = 128"""
    cond = {}
    for regime in fc.REGIMES:
        X, Y, ell, sf2, sn2 = (a[0] for a in fc.make(regime, 128, 3, 1))
        K = fo.gram(X, X, ell[0], sf2[0]).astype(np.float64) + sn2[0] * np.eye(128)
        cond[regime] = np.linalg.cond(K)
    assert cond["short_ell"] < 10
    for regime in ("noise_floor", "episodes6", "long_ell"):
        assert cond[regime] > 1e7, (regime, cond[regime])
    X, _, Z, ell, sf2, _ = fc.make_fitc("fitc_clustered", 100, 33, 3, 1)
    assert np.linalg.cond(fo.gram(Z, Z, ell[0], sf2[0]).astype(np.float64) + 1e-6 * np.eye(33)) > 1e5
