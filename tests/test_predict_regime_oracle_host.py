"""The extended-precision predict and conditioning oracle (tests/predict_regime_oracle.py) on the host: against
40-digit mpmath at hard points of the regimes, against the fp64 consistent-sampler oracle teacher-forced on that
oracle's own trajectory, its VJP against the fp64 closed form, and the size cells of tests/predict_cases.py."""
import numpy as np
import pytest

import particle_grad_oracle as pgo
import particle_oracle as po
import predict_cases as pc
import predict_regime_oracle as pro
from particle_cases import _problem

pytestmark = pytest.mark.skipif(not pro.HAVE_EXTENDED, reason=pro.NEED_EXTENDED)


def test_size_cells_are_covered():
    assert pc.REQUIRED_CELLS - pc.covered() == set()
    assert max(T * n * n * ne for n, _, _, T, _, ne, _ in pc.SIZE_CASES) <= 3e8      # the oracle stays quick
    assert [(i, j) for i, j in pc.probe_pairs(513) if not (0 <= i < 513 and 0 <= j < 513)] == []
    idx = pc.probe_indices(448)
    assert {15, 16, 63, 64, 255, 256, 447} <= set(idx)


def _mp_predict(C, ell, sf2, beta, iK, x):
    import mpmath
    mpmath.mp.dps = 40
    k = [mpmath.mpf(sf2) * mpmath.exp(-sum((mpmath.mpf(x[d]) - mpmath.mpf(C[i, d])) ** 2 / mpmath.mpf(ell[d]) ** 2
                                           for d in range(C.shape[1])) / 2) for i in range(C.shape[0])]
    n = C.shape[0]
    mean = sum(k[i] * mpmath.mpf(beta[i]) for i in range(n))
    var = mpmath.mpf(sf2) - sum(k[i] * mpmath.mpf(iK[i, j]) * k[j] for i in range(n) for j in range(n))
    return mean, var


@pytest.mark.parametrize("regime,family", [("noise_floor", "rows"), ("duplicates", "rows"), ("duplicates", "rows_1e-8"),
                                           ("long_ell", "uniform"), ("benign", "far"), ("fitc_clustered", "rows"),
                                           ("scales_hi", "offset_1e4")])
def test_oracle_against_mpmath_at_hard_points(regime, family):
    import mpmath
    f = pc.factors(regime, 24, 3, 1, seed=2)
    C, Xs = pc.points(family, f, 4, seed=3)
    dyn = pro.ld_model(C, f["ell"], f["sf2"], f["beta"], f["iK"])
    ref = pro.predict(dyn, Xs)
    for r in range(Xs.shape[0]):
        m, v = _mp_predict(C, f["ell"][0], f["sf2"][0], f["beta"][0], f["iK"][0], Xs[r])
        for got, want, sc in ((ref["mean"][r, 0], m, ref["cmean"][r, 0]), (ref["var"][r, 0], v, ref["cvar"][r, 0])):
            err = abs(mpmath.mpf(float(got)) + mpmath.mpf(float(got - pro.LD(float(got)))) - want)
            assert float(err) <= 64 * float(np.finfo(pro.LD).eps) * float(sc) + 1e-300, (regime, family, r, got, want)
    if family == "far":
        assert np.all(ref["mean"] == 0) or np.all(np.abs(ref["mean"]) < 1e-300)


def test_oracle_matches_the_fp64_consistent_oracle_on_its_own_trajectory():
    """po.consistent_rollout in fp64; the longdouble conditioning at its inputs gives the same increments within the
    fp64 oracle's own rounding (the condition scale)"""
    dyn, rng = _problem(3, n=25, Ds=3, U=1)
    pol = dict(kind=po._lib.POLICY_LINEAR, squash=True, maxa=np.array([1.0]), W=0.5 * rng.randn(1, 3), b=rng.randn(1))
    P, H = 6, 36
    x0, eps = 0.5 + 0.1 * rng.randn(P, 3), rng.randn(P, H, 3)
    traj, act = po.consistent_rollout(dyn, pol, [], x0, eps)[:2]
    dld = pro.ld_model(dyn["C"], dyn["ell"], dyn["sf2"], dyn["beta"], dyn["iK"])
    worst, share, mmin = pro.increment_ratios(dld, traj, act, eps)
    print("fp64 oracle vs longdouble conditioning, H=%d: worst ratio %.3g, left out %.3g, smallest margin %.3g"
          % (H, worst, share, mmin))
    assert worst <= 10.0


def test_fp64_oracle_is_unchanged_by_the_longdouble_run():
    """FunctionSample in fp64 stays fp64 (no longdouble leaks into the shared oracle's results)"""
    dyn, rng = _problem(4)
    fs = po.FunctionSample(dyn, 3)
    for t in range(4):
        f = fs.step(rng.rand(3, 4), rng.randn(3, 3))
        assert f.dtype == np.float64 and fs.mean[t].dtype == np.float64


@pytest.mark.parametrize("regime", ["benign", "noise_floor", "offset"])
def test_vjp_matches_the_fp64_closed_form(regime):
    f = pc.factors("noise_floor" if regime == "noise_floor" else "benign", 40, 4, 3, seed=5)
    C, Xs = pc.points("offset_1e4" if regime == "offset" else "uniform", f, 20, seed=6)
    rng = np.random.RandomState(7)
    gm, gv = rng.randn(20, 3), rng.randn(20, 3)
    dyn64 = dict(C=C, ell=f["ell"], sf2=f["sf2"], beta=f["beta"], iK=f["iK"])
    g64, sc64 = pgo.predict_vjp(dyn64, Xs, gm, gv)
    g, sc = pro.predict_vjp(pro.ld_model(C, f["ell"], f["sf2"], f["beta"], f["iK"]), Xs, gm, gv)
    ratio = float(np.max(np.abs(g64.astype(pro.LD) - g) / (pro.EPS64 * sc)))
    print("fp64 VJP vs longdouble (%s): ratio %.3g" % (regime, ratio))
    assert ratio <= 100.0 and np.allclose(sc64, sc.astype(np.float64), rtol=1e-12)
    ref = pro.predict(pro.ld_model(C, f["ell"], f["sf2"], f["beta"], f["iK"]), Xs)
    mean64, var64 = po.gp_latent(dyn64, Xs)
    assert np.max(np.abs(mean64 - ref["mean"]) / (pro.EPS64 * ref["cmean"])) <= 100.0
    assert np.max(np.abs(var64 - ref["var"]) / (pro.EPS64 * ref["cvar"])) <= 100.0
