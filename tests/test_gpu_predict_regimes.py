"""The predict kernels (pilco_gp_predict, diagonal and full covariance, and pilco_gp_predict_vjp) away from the benign
regime (``-m gpu``): every regime of tests/predict_cases.py x every test-point family at two shapes, and every size
cell at benign numbers, against the extended-precision oracle tests/predict_regime_oracle.py.  An entry is judged by
``|error| / (eps64 * condition scale)`` (the ratio); one-hot factors pin every 16-row chunk, 64-column warp and
256-column j block edge and row n - 1; far points must give exactly (0, sf2); the largest T is computed and T + 1
refused.  The factors are inputs (``engine.DeviceGP`` directly, zero-padded iK), so nothing here depends on the
factorisation kernels.

Bars: about 10 x the largest ratio observed on an H100 80GB HBM3 (700 W power limit, 1980 MHz max SM clock).  Observed,
worst over a regime's two shapes and four finite-point families (mean / var / full covariance / VJP):
  benign 0.28 / 0.10 / 0.42 / 0.12     noise_floor 0.38 / 0.10 / 0.51 / 0.10   episodes4 0.47 / 0.05 / 0.27 / 0.05
  episodes6 0.26 / 0.05 / 0.15 / 0.04  duplicates 0.32 / 0.13 / 0.23 / 0.12    long_ell 0.23 / 0.12 / 0.27 / 0.13
  ard_mixed 7.8 / 1.6 / 15 / 3.8       scales_lo 0.37 / 0.09 / 0.36 / 0.11     scales_hi 0.36 / 0.09 / 0.41 / 0.11
  fitc_benign 0.35 / 0.05 / 0.25 / 0.05  fitc_clustered 0.57 / 0.13 / 0.86 / 0.11
  size cells 0.73 / 0.15 / 0.57 / 0.28   largest T 0.26 / 0.08 / - / 0.11      one-hot probes: VJP 1.5
  short_ell 627 / 0.65 / 793 / 628: ell = 1e-2 puts the exponent -d2/2 near -3e3, and exp multiplies the rounding of its
  argument by that much; the sum of |terms| does not carry the factor, so short_ell has its own bars.
One-hot probes: mean and var within 2.6e-16 of the element.  Runtime of this file on that card: about 90 s."""
import numpy as np
import pytest

import predict_cases as pc
import predict_regime_oracle as pro

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not pro.HAVE_EXTENDED, reason=pro.NEED_EXTENDED)]

BARS = dict(mean=80.0, var=20.0, cov=150.0, vjp=40.0)
SHORT_ELL_BARS = dict(mean=6.3e3, var=10.0, cov=8e3, vjp=6.3e3)
PROBE_RTOL = 1e-13     # one exp, a D-term distance and one product: no cancellation


def _engine():
    from pilco_b200 import engine
    return engine


def device_gp(C, f, ldk_extra=0):
    eng = _engine()
    n = C.shape[0]
    ldk = pc.pad64(n) + ldk_extra
    iK = np.zeros((f["iK"].shape[0], ldk, ldk))
    iK[:, :n, :n] = f["iK"]
    return eng.DeviceGP(eng.dev(C), eng.dev(f["ell"]), eng.dev(f["sf2"]), eng.dev(f["beta"]), eng.dev(iK), ldk)


def _ratio(got, want, scale):
    return float(np.max(np.abs(np.asarray(got, dtype=pro.LD) - want) / (pro.EPS64 * scale + pro.TINY)))


def _cotangents(T, E, seed):
    rng = np.random.RandomState(seed)
    return rng.randn(T, E), rng.randn(T, E)


def check_all(C, f, Xs, e0=0, ne=None, ldk_extra=0, full=True, seed=0):
    """mean, var (diagonal), the full covariance of the first output (T <= 256) and the VJP over all outputs against
    the oracle -> their worst ratios"""
    eng = _engine()
    E = f["ell"].shape[0]
    ne = E - e0 if ne is None else ne
    gp = device_gp(C, f, ldk_extra)
    dyn = pro.ld_model(C, f["ell"], f["sf2"], f["beta"], f["iK"])
    ref = pro.predict(dyn, Xs, e0, ne)
    mean, var = (a.cpu().numpy() for a in eng.gp_predict(gp, Xs, e0=e0, ne=ne))
    out = dict(mean=_ratio(mean, ref["mean"], ref["cmean"]), var=_ratio(var, ref["var"], ref["cvar"]))
    if full and Xs.shape[0] <= 256:
        mc, cov = (a.cpu().numpy() for a in eng.gp_predict(gp, Xs, e0=e0, ne=1, full_cov=True))
        want, sc = pro.full_cov(dyn, Xs, e0)
        out["cov"] = max(_ratio(cov[0], want, sc), _ratio(mc[:, 0], ref["mean"][:, 0], ref["cmean"][:, 0]))
    gm, gv = _cotangents(Xs.shape[0], E, seed)
    gx = eng.gp_predict_vjp(gp, Xs, gm, gv).cpu().numpy()
    want, sc = pro.predict_vjp(dyn, Xs, gm, gv)
    out["vjp"] = _ratio(gx, want, sc)
    return out


def assert_bars(r, what, bars=BARS):
    print("%s: ratios %s" % (what, ", ".join("%s %.3g" % kv for kv in sorted(r.items()))))
    for k, v in r.items():
        assert v <= bars[k], (what, k, v)


def test_size_cells_are_covered():
    assert pc.REQUIRED_CELLS - pc.covered() == set()


@pytest.mark.parametrize("n,D,E,T,e0,ne,ldk_extra", pc.SIZE_CASES,
                         ids=["n%d-D%d-E%d-T%d-e%d+%d-ldk%+d" % c for c in pc.SIZE_CASES])
def test_every_size_cell_at_benign_numbers(n, D, E, T, e0, ne, ldk_extra):
    f = pc.factors("benign", n, D, E, seed=n + D)
    C, Xs = pc.points("uniform", f, T, seed=T)
    assert_bars(check_all(C, f, Xs, e0, ne, ldk_extra, seed=n), "size n=%d D=%d E=%d T=%d" % (n, D, E, T))


REGIME_CASES = [(r,) + s for r in pc.REGIMES for s in pc.REGIME_SHAPES]


@pytest.mark.parametrize("regime,n,D,E,T", REGIME_CASES, ids=["%s-n%d-D%d-E%d-T%d" % c for c in REGIME_CASES])
def test_every_regime_and_point_family(regime, n, D, E, T):
    f = pc.factors(regime, n, D, E, seed=n)
    for family in pc.FAMILIES:
        C, Xs = pc.points(family, f, T, seed=n)
        if family == "far":
            check_far(C, f, Xs)
            continue
        assert_bars(check_all(C, f, Xs, seed=T), "%s n=%d %s" % (regime, n, family),
                    SHORT_ELL_BARS if regime == "short_ell" else BARS)


def check_far(C, f, Xs):
    """every k* underflows to 0: mean exactly 0, var exactly sf2, the covariance exactly k(x, x'), the VJP exactly 0"""
    eng = _engine()
    gp = device_gp(C, f)
    E = f["ell"].shape[0]
    mean, var = (a.cpu().numpy() for a in eng.gp_predict(gp, Xs))
    assert np.all(mean == 0.0) and np.all(var == f["sf2"][None, :])
    _, cov = eng.gp_predict(gp, Xs[:8], ne=1, full_cov=True)
    d = (Xs[:8, None] - Xs[None, :8]) / f["ell"][0]
    a = 0.5 * (d * d).sum(-1)                   # exp multiplies the rounding of its argument a by a
    ref = f["sf2"][0] * np.exp(-a)
    assert np.all(np.abs(cov[0].cpu().numpy() - ref) <= 8 * pro.EPS64 * (1.0 + a) * ref)
    gm, gv = _cotangents(Xs.shape[0], E, 1)
    assert np.all(eng.gp_predict_vjp(gp, Xs, gm, gv).cpu().numpy() == 0.0)


def test_far_points_of_every_size():
    for n, D, E, T, e0, ne, _ in pc.SIZE_CASES[:-1]:
        f = pc.factors("benign", n, D, E, seed=n)
        C, Xs = pc.points("far", f, min(T, 300), seed=n)
        check_far(C, f, Xs)


def _probe_model(n, D, pairs, seed):
    """E = len(pairs) outputs: beta_e = e_i, iK_e = e_i e_j' + e_j e_i' for (i, j) = pairs[e]"""
    rng = np.random.RandomState(seed)
    E = len(pairs)
    C = rng.rand(n, D)
    beta, iK = np.zeros((E, n)), np.zeros((E, n, n))
    for e, (i, j) in enumerate(pairs):
        beta[e, i] = 1.0
        iK[e, i, j] += 1.0
        iK[e, j, i] += 1.0
    return C, dict(ell=1.0 + rng.rand(E, D), sf2=1.0 + rng.rand(E), beta=beta, iK=iK)


@pytest.mark.parametrize("n", pc.PROBE_NS)
def test_one_hot_probes_pin_every_tile_edge(n):
    """mean = k_i and var = sf2 - 2 k_i k_j to 1e-13 of the element for every probe pair, and the VJP's ratio"""
    eng = _engine()
    pairs = pc.probe_pairs(n)
    D, T = 3, 33
    worst = dict(mean=0.0, var=0.0, vjp=0.0)
    for g in range(0, len(pairs), pc.MAXE):
        grp = pairs[g:g + pc.MAXE]
        C, f = _probe_model(n, D, grp, seed=n + g)
        Xs = C.min(0) + (C.max(0) - C.min(0)) * np.random.RandomState(g).rand(T, D)
        gp = device_gp(C, f, ldk_extra=64 if (g // pc.MAXE) % 2 else 0)
        mean, var = (a.cpu().numpy() for a in eng.gp_predict(gp, Xs))
        dyn = pro.ld_model(C, f["ell"], f["sf2"], f["beta"], f["iK"])
        for e, (i, j) in enumerate(grp):
            ki = pro.po.se_k(pro.mo._ld(Xs), dyn["C"][i:i + 1], dyn["ell"][e], dyn["sf2"][e])[:, 0]
            kj = pro.po.se_k(pro.mo._ld(Xs), dyn["C"][j:j + 1], dyn["ell"][e], dyn["sf2"][e])[:, 0]
            em = float(np.max(np.abs(mean[:, e] - ki) / ki))
            ev = float(np.max(np.abs(var[:, e] - (dyn["sf2"][e] - 2 * ki * kj)) / (dyn["sf2"][e] + 2 * ki * kj)))
            worst["mean"], worst["var"] = max(worst["mean"], em), max(worst["var"], ev)
            assert em <= PROBE_RTOL and ev <= PROBE_RTOL, (n, i, j, em, ev)
        gm, gv = _cotangents(T, len(grp), g)
        want, sc = pro.predict_vjp(dyn, Xs, gm, gv)
        r = _ratio(eng.gp_predict_vjp(gp, Xs, gm, gv).cpu().numpy(), want, sc)
        worst["vjp"] = max(worst["vjp"], r)
        assert r <= BARS["vjp"], (n, grp, r)
    print("one-hot probes n=%d (%d pairs): mean %.2g, var %.2g of the element, VJP ratio %.3g"
          % (n, len(pairs), worst["mean"], worst["var"], worst["vjp"]))


def test_largest_T_is_computed_and_one_more_refused():
    """T = 65535 * 32 rows (a pattern of 97 points repeated): every row right, a row's result independent of its
    position (bitwise), and T + 1 a dimension error of both calls"""
    eng = _engine()
    n, D, E, T = pc.T_LIMIT_CASE[:4]
    f = pc.factors("benign", n, D, E, seed=3)
    C, pat = pc.points("uniform", f, 97, seed=4)
    Xs = pat[np.arange(T) % 97]
    gp = device_gp(C, f)
    mean, var = (a.cpu().numpy() for a in eng.gp_predict(gp, Xs))
    ref = pro.predict(pro.ld_model(C, f["ell"], f["sf2"], f["beta"], f["iK"]), pat)
    r = dict(mean=_ratio(mean[:97], ref["mean"], ref["cmean"]), var=_ratio(var[:97], ref["var"], ref["cvar"]))
    same = np.arange(T) % 97
    assert np.array_equal(mean, mean[same]) and np.array_equal(var, var[same])
    gm, gv = np.ones((T, E)), np.ones((T, E))
    gx = eng.gp_predict_vjp(gp, Xs, gm, gv).cpu().numpy()
    want, sc = pro.predict_vjp(pro.ld_model(C, f["ell"], f["sf2"], f["beta"], f["iK"]), pat, gm[:97], gv[:97])
    r["vjp"] = _ratio(gx[:97], want, sc)
    assert np.array_equal(gx, gx[same])
    assert_bars(r, "T = %d" % T)
    big = np.vstack([Xs, Xs[:1]])
    with pytest.raises(Exception, match="(?i)dim|unsupported"):
        eng.gp_predict(gp, big)
    with pytest.raises(Exception, match="(?i)dim|unsupported"):
        eng.gp_predict_vjp(gp, big, np.ones((T + 1, E)), np.ones((T + 1, E)))
