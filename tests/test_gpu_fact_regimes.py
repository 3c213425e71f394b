"""The factorisation and training kernels of factorize.cu away from the benign regime, against the extended-precision
oracle of tests/fact_oracle.py, in every regime x size of tests/fact_cases.py.

Every device result is judged as |error| / (eps64 * scale) with the oracle's condition scale, so one bar holds from
cond(K) ~ 1 to cond(K) ~ 1e9: L by its backward error |K - L L'| against |L||L'|, beta by its normwise backward error,
iK entry by entry against |K^-1||L||L'||K^-1|, nlml and its gradient against the propagated factor scales.

The scales of L and iK include the Gram entries' own conditioning, |K| (1 + d2): exp(-d2 / 2) turns the rounding
of the scaled squared distance d2 into a relative error of about d2 eps, which dominates at short length-scales.

Bars: about 10x the largest ratio observed on an NVIDIA H100 80GB HBM3 (power limit 700 W):
  pilco_gp_factorize  L 3.4, beta 0.76, iK 1.9 (all regimes and sizes)                    bars 35, 8, 20
  one-hot probes      beta_j against column j of the device's own iK 0.0008               bar 0.01
  pilco_gp_nlml       value 0.011, directional derivative 0.016                          bars 0.12, 0.16
  pilco_fitc_*        iK 1.3e-7, beta 1.5, bound 1.6, derivative (relative) 4.0e-10      bars 1.3e-6, 15, 16, 4e-9
  n = 5088 / 5089     beta 0.096 / 0.13                                                   beta bar
  pilco_gp_append_tri     iK 8.2, beta 15.6 (episodes at sn2 = 1e-6, after 7 appends of 40 rows and after 3 of 100)
                      bars 85, 160; the Schur-complement update of iK it replaced reached about 3e6 for both there
The appended model's ratios run 4-20x above a refactorisation's and grow slowly along a chain.  The nlml, gradient and
FITC scales are looser than the factor scales (most observed ratios sit far below 1), so those bars rest on the
observations alone.  Every ratio is far below 4n, the bound of a backward-stable Cholesky.
"""
import functools

import numpy as np
import pytest
import torch

import fact_cases as fc
import fact_oracle as fo

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not fo.HAVE_EXTENDED, reason=fo.NEED_EXTENDED)]

BAR = dict(L=35.0, beta=8.0, iK=20.0, probe=0.01, nlml=0.12, dnlml=0.16, fitc_iK=1.3e-6, fitc_beta=15.0, bound=16.0,
           dbound_rel=4e-9)
BAR_APPEND = dict(iK=85.0, beta=160.0)
EPS = fo.EPS64


def _engine():
    from pilco_b200 import engine
    return engine


def _np(t):
    torch.cuda.synchronize()
    return t.detach().cpu().numpy()


def _report(tag, **ratios):
    print("RATIO %s %s" % (tag, " ".join("%s=%.3g" % kv for kv in ratios.items())))


@functools.lru_cache(maxsize=None)
def _oracle(regime, n, D, E, B, b, e):
    X, Y, ell, sf2, sn2 = fc.make(regime, n, D, E, B)
    f = fo.gp_factor(X[b], Y[b][:, e], ell[b, e], sf2[b, e], sn2[b, e])
    return f, fo.gp_scales(f, X[b], ell[b, e])


def _L_ratio(K, Lhat, LL):
    Lh = fo._x(np.tril(Lhat))
    return fo.max_ratio((K - Lh @ Lh.T).astype(np.float64), LL)


def _judge(tag, f, sc, y, iK, beta, L=None, bar=BAR):
    r = dict(iK=fo.max_ratio(iK - f["iK"].astype(np.float64), sc["iK"]) if iK is not None else 0.0,
             beta=fo.beta_backward(f["K"], beta, y) / EPS)
    if L is not None:
        r["L"] = _L_ratio(f["K"], L, sc["LL"])
    fwd = float(np.abs(beta - f["beta"].astype(np.float64)).max() / np.abs(f["beta"].astype(np.float64)).max())
    _report(tag, fwd_beta=fwd, **r)
    for k, v in r.items():
        assert v < bar[k], (tag, k, v)


@pytest.mark.parametrize("case", fc.FACT_CASES, ids=lambda c: "%s-n%d-D%d-E%d-B%d" % c)
def test_gp_factorize_regimes(case):
    regime, n, D, E, B = case
    engine = _engine()
    X, Y, ell, sf2, sn2 = fc.make(regime, n, D, E, B)
    sq = (lambda a: a[0]) if B == 1 else (lambda a: a)
    gp = engine.gp_factorize(sq(X), sq(Y), sq(ell), sq(sf2), sq(sn2))
    assert not _np(gp.info).any()
    ldw = engine.pad_n(n)
    iK = _np(gp.iK).reshape(B, E, ldw, ldw)
    beta = _np(gp.beta).reshape(B, E, n)
    L = _np(gp.fact_ws[:B * E * ldw * ldw]).reshape(B, E, ldw, ldw)
    assert np.all(iK[:, :, n:, :] == 0) and np.all(iK[:, :, :, n:] == 0)
    for b in range(B):
        for e in range(E):
            f, sc = _oracle(regime, n, D, E, B, b, e)
            _judge("factorize %s n=%d b=%d e=%d" % (regime, n, b, e), f, sc, Y[b][:, e], iK[b, e, :n, :n],
                   beta[b, e], L[b, e, :n, :n])


@pytest.mark.parametrize("regime,n", [("benign", 129), ("episodes6", 129), ("noise_floor", 545), ("duplicates", 513)])
def test_one_hot_probes(regime, n):
    """Y = one-hot columns at j in {0, 31, 32, n-1}: beta_j = (K + sn2 I)^-1 e_j is column j of iK, so the blocked
    substitution of chol_solve_vec_kernel meets tri_inverse + GEMM block edge by block edge"""
    engine = _engine()
    X, _, ell, sf2, sn2 = fc.make(regime, n, 5, 1)
    js = [0, 31, 32, n - 1]
    E = len(js)
    Y = np.zeros((n, E))
    Y[js, np.arange(E)] = 1.0
    gp = engine.gp_factorize(X[0], Y, np.repeat(ell[0], E, 0), np.repeat(sf2[0], E), np.repeat(sn2[0], E))
    assert not _np(gp.info).any()
    iK, beta = _np(gp.iK), _np(gp.beta)
    f, sc = _oracle(regime, n, 5, 1, 1, 0, 0)
    for e, j in enumerate(js):
        r_self = fo.max_ratio(beta[e] - iK[e, :n, j], sc["iK"][:, j])
        r_true = fo.max_ratio(beta[e] - f["iK"][:, j].astype(np.float64), sc["iK"][:, j])
        _report("probe %s n=%d j=%d" % (regime, n, j), self=r_self, true=r_true)
        assert r_self < BAR["probe"] and r_true < BAR["iK"]


def _direction(D, seed):
    rng = np.random.RandomState(seed)
    return rng.randn(D + 2)


@pytest.mark.parametrize("case", fc.NLML_CASES, ids=lambda c: "%s-n%d-D%d-E%d" % c)
def test_gp_nlml_regimes(case):
    """pilco_gp_nlml: the value and the gradient along a random direction of (ell, sf2, sn2), against the closed form
    in longdouble and the complex-step derivative"""
    regime, n, D, E = case
    engine = _engine()
    X, Y, ell, sf2, sn2 = fc.make(regime, n, D, E)
    ev = engine.GpNlml(X[0], Y[0], 1)
    nlml, g_ell, g_sf2, g_sn2, bad = ev(ell, sf2, sn2)
    assert not bad.any()
    for e in range(E):
        o = fo.gp_nlml(X[0], Y[0][:, e], ell[0, e], sf2[0, e], sn2[0, e])
        v = _direction(D, e)
        # directions scaled to the parameters, so every component moves by a comparable relative amount
        vs = v * np.r_[ell[0, e], sf2[0, e], sn2[0, e]]
        d_dev = vs @ np.r_[g_ell[0, e], g_sf2[0, e], g_sn2[0, e]]
        d_cs = fo.gp_nlml_cs(X[0], Y[0][:, e], ell[0, e], sf2[0, e], sn2[0, e], vs)
        assert abs(float(d_cs - vs @ o["grad"])) <= 1e-3 * EPS * float(np.abs(vs) @ o["c_grad"])   # oracle vs oracle
        r = dict(nlml=fo.max_ratio(nlml[0, e] - float(o["nlml"]), o["c_nlml"]),
                 dnlml=fo.max_ratio(d_dev - float(d_cs), np.abs(vs) @ o["c_grad"]))
        _report("nlml %s n=%d e=%d" % (regime, n, e), **r)
        for k, val in r.items():
            assert val < BAR[k], (k, val)


@pytest.mark.parametrize("case", fc.FITC_CASES, ids=lambda c: "%s-N%d-M%d-D%d-E%d" % c)
def test_fitc_regimes(case):
    """pilco_fitc_factorize (iK, beta) and pilco_fitc_nlml (bound, derivative along (ell, sf2, sn2, Z))"""
    regime, N, M, D, E = case
    engine = _engine()
    X, Y, Z, ell, sf2, sn2 = fc.make_fitc(regime, N, M, D, E)
    gp = engine.fitc_factorize(X, Z, Y, ell, sf2, sn2)
    assert not _np(gp.info).any()
    iK, beta = _np(gp.iK)[:, :M, :M], _np(gp.beta)
    ev = engine.FitcNlml(X, Y, M, 1)
    Zb = np.broadcast_to(Z, (1, E, M, D))
    val, g_ell, g_sf2, g_sn2, g_Z, bad = ev(Zb, ell[None], sf2[None], sn2[None])
    assert not bad.any()
    for e in range(E):
        o = fo.fitc_factor(X, Z, Y[:, e], ell[e], sf2[e], sn2[e])
        r = dict(fitc_iK=fo.max_ratio(iK[e] - o["iK"].astype(np.float64), o["c_iK"]),
                 fitc_beta=fo.max_ratio(beta[e] - o["beta"].astype(np.float64), o["c_beta"]))
        if M <= 65:                                             # the bound: Cholesky factorisations of M x M only
            bnd, c_bnd = fo.fitc_bound(X, Y[:, e], Z, ell[e], sf2[e], sn2[e])
            rng = np.random.RandomState(e)
            v_ell, v_sf2, v_sn2, v_Z = rng.randn(D) * ell[e], rng.randn() * sf2[e], rng.randn() * sn2[e], \
                0.1 * rng.randn(M, D)
            d_cs = float(fo.fitc_bound_cs(X, Y[:, e], Z, ell[e], sf2[e], sn2[e], v_ell, v_sf2, v_sn2, v_Z))
            terms = np.r_[v_ell * g_ell[0, e], v_sf2 * g_sf2[0, e], v_sn2 * g_sn2[0, e], (v_Z * g_Z[0, e]).ravel()]
            r["bound"] = fo.max_ratio(val[0, e] - float(bnd), c_bnd)
            r["dbound_rel"] = abs(terms.sum() - d_cs) / np.abs(terms).sum()
        _report("fitc %s N=%d M=%d e=%d" % (regime, N, M, e), **r)
        for k, v in r.items():
            assert v < BAR[k], (k, v)


# ---- failure reporting and batch independence ------------------------------------------------------------------------
def _indefinite_batch(n=100, D=3, E=2, B=3, bad=1):
    X, Y, ell, sf2, sn2 = fc.make("benign", n, D, E, B)
    sn2 = sn2.copy()
    sn2[bad] = -0.1 * sf2[bad]            # K - 0.1 sf2 I: a smooth Gram matrix has eigenvalues far below 0.1 sf2
    return X, Y, ell, sf2, sn2


def test_failure_flags_the_failing_batch_element_only():
    """info bit 1 marks exactly the indefinite batch element; every other element is bitwise what an unbatched call
    gives (gp_factorize, gp_nlml and GpNlml's ``bad`` flag, which the training loop turns into its BIG loss)"""
    engine = _engine()
    X, Y, ell, sf2, sn2 = _indefinite_batch()
    gp = engine.gp_factorize(X, Y, ell, sf2, sn2)
    assert list(_np(gp.info)) == [0, 2, 0]
    iK, beta = _np(gp.iK), _np(gp.beta)
    for b in (0, 2):
        one = engine.gp_factorize(X[b], Y[b], ell[b], sf2[b], sn2[b])
        assert int(_np(one.info)[0]) == 0
        assert np.array_equal(iK[b], _np(one.iK)) and np.array_equal(beta[b], _np(one.beta))
    # gp_nlml shares X, Y across the batch: the batch runs over hyper-parameter sets
    ev = engine.GpNlml(X[0], Y[0], 3)
    out = ev(ell, sf2, sn2)
    assert list(out[-1]) == [False, True, False]
    assert list(_np(ev.info)) == [0, 2, 0]
    for b in (0, 2):
        one = engine.GpNlml(X[0], Y[0], 1)(ell[b:b + 1], sf2[b:b + 1], sn2[b:b + 1])
        assert not one[-1].any()
        for a, c in zip(out[:4], one[:4]):
            assert np.array_equal(a[b], c[0])


def test_fitc_nlml_failure_flags_the_failing_batch_element_only():
    engine = _engine()
    X, Y, Z, ell, sf2, sn2 = fc.make_fitc("benign", 200, 33, 3, 1)
    B, E, M, D = 3, 1, 33, 3
    Zb = np.broadcast_to(Z, (B, E, M, D)).copy()
    ellb, sf2b, sn2b = np.repeat(ell[None], B, 0), np.repeat(sf2[None], B, 0), np.repeat(sn2[None], B, 0)
    sn2b[1] = -10.0 * sf2b[1]             # nu < 0 everywhere: I + V diag(1/nu) V' is indefinite
    ev = engine.FitcNlml(X, Y, M, B)
    out = ev(Zb, ellb, sf2b, sn2b)
    assert list(out[-1]) == [False, True, False]
    for b in (0, 2):
        one = engine.FitcNlml(X, Y, M, 1)(Zb[b:b + 1], ellb[b:b + 1], sf2b[b:b + 1], sn2b[b:b + 1])
        assert not one[-1].any()
        for a, c in zip(out[:5], one[:5]):
            assert np.array_equal(a[b], c[0])


@pytest.mark.parametrize("n", [65, 513])
def test_results_do_not_depend_on_the_batch(n):
    """batch element b of a B = 3 call is bitwise the B = 1 call (single-CTA and multi-CTA Cholesky)"""
    engine = _engine()
    X, Y, ell, sf2, sn2 = fc.make("episodes4", n, 5, 2, 3)
    gp = engine.gp_factorize(X, Y, ell, sf2, sn2)
    ev = engine.GpNlml(X[1], Y[1], 3)
    out = ev(ell, sf2, sn2)
    for b in range(3):
        one = engine.gp_factorize(X[b], Y[b], ell[b], sf2[b], sn2[b])
        assert np.array_equal(_np(gp.iK)[b], _np(one.iK)) and np.array_equal(_np(gp.beta)[b], _np(one.beta))
        o1 = engine.GpNlml(X[1], Y[1], 1)(ell[b:b + 1], sf2[b:b + 1], sn2[b:b + 1])
        for a, c in zip(out[:4], o1[:4]):
            assert np.array_equal(a[b], c[0])


# ---- incremental set_data ---------------------------------------------------------------------------------------------
def _episode_problem(n, sn2, D=5, E=2, seed=0):
    rng = np.random.RandomState(seed)
    X = fc.episodes(n, D, rng)
    Y = 0.1 * np.sin(3.0 * X).dot(rng.rand(D, E))
    return X, Y, np.ones((E, D)) + 0.1 * rng.rand(E, D), np.ones(E), sn2 * np.ones(E)


def _judge_model(tag, gp, X, Y, ell, sf2, sn2):
    n = gp.n
    iK, beta = _np(gp.iK), _np(gp.beta)
    assert np.all(iK[:, n:, :] == 0) and np.all(iK[:, :, n:] == 0)
    for e in range(gp.E):
        f = fo.gp_factor(X[:n], Y[:n, e], ell[e], sf2[e], sn2[e])
        _judge("%s n=%d e=%d" % (tag, n, e), f, fo.gp_scales(f, X[:n], ell[e]), Y[:n, e], iK[e, :n, :n], beta[e], bar=BAR_APPEND)


@pytest.mark.parametrize("sn2", [1e-2, 1e-4, 1e-6])
@pytest.mark.parametrize("n0,k,steps", [(40, 40, 8), (300, 100, 3)], ids=["8x40", "300+3x100"])
def test_gp_append_chain(n0, k, steps, sn2):
    """PILCO's episode pattern: rows appended episode by episode, each appended model judged against the oracle by the
    factor scales of a refactorisation (300 + 3 x 100 crosses the multi-CTA Cholesky size on the way)"""
    engine = _engine()
    n = n0 + k * steps
    X, Y, ell, sf2, sn2v = _episode_problem(n, sn2, seed=int(-np.log10(sn2)))
    gp = engine.gp_factorize(X[:n0], Y[:n0], ell, sf2, sn2v)
    for s in range(1, steps + 1):
        n1 = n0 + k * s
        gp = engine.gp_append(gp, X[:n1], Y[:n1])
        assert int(_np(gp.info)[0]) == 0 and gp.n == n1 and gp.appends == s
        _judge_model("append sn2=%g step=%d" % (sn2, s), gp, X, Y, ell, sf2, sn2v)


def test_gp_append_multi_cta_schur():
    """k >= 512 appended rows: the Cholesky of the new rows' Schur complement takes the multi-CTA path"""
    engine = _engine()
    X, Y, ell, sf2, sn2 = _episode_problem(620, 1e-4, seed=7)
    gp = engine.gp_append(engine.gp_factorize(X[:100], Y[:100], ell, sf2, sn2), X, Y)
    assert int(_np(gp.info)[0]) == 0
    _judge_model("append k=520", gp, X, Y, ell, sf2, sn2)


@pytest.mark.parametrize("sn2", [1e-4, 1.1e-6])
def test_mgpr_set_data_chain_predicts_like_a_fresh_model(sn2):
    """MGPR.set_data episode by episode (appends up to MAX_APPENDS, then a refactorisation) predicts what a fresh MGPR
    of the same data predicts: the appended model's moment-match error against the oracle is within 10x the fresh
    model's own, plus the moment-match bar"""
    import mm_oracle as mo
    from pilco.models import MGPR
    from util import make_input
    T, n_ep = 40, 9
    X, Y, ell, sf2, sn2v = _episode_problem(T * n_ep, sn2, seed=3)
    m, s = make_input(5, seed=2, scale=0.05)
    m = X[0:1] + 0.01

    def fixed(mg):
        for i, mod in enumerate(mg.models):
            mod.kernel.lengthscales.assign(ell[i]); mod.kernel.variance.assign(sf2[i]); mod.likelihood.variance.assign(sn2v[i])
    mg = MGPR((X[:T], Y[:T])); fixed(mg)
    mg.predict_on_noisy_inputs(m, s)
    for j in range(2, n_ep + 1):
        mg.set_data((X[:T * j], Y[:T * j]))
        out = mg.predict_on_noisy_inputs(m, s)
        assert mg.last_update == "append"
    fresh = MGPR((X, Y)); fixed(fresh)
    ref = fresh.predict_on_noisy_inputs(m, s)
    noise = np.array([float(mod.likelihood.variance) for mod in mg.models])
    fs = [fo.gp_factor(X, Y[:, e], ell[e], sf2[e], noise[e]) for e in range(2)]
    tr = mo.moment_match(X, ell, sf2, np.stack([f["beta"] for f in fs]), np.stack([f["iK"] for f in fs]), m[0], s)
    for name, a, b, t, c in zip("MSV", out, ref, (tr["M"], tr["S"], tr["V"]), (tr["cM"], tr["cS"], tr["cV"])):
        a, b = np.asarray(a).reshape(t.shape), np.asarray(b).reshape(t.shape)
        err_a, err_b = np.abs(a - t.astype(np.float64)), np.abs(b - t.astype(np.float64))
        _report("mgpr chain sn2=%g %s" % (sn2, name), chain=float((err_a / (EPS * c.astype(np.float64))).max()),
                fresh=float((err_b / (EPS * c.astype(np.float64))).max()))
        assert np.all(err_a <= 10 * err_b + 64 * EPS * c.astype(np.float64)), name


# ---- sizes above the old shared-memory limit of the substitution -----------------------------------------------------
@pytest.mark.parametrize("n", [5088, 5089])
def test_gp_factorize_large_n(n):
    """chol_solve_vec_kernel holds n doubles of dynamic shared memory: past 48 KB it needs the opt-in attribute"""
    engine = _engine()
    X, Y, ell, sf2, sn2 = fc.make("benign", n, 3, 1)
    gp = engine.gp_factorize(X[0], Y[0], ell[0], sf2[0], sn2[0], need_iK=False)
    assert not _np(gp.info).any()
    beta = _np(gp.beta)[0]
    r = fo.beta_backward_chunked(X[0], ell[0, 0], sf2[0, 0], sn2[0, 0], beta, Y[0][:, 0]) / EPS
    _report("factorize n=%d" % n, beta=r)
    assert r < BAR["beta"]
