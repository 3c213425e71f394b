"""CPU checks of the moment-match test infrastructure: the extended-precision oracle (tests/mm_oracle.py) against the
fp64 port of the reference path, against a 40-digit mpmath evaluation in every hard regime, and its directional
derivative against the hand-derived VJP (oracle/staged.py); and the path matrix of tests/mm_cases.py -- every cell
(KS x pass form x chunking x tail x partial octets x taped row splits x setup form x model kind) is reached by a case on
a 132-SM machine (H100 SXM)."""
import numpy as np
import pytest

import mm_cases as mc
import mm_oracle as mo

pytestmark = pytest.mark.skipif(not mo.HAVE_EXTENDED, reason=mo.NEED_EXTENDED)


def _ratio(got, ref, scale):
    return float(np.max(np.abs(mo._ld(got) - ref) / scale))


@pytest.mark.parametrize("n,D,E,kind", [(60, 3, 2, "exact"), (130, 7, 3, "exact"), (90, 13, 2, "mode1")])
def test_oracle_matches_the_fp64_port(n, D, E, kind):
    from oracle import python_port as pp
    d = mc.benign(n, D, E, 1, kind, seed=n)
    ref = mo.moment_match(d["X"], d["ell"], d["sf2"], d["beta"], d["iK"], d["m"][0], d["s"][0], d["mode"])
    iK = d["iK"] if d["iK"] is not None else np.zeros((E, n, n))
    M, S, V = pp.predict_given_factorizations(d["X"], d["ell"], d["sf2"], d["m"][:1], d["s"][0], iK, d["beta"])
    if kind == "mode1":
        S = S - np.diag(d["sf2"] - 1e-6)
    assert _ratio(M[0], ref["M"], ref["cM"]) < 1e-12
    assert _ratio(S, ref["S"], ref["cS"]) < 1e-12
    assert _ratio(V, ref["V"], ref["cV"]) < 1e-12


def _mp_moment_match(d):
    """the same sums at 40 digits, written from the closed form: L'[n,m] = sf2_a sf2_b det(R)^-1/2
    exp(-(p_a.zn^2 + p_b.zm^2)/2 + z'Qz), z = p_a zn + p_b zm, R = s diag(p_a + p_b) + I, Q = R^-1 s / 2"""
    import mpmath as mp
    mp.mp.dps = 40
    X, ell, sf2, beta, iK = d["X"], d["ell"], d["sf2"], d["beta"], d["iK"]
    n, D = X.shape
    E = ell.shape[0]
    m = [mp.mpf(float(v)) for v in d["m"][0]]
    s = mp.matrix(D, D)
    for i in range(D):
        for j in range(D):
            s[i, j] = (mp.mpf(float(d["s"][0][i, j])) + mp.mpf(float(d["s"][0][j, i]))) / 2
    zeta = [[mp.mpf(float(X[k, i])) - m[i] for i in range(D)] for k in range(n)]
    p = [[1 / mp.mpf(float(ell[a, i])) ** 2 for i in range(D)] for a in range(E)]
    M, V, S = [mp.mpf(0)] * E, [[mp.mpf(0)] * E for _ in range(D)], [[mp.mpf(0)] * E for _ in range(E)]
    for a in range(E):
        A = s + mp.diag([1 / v for v in p[a]])
        W = mp.inverse(A)
        c = mp.mpf(float(sf2[a])) / mp.sqrt(mp.det(A) * mp.fprod(p[a]))
        for k in range(n):
            z = mp.matrix(zeta[k])
            t = W * z
            w = c * mp.mpf(float(beta[a, k])) * mp.exp(-(z.T * t)[0] / 2)
            M[a] += w
            for i in range(D):
                V[i][a] += w * t[i]
    for a in range(E):
        for b in range(a, E):
            Rm = s * mp.diag([p[a][i] + p[b][i] for i in range(D)]) + mp.eye(D)
            Q = mp.inverse(Rm) * s / 2
            c = mp.mpf(float(sf2[a])) * mp.mpf(float(sf2[b])) / mp.sqrt(mp.det(Rm))
            T = mp.mpf(0)
            for k in range(n):
                for l in range(n):
                    g = mp.mpf(float(beta[a, k])) * mp.mpf(float(beta[b, l]))
                    if a == b and iK is not None and d["mode"] == 0:
                        g -= mp.mpf(float(iK[a, k, l]))
                    z = mp.matrix([p[a][i] * zeta[k][i] + p[b][i] * zeta[l][i] for i in range(D)])
                    e = -sum(p[a][i] * zeta[k][i] ** 2 + p[b][i] * zeta[l][i] ** 2 for i in range(D)) / 2 + (z.T * Q * z)[0]
                    T += g * c * mp.exp(e)
            S[a][b] = S[b][a] = T + (mp.mpf(float(sf2[a])) if a == b else 0) - M[a] * M[b]
    return M, S, V


@pytest.mark.parametrize("regime", list(mc.REGIMES))
def test_oracle_matches_40_digits_in_every_regime(regime):
    """n = 6, D = 2 (3 for the regimes that need a third dimension), E = 2.  The oracle's own error is a few longdouble
    roundings of the LARGEST PART of an exponent (its parts cancel: up to ~1e3 at short length-scales), so the bar is
    1e-17 of the condition scale per unit of that, capped at 1e-15 -- four decades below what fp64 can resolve."""
    import mpmath as mp
    D = 3 if regime in ("ard_mixed", "s_singular") else 2
    d = mc.REGIMES[regime](6, D, 2, 1, seed=11)
    ref = mo.moment_match(d["X"], d["ell"], d["sf2"], d["beta"], d["iK"], d["m"][0], d["s"][0], d["mode"])
    M, S, V = _mp_moment_match(d)
    zeta = d["X"] - d["m"][0]
    big = max(1.0, float(np.max((zeta / d["ell"][:, None, :]) ** 2)) * D)
    bar = min(1e-17 * big, 1e-15)
    ld = lambda v: np.longdouble(mp.nstr(v, 30))
    for a in range(2):
        assert abs(ld(M[a]) - ref["M"][a]) <= bar * ref["cM"][a]
        for b in range(2):
            assert abs(ld(S[a][b]) - ref["S"][a, b]) <= bar * ref["cS"][a, b], (a, b)
        for i in range(D):
            assert abs(ld(V[i][a]) - ref["V"][i, a]) <= bar * ref["cV"][i, a] + np.longdouble(1e-300)


@pytest.mark.parametrize("regime,n,D,E", [("benign", 40, 3, 2), ("benign", 70, 5, 3), ("s_singular", 50, 6, 2),
                                          ("short_ell", 50, 3, 2), ("scales", 40, 4, 2)])
def test_directional_derivative_matches_the_staged_vjp(regime, n, D, E):
    from oracle import staged as st
    d = mc.benign(n, D, E, 1, seed=n) if regime == "benign" else mc.REGIMES[regime](n, D, E, 1, seed=n)
    rng = np.random.RandomState(n)
    gM, gS, gV = rng.randn(E), rng.randn(E, E), rng.randn(D, E)
    dm, ds = rng.randn(D), rng.randn(D, D)
    ds = 0.5 * (ds + ds.T)
    args = (d["X"], d["ell"], d["sf2"], d["beta"], d["iK"], d["m"][0], d["s"][0])
    want = mo.directional_derivative(*args, dm, ds, gM, gS, gV, d["mode"])
    gm, gs = st.mm_backward_staged(*args, gM, gS, gV, d["mode"])[:2]
    fscale = mo.contraction(mo.moment_match(*args, d["mode"]), gM, gS, gV)[1]
    scale = np.abs(gm * dm).sum() + np.abs(gs * ds).sum() + float(fscale)
    assert abs(float(want) - (gm @ dm + (gs * ds).sum())) <= 1e-9 * scale


def test_solve_logdet_in_extended_precision():
    rng = np.random.RandomState(0)
    A = rng.rand(7, 7)
    A = A @ A.T + 1e-3 * np.eye(7)
    X, ld = mo.solve_logdet(A, np.eye(7))
    assert np.max(np.abs(mo._ld(A) @ X - np.eye(7))) < 1e-14
    assert abs(float(ld) - np.linalg.slogdet(A)[1]) < 1e-10


def test_every_cell_of_the_path_matrix_is_covered_at_132_sms():
    """the matrix is enumerated cell by cell (mm_cases.coverage_cells), so an uncovered cell is a named failure"""
    names = [name for name, _ in mc.coverage_cells()]
    assert len(names) == len(set(names)) == 96
    assert mc.uncovered(132) == []
    # the named shapes run what their comments say
    assert mc.path_of(500, 10, 8, 1, "exact", 132)["rpc"] == 1           # the odd form at a single restart ...
    p = mc.path_of(300, 12, 10, 32, "exact", 132)                          # ... the metric batch: all five row blocks per CTA
    assert p["rpc"] == 5 and p["mixed_cta"] and p["KS"] == 3 and p["setup"] == "split" and p["cs"] == 1
    for KS in (1, 4):
        ns = {c[0] for c in mc.PATH_CASES if (c[1] + 3) // 4 == KS}
        assert {1, 8, 9, 63, 64, 65} <= ns
    for n, D, E, R in mc.SUBSET:
        assert mc.path_of(n, D, E, R, "exact", 132)["forms"]
    assert {frozenset(mc.path_of(*c, "exact", 132)["forms"]) for c in mc.SUBSET} == {frozenset({"paired"}), frozenset({"odd"}),
                                                                                      frozenset({"paired", "odd"})}
    assert {mc.path_of(*c, "exact", 132)["KS"] for c in mc.SUBSET} == {1, 2, 3, 4}


def test_a_removed_case_uncovers_its_cell():
    """the coverage assertion bites: without the three-row-split cases those cells are named"""
    cases = [c for c in mc.PATH_CASES if not (c[0] == 200 and c[3] == 15)]
    assert mc.uncovered(132, cases) == ["KS%d taped, 3 row splits" % KS for KS in (1, 2, 3, 4)]


def test_probe_indices_sit_on_the_boundaries():
    for n in (100, 150, 600):
        for E in (8, 16):
            idx = mc.probe_indices(n, E)
            assert len(set(idx)) == E and all(0 <= i < n for i in idx) and idx[0] == n - 1
            tiles = {i // 8 for i in idx}
            last = (n - 1) // 8
            assert {last, last - 1, last - 2, last - 3} <= tiles          # every tile of the largest tail group (GM = 4)
            assert {63, 64} <= set(idx) or E == 8 and n == 600
            if n == 600:
                assert {511, 512} <= set(idx)
    assert {0, 7, 8, 15, 56, 63, 64, 71, 72} <= set(mc.probe_indices(150, 16))


def test_far_probe_elements_straddle_the_exp_clamp():
    """the probe that pins the exp clamp is not vacuous: it holds elements between 2^-600 and 2^-1008 and below 2^-1008"""
    d = mc.far_probe(100, 3, seed=103)
    E = len(d["idx"])
    lg = [float(mo.log_element(d["X"], d["ell"], d["sf2"], d["m"][0], d["s"][0], a, b, d["idx"][a], d["idx"][b]))
          for a in range(E) for b in range(a + 1, E)]
    ln2 = np.log(2.0)
    assert sum(-1000 * ln2 < v < -620 * ln2 for v in lg) >= 3 and sum(v < -1020 * ln2 for v in lg) >= 3
    assert sum(v > -50 for v in lg) >= 1
