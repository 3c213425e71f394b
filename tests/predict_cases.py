"""Inputs for the predict-family regime tests: factors per regime, test-point families and size cells, chosen so that
every tile edge of predict.cu is reached.

Regimes: tests/fact_cases.py's exact-GP regimes (benign, noise_floor, episodes4/6, duplicates, long_ell, short_ell,
ard_mixed, scales_lo/hi) with the fp64 factors of oracle/python_port, and FITC factors over inducing points
(fitc_benign, fitc_clustered: iK indefinite).  The factors are inputs (zero-padded to ldk), not recomputed on the
device.

Test-point families (``points``): uniform over the data's box; exactly the centres (var ~ sn2: sf2 - k iK k cancels);
the centres + 1e-8; far points where every k* underflows (mean exactly 0, var exactly sf2); data and points offset by
1e4 (only the difference form x - c keeps the bits).

Size cells (``cells_of``): predict.cu stages iK in 16-row chunks (PR_KC), 64-column warps and 256-column j blocks
(PR_JB) over np = pad64(n) and the points in 32-row blocks (PR_TR) on a grid of at most 65535 row blocks.  n on both
sides of the chunk, warp and block edges and a last j block of every width (64, 128, 192, 256), T on the row-block
edges and at the grid limit, D = 1 and D = MAXD, E = MAXE with an output subset, and ldk above pad64(n), as an
appended model has it.
"""
import numpy as np

import fact_cases

PR_KC, PR_JB, PR_TR, MAXD, MAXE = 16, 256, 32, 16, 16
T_MAX = 65535 * PR_TR
REGIMES = fact_cases.REGIMES + ("fitc_benign", "fitc_clustered")
FAMILIES = ("uniform", "rows", "rows_1e-8", "far", "offset_1e4")


def pad64(n):
    return (n + 63) // 64 * 64


def factors(regime, n, D, E, seed=0):
    """-> dict(C [n,D], ell [E,D], sf2 [E], beta [E,n], iK [E,n,n], sn2 [E]) of one regime (FITC: n inducing points
    over 4 n data rows)"""
    from oracle import python_port as pp
    if regime.startswith("fitc_"):
        X, Y, Z, ell, sf2, sn2 = fact_cases.make_fitc("benign" if regime == "fitc_benign" else regime, 4 * n, n, D, E,
                                                      seed)
        iK, beta = pp.fitc_factorizations(X, Z, Y, ell, sf2, sn2)
        return dict(C=Z, ell=ell, sf2=sf2, beta=beta, iK=iK, sn2=sn2)
    X, Y, ell, sf2, sn2 = (a[0] for a in fact_cases.make(regime, n, D, E, seed=seed))
    iK, beta = pp.calculate_factorizations(X, Y, ell, sf2, sn2)
    return dict(C=X, ell=ell, sf2=sf2, beta=beta, iK=iK, sn2=sn2)


def points(family, f, T, seed=0):
    """-> (C, Xs [T,D]): the centres the device sees (offset for offset_1e4) and the test points of a family"""
    C = f["C"]
    rng = np.random.RandomState(seed + 17)
    lo, hi = C.min(0), C.max(0)
    if family == "uniform":
        return C, lo + (hi - lo) * rng.rand(T, C.shape[1])
    if family in ("rows", "rows_1e-8"):
        Xs = C[np.arange(T) % C.shape[0]]
        return C, Xs + 1e-8 if family == "rows_1e-8" else Xs.copy()
    if family == "far":                                 # |x - c| / ell >= 60 in every dimension: exp(-0.5 d2) == 0
        far = hi + 60.0 * f["ell"].max(0) * (1.0 + rng.rand(T, C.shape[1]))
        return C, far
    assert family == "offset_1e4"
    return C + 1e4, lo + (hi - lo) * rng.rand(T, C.shape[1]) + 1e4


def probe_indices(n):
    """every index on either side of a 16-row chunk edge (so of every 64-column warp and 256-column j block edge), and
    0 and n - 1"""
    idx = {0, n - 1}
    for k in range(PR_KC, n, PR_KC):
        idx |= {k - 1, k}
    return sorted(idx)


def probe_pairs(n):
    """(i, j) pairs in which every probe index is an i and a j: i in order, j the list rotated by a third, and i = j
    at the two ends"""
    idx = probe_indices(n)
    m = len(idx)
    return [(idx[a], idx[(a + m // 3) % m]) for a in range(m)] + [(0, 0), (n - 1, n - 1)]


# (n, D, E, T, e0, ne, ldk - pad64(n)) of the size cases at benign numbers: T n^2 ne stays below 3e8 for the oracle
SIZE_CASES = [(1, 1, 1, 1, 0, 1, 0), (15, 3, 2, 31, 0, 2, 0), (16, MAXD, 1, 32, 0, 1, 64), (17, 2, 3, 33, 1, 2, 0),
              (63, 4, 1, 4099, 0, 1, 0), (64, 1, MAXE, 33, 3, 10, 64), (65, 5, 2, 4099, 0, 2, 64),
              (255, 3, 1, 1000, 0, 1, 0), (256, MAXD, MAXE, 31, 0, MAXE, 0), (257, 2, 2, 500, 0, 2, 64),
              (448, 3, 1, 300, 0, 1, 0), (513, 4, MAXE, 40, 12, 4, 64), (2000, 6, 2, 64, 1, 1, 0)]
T_LIMIT_CASE = (64, 1, 1, T_MAX, 0, 1, 0)
# (n, D, E, T) of the regime x family cases
REGIME_SHAPES = [(65, 3, 2, 97), (300, 5, 1, 64)]
PROBE_NS = (65, 448, 513)

REQUIRED_N = (1, 15, 16, 17, 63, 64, 65, 255, 256, 257, 448, 513, 2000)
REQUIRED_T = (1, 31, 32, 33, 4099, T_MAX)


def cells_of(n, D, E, T, e0, ne, ldk_extra):
    out = {"n=%d" % n, "jw=%d" % (pad64(n) - (pad64(n) - 1) // PR_JB * PR_JB)}
    if T in REQUIRED_T:
        out.add("T=%d" % T)
    if D in (1, MAXD):
        out.add("D=%d" % D)
    if E == MAXE and ne < E:
        out.add("E=MAXE subset")
    if ldk_extra > 0:
        out.add("ldk>pad64")
    return out


REQUIRED_CELLS = ({"n=%d" % n for n in REQUIRED_N} | {"T=%d" % T for T in REQUIRED_T}
                  | {"jw=64", "jw=128", "jw=192", "jw=256", "D=1", "D=%d" % MAXD, "E=MAXE subset", "ldk>pad64"})


def covered():
    cells = set()
    for case in SIZE_CASES + [T_LIMIT_CASE]:
        cells |= cells_of(*case)
    return cells
