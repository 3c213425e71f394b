"""Inputs for the factorisation tests: regimes x sizes, chosen so that every code path edge of factorize.cu is reached.

Regimes (one exact-GP problem per call, ``make(regime, n, D, E, B, seed)`` -> X [B,n,D], Y [B,n,E], ell [B,E,D],
sf2 [B,E], sn2 [B,E]; different hyper-parameters per output and per batch element):
  benign        tests/util.make_gp_problem's family: X in [0,1]^D, ell in [1,2], sf2 in [1,2], sn2 = 1e-2 (cond ~1e4)
  noise_floor   the same at sn2 = 1e-6, the Softplus floor of MGPR's likelihood variance
  episodes4/6   rows as PILCO collects them -- 40-step random walks from one shared x0 -- at sn2 = 1e-4 / 1e-6
  duplicates    every row present twice, exactly
  long_ell      ell 30x the data spread: numerically low rank, the pivots fall to sn2
  short_ell     ell = 1e-2: almost every off-diagonal entry underflows, K is close to diagonal
  ard_mixed     ell from 1e-2 to 1e2 across the dimensions
  scales_lo/hi  sf2 and Y at 1e-4 / at 1e4
FITC (``make_fitc``): benign inducing points, and ``fitc_clustered``: inducing points in near-duplicate clusters, so
Kmm + 1e-6 I is nearly singular.

The size cells (``cells_of``): the FB = 32 block and pad64 edges (n = 1, 2, 31-33, 63-65, 127-129), the single-CTA /
multi-CTA Cholesky switch at CHOL_MULTI_N = 512 (511 / 512), a multi-CTA last block one row wide and panel rows of
256 k + 1 crossing a CTA edge (513, 545), D = 1 and D = MAXD, E > 1, B = 3, FITC with M = 1, 33, 65 and M >= 512.
"""
import numpy as np

FB, CHOL_MULTI_N, PANEL_ROWS, MAXD = 32, 512, 256, 16
REGIMES = ("benign", "noise_floor", "episodes4", "episodes6", "duplicates", "long_ell", "short_ell", "ard_mixed",
           "scales_lo", "scales_hi")
HARD = REGIMES[1:]


def episodes(n, D, rng, T=40, step=0.05, jitter=0.01):
    """rows of ceil(n / T) episodes: random walks of T steps from one shared x0 (+ jitter), first n rows"""
    x0 = rng.rand(D)
    eps = [x0 + jitter * rng.randn(1, D) + np.cumsum(step * rng.randn(T, D), 0) for _ in range((n + T - 1) // T)]
    return np.vstack(eps)[:n]


def _one(regime, n, D, E, rng):
    X = rng.rand(n, D)
    ell = 1.0 + rng.rand(E, D)
    sf2 = 1.0 + rng.rand(E)
    sn2 = 1e-2 * np.ones(E)
    ys = 1.0
    if regime == "noise_floor":
        sn2 = 1e-6 * np.ones(E)
    elif regime in ("episodes4", "episodes6"):
        X = episodes(n, D, rng)
        ell, sf2 = np.ones((E, D)) + 0.1 * rng.rand(E, D), np.ones(E) + 0.1 * rng.rand(E)
        sn2 = (1e-4 if regime == "episodes4" else 1e-6) * np.ones(E)
    elif regime == "duplicates":
        base = rng.rand((n + 1) // 2, D)
        X = np.vstack([base, base])[:n]
        sn2 = 1e-4 * np.ones(E)
    elif regime == "long_ell":
        ell = 30.0 * (1.0 + 0.1 * rng.rand(E, D))
        sn2 = 1e-6 * np.ones(E)
    elif regime == "short_ell":
        ell = 1e-2 * (1.0 + 0.1 * rng.rand(E, D))
    elif regime == "ard_mixed":
        ell = np.logspace(-2, 2, D)[None, :] * (1.0 + 0.1 * rng.rand(E, D))
        sn2 = 1e-4 * np.ones(E)
    elif regime in ("scales_lo", "scales_hi"):
        ys = 1e-4 if regime == "scales_lo" else 1e4
        sf2, sn2 = ys * sf2, ys * sn2
    A = rng.rand(D, E)
    Y = ys * (np.sin(3.0 * X).dot(A) / D + 1e-3 * (rng.rand(n, E) - 0.5))
    return X, Y, ell, sf2, sn2


def make(regime, n, D, E, B=1, seed=0):
    """-> X [B,n,D], Y [B,n,E], ell [B,E,D], sf2 [B,E], sn2 [B,E]"""
    rng = np.random.RandomState(seed * 1000 + n)
    parts = [_one(regime, n, D, E, rng) for _ in range(B)]
    return tuple(np.stack([p[i] for p in parts]) for i in range(5))


# (regime, n, D, E, B) of the pilco_gp_factorize cases
FACT_CASES = ([("benign", n, 3, 1, 1) for n in (1, 2, 31, 32, 33, 63, 64, 65, 127, 128, 129)]
              + [("benign", n, 5, 1, 1) for n in (511, 512, 513, 545)]
              + [("benign", 100, 1, 2, 1), ("benign", 100, MAXD, 2, 1), ("benign", 65, 4, 3, 3)]
              + [("noise_floor", 33, 3, 2, 1), ("noise_floor", 129, 5, 1, 1), ("noise_floor", 513, 5, 1, 1),
                 ("episodes4", 64, 5, 1, 1), ("episodes4", 512, 5, 1, 1),
                 ("episodes6", 65, 5, 2, 1), ("episodes6", 545, 5, 1, 1),
                 ("duplicates", 32, 3, 1, 1), ("duplicates", 128, 3, 1, 3), ("duplicates", 511, 3, 1, 1),
                 ("long_ell", 63, 3, 1, 1), ("long_ell", 513, 3, 1, 1),
                 ("short_ell", 31, 3, 1, 1), ("short_ell", 545, 3, 1, 1),
                 ("ard_mixed", 127, MAXD, 1, 1), ("ard_mixed", 512, 6, 1, 1),
                 ("scales_lo", 65, 3, 2, 1), ("scales_hi", 129, 3, 1, 1), ("scales_hi", 513, 3, 1, 1)])

# (regime, n, D, E) of the pilco_gp_nlml cases (value and directional derivative)
NLML_CASES = [("benign", 33, 3, 2), ("noise_floor", 129, 4, 1), ("episodes6", 200, 5, 1), ("duplicates", 64, 3, 1),
              ("long_ell", 65, 3, 1), ("short_ell", 31, 3, 1), ("ard_mixed", 100, 6, 1), ("scales_hi", 63, 3, 1),
              ("benign", 513, 5, 1), ("episodes4", 545, 5, 1)]

# (regime, N, M, D, E) of the FITC cases
FITC_CASES = [("benign", 200, 1, 3, 1), ("benign", 200, 33, 3, 2), ("benign", 300, 65, 4, 1),
              ("fitc_clustered", 200, 33, 3, 1), ("fitc_clustered", 300, 65, 4, 1), ("benign", 600, 520, 3, 1)]


def make_fitc(regime, N, M, D, E, seed=0):
    """-> X [N,D], Y [N,E], Z [M,D], ell [E,D], sf2 [E], sn2 [E]"""
    rng = np.random.RandomState(seed * 1000 + N + M)
    X = rng.rand(N, D)
    Y = np.sin(3.0 * X).dot(rng.rand(D, E)) / D + 1e-3 * (rng.rand(N, E) - 0.5)
    if regime == "fitc_clustered":
        c = rng.rand((M + 2) // 3, D)
        Z = (np.repeat(c, 3, axis=0) + 1e-4 * rng.randn(3 * c.shape[0], D))[:M]
    else:
        Z = rng.rand(M, D)
    return X, Y, Z, 1.0 + rng.rand(E, D), 1.0 + rng.rand(E), 1e-2 * np.ones(E)


def cells_of(n=None, D=None, E=None, B=None, M=None):
    """the size cells one factorisation of these sizes reaches"""
    out = set()
    for tag, m in (("n", n), ("M", M)):
        if m is None:
            continue
        if m <= 2:
            out.add("%s=%d" % (tag, m))
        if m >= 31 and m % FB in (31, 0, 1) and m < CHOL_MULTI_N:
            out.add("%s:FB%+d" % (tag, (m % FB) - FB if m % FB == 31 else m % FB))
        if m >= 63 and m % 64 in (63, 0, 1) and m < CHOL_MULTI_N:
            out.add("%s:pad64%+d" % (tag, (m % 64) - 64 if m % 64 == 63 else m % 64))
        if m == CHOL_MULTI_N - 1:
            out.add("%s:single_cta_top" % tag)
        if m >= CHOL_MULTI_N:
            out.add("%s:multi_cta" % tag)
            if tag == "n" and m % FB == 1:
                out.add("n:multi_last_block_1")
            if tag == "n" and any((m - t0) % PANEL_ROWS == 1 and m - t0 > PANEL_ROWS for t0 in range(FB, m, FB)):
                out.add("n:panel_256k+1")
    if D == 1:
        out.add("D=1")
    if D == MAXD:
        out.add("D=MAXD")
    if E is not None and E > 1:
        out.add("E>1")
    if B == 3:
        out.add("B=3")
    return out


REQUIRED_CELLS = ({"n=1", "n=2", "n:FB-1", "n:FB+0", "n:FB+1", "n:pad64-1", "n:pad64+0", "n:pad64+1",
                   "n:single_cta_top", "n:multi_cta", "n:multi_last_block_1", "n:panel_256k+1",
                   "D=1", "D=MAXD", "E>1", "B=3"}
                  | {"M=1", "M:FB+1", "M:pad64+1", "M:multi_cta"})


def covered():
    cells = set()
    for _, n, D, E, B in FACT_CASES:
        cells |= cells_of(n=n, D=D, E=E, B=B)
    for _, N, M, D, E in FITC_CASES:
        cells |= cells_of(M=M, D=D, E=E)
    return cells
