"""Cases for the moment-match kernels: numerical REGIMES (what the numbers look like) x kernel PATHS (which branch of
the setup / tile / taped kernels a shape runs), and ``path_of``: a statement of the path a case takes on a machine of
``nsm`` SMs, derived from the launch decisions of the library itself (tests/host_harness/layout_harness.cpp compiles
``mm_tile_rpc``, ``mm_tape_splits_on`` and ``mm_setup_is_fused`` for the host) and the loop bounds of
``mm_tile_body_m16`` / ``tile_sweep_m16`` / ``mm_tape_body_m16``."""
import atexit
import ctypes
import functools
import os
import shutil
import subprocess
import tempfile

import numpy as np

from util import ROOT, make_gp_problem, make_input

TILE_CM = 512                                   # columns staged per chunk (mm_kernels.cuh)
GM = {1: 4, 2: 4, 3: 3, 4: 2}                   # column tiles per group of tile_sweep_m16, by KS
KINDS = ("exact", "mode1")                      # exact GP with its inverse (trace term, no hc) | RBF-policy mode (hc)


@functools.lru_cache(maxsize=None)
def harness():
    tmp = tempfile.mkdtemp(prefix="mm_cases_")
    atexit.register(shutil.rmtree, tmp, ignore_errors=True)
    so = os.path.join(tmp, "layout_harness.so")
    subprocess.check_call(["g++", "-O1", "-shared", "-fPIC", "-x", "c++", "-I/usr/local/cuda/include", "-o", so,
                           os.path.join(ROOT, "tests", "host_harness", "layout_harness.cpp")])
    return ctypes.CDLL(so)


def path_of(n, D, E, R, kind, nsm):
    """Which branches the forward and the taped moment match of shape (n, D, E) x R restarts run on ``nsm`` SMs."""
    h = harness()
    KS, np_, P = (D + 3) // 4, (n + 63) // 64 * 64, E * (E + 1) // 2
    NB, NO, NS = np_ // 64, (n + 7) // 8, np_ // 8
    rpc = min(h.launch_tile_rpc(NB, P, R, nsm), NB)
    # forward, off-diagonal pairs (mm_tile_body_m16): passes of two row blocks, an odd last block as octet pairs
    forms, act1_false, mixed_cta = set(), set(), False
    for rb0 in range(0, NB, rpc) if E > 1 else ():
        rb1 = min(rb0 + rpc, NB)
        mixed_cta |= (rb1 - rb0) % 2 == 1 and rb1 - rb0 >= 3
        for rb in range(rb0, rb1, 2):
            odd = rb + 1 >= rb1
            for w in range(4 if odd else 8):
                oct0, ostep = (rb * 8 + 2 * w, 1) if odd else (rb * 8 + w, 8)
                if 8 * oct0 < n:
                    forms.add("odd" if odd else "paired")
                    if not 8 * (oct0 + ostep) < n:
                        act1_false.add("odd" if odd else "paired")
    # column chunks and the tail group of each chunk's sweep (tile_sweep_m16)
    ncol8, CM = NO * 8, min(np_, TILE_CM)
    tails = set()
    for c0 in range(0, ncol8, CM):
        cend = min(ncol8 - c0, min(np_ - c0, CM))
        tails.add((cend // 8) % GM[KS])
    # taped kernel (mm_tape_body_m16): row splits, and a pass whose second block of octets is past the last row
    cs = h.launch_tape_splits(n, P, R, nsm)
    GW = 8 * cs
    npass = (NS + 2 * GW - 1) // (2 * GW)
    second_past = any(sidx * 8 + 2 * ps * GW < NO <= sidx * 8 + 2 * ps * GW + GW
                      for sidx in range(cs) for ps in range(npass))
    return dict(KS=KS, rpc=rpc, forms=frozenset(forms), mixed_cta=mixed_cta, act1_false=frozenset(act1_false),
                chunks=(ncol8 + CM - 1) // CM, tails=frozenset(tails), partial_octet=n % 8 != 0,
                cs=cs, tape_second_past=second_past, ones_column_free=KS % 2 == 1,
                setup="fused" if h.launch_setup_fused(E + P, R, nsm) else "split", spilling_stage1=D > 12, kind=kind)


# (n, D, E, R, kind).  E = 3, R = 22 gives pairs x restarts = 132: every SM a CTA, so a CTA takes all row blocks of its pair.
DK = {1: 3, 2: 7, 3: 10, 4: 14}


def _path_cases():
    cases = []
    for KS in (1, 2, 3, 4):
        D = DK[KS]
        # three row blocks per CTA: a paired pass and an odd pass; 17 .. 20 column tiles give every tail length, 17 and
        # 19 an odd count of live octets in the last block (act[1] false in the odd pass), n % 8 in {1, 7, 0}
        for i, n in enumerate(((129, 143, 152, 153), (129, 143, 152, 153), (137, 145, 159), (129, 143))[KS - 1]):
            cases.append((n, 16 if (KS == 4 and i == 0) else D, 3, 22, "mode1" if i == 1 else "exact"))
        # two row blocks per CTA, the second one partly filled: paired passes only, act[1] false in the paired form
        cases.append((100, D, 3, 22, "exact"))
        # one row block (odd passes only, fused setup): the smallest and the block-boundary sizes
        for n in ((1, 8, 9, 63, 64, 65) if KS in (1, 4) else (9, 63)):
            cases.append((n, 16 if (KS == 4 and n == 63) else D, 2, 1, "mode1" if n == 9 else "exact"))
        cases.append((520, D, 3, 22, "exact"))            # two column chunks, nine row blocks per CTA (4 paired + 1 odd)
        cases.append((200, D, 3, 15, "exact"))            # taped: three row splits
        cases.append((257, D, 2, 1, "mode1" if KS == 2 else "exact"))   # taped: four row splits
    cases.append((600, 3, 2, 1, "exact"))                  # two chunks, one row block per CTA, single restart
    return cases


PATH_CASES = _path_cases()
# the subset every regime runs at: all four KS, the paired, the odd and the mixed form, fused and split setup
SUBSET = [(129, 3, 3, 22), (100, 7, 3, 22), (63, 7, 2, 1), (137, 10, 3, 22), (65, 14, 2, 1), (143, 14, 3, 22)]
# shapes of the batch-size test: five row blocks, restart 0 at R = 1 (rpc 1, fused setup), 8 (rpc 1, two-stage setup),
# 18 (rpc 2) and 22 (rpc 5)
BATCH_SHAPES = [(300, DK[KS], 3) for KS in (1, 2, 3, 4)]
BATCH_R = (1, 8, 18, 22)


def coverage_cells():
    """The cells of the path matrix, each as (name, predicate over a path dict)."""
    cells = []
    for KS in (1, 2, 3, 4):
        is_ks = lambda p, KS=KS: p["KS"] == KS
        for form in ("paired", "odd"):
            cells.append(("KS%d forward %s only" % (KS, form), lambda p, f=is_ks, form=form: f(p) and p["forms"] == {form}))
            cells.append(("KS%d forward %s, act[1] false" % (KS, form),
                          lambda p, f=is_ks, form=form: f(p) and form in p["act1_false"]))
            cells.append(("KS%d forward %s, several chunks" % (KS, form),
                          lambda p, f=is_ks, form=form: f(p) and form in p["forms"] and p["chunks"] > 1))
            for tail in range(GM[KS]):
                cells.append(("KS%d forward %s, tail of %d tiles" % (KS, form, tail),
                              lambda p, f=is_ks, form=form, tail=tail: f(p) and form in p["forms"] and tail in p["tails"]
                              and p["chunks"] == 1))
        cells.append(("KS%d forward mixed (odd rpc >= 3)" % KS, lambda p, f=is_ks: f(p) and p["mixed_cta"]))
        cells.append(("KS%d n %% 8 != 0" % KS, lambda p, f=is_ks: f(p) and p["partial_octet"]))
        for cs in (1, 2, 3, 4):
            cells.append(("KS%d taped, %d row splits" % (KS, cs), lambda p, f=is_ks, cs=cs: f(p) and p["cs"] == cs))
        for setup in ("fused", "split"):
            cells.append(("KS%d setup %s" % (KS, setup), lambda p, f=is_ks, s=setup: f(p) and p["setup"] == s))
        for kind in KINDS:
            cells.append(("KS%d %s" % (KS, kind), lambda p, f=is_ks, k=kind: f(p) and p["kind"] == k))
        cells.append(("KS%d taped, second octet block past the last row" % KS, lambda p, f=is_ks: f(p) and p["tape_second_past"]))
    for setup in ("fused", "split"):
        cells.append(("D = 16 (spilling stage 1), setup %s" % setup, lambda p, s=setup: p["spilling_stage1"] and p["setup"] == s))
    return cells


def uncovered(nsm, cases=None):
    """names of the cells of the path matrix that no case reaches on a machine of ``nsm`` SMs"""
    paths = [path_of(*c, nsm) for c in (PATH_CASES if cases is None else cases)]
    return [name for name, pred in coverage_cells() if not any(pred(p) for p in paths)]


# ---------------------------------------------------------------------------------------------------------------------
# regimes: seeded builders -> dict(X, ell, sf2, beta, iK, mode, m [R,D], s [R,D,D]); factors from the fp64 oracle
# factorisation unless stated.  Restart r > 0 repeats the regime with another seed (the device batch), r = 0 is checked.
# ---------------------------------------------------------------------------------------------------------------------
def _factors(X, Y, ell, sf2, sn2):
    from oracle import python_port as pp
    return pp.calculate_factorizations(X, Y, ell, sf2, sn2)


def _targets(X, E, rng):
    return np.sin(X).dot(rng.rand(X.shape[1], E)) + 1e-3 * (rng.rand(X.shape[0], E) - 0.5)


def _inputs(D, R, seed, scale=0.5):
    ms = [make_input(D, seed=seed + r, scale=scale) for r in range(R)]
    return np.concatenate([a for a, _ in ms]), np.stack([b for _, b in ms])


def _base(n, D, E, seed, noise=1e-2):
    X, Y, ell, sf2, sn2 = make_gp_problem(n, D, E, seed=seed, noise=noise)
    return X, Y, ell, sf2, sn2, np.random.RandomState(seed + 7)


def benign(n, D, E, R, kind="exact", seed=0):
    """today's make_gp_problem / make_input: every exponent within a few units of 0"""
    X, Y, ell, sf2, sn2, _ = _base(n, D, E, seed)
    if kind == "mode1":
        sf2, sn2 = np.ones(E), 1e-4 * np.ones(E)
    iK, beta = _factors(X, Y, ell, sf2, sn2)
    m, s = _inputs(D, R, seed + 20)
    return dict(X=X, ell=ell, sf2=sf2, beta=beta, iK=iK if kind == "exact" else None, mode=int(kind == "mode1"), m=m, s=s)


def short_ell(n, D, E, R, seed=0):
    """length-scales far below the data range: most of L' underflows (the exp clamp, large negative A'); m sits on a
    data point and s is a few length-scales wide so that the result is not all zero"""
    X, Y, ell, sf2, sn2, rng = _base(n, D, E, seed)
    ell = 0.03 + 0.17 * rng.rand(E, D)
    iK, beta = _factors(X, Y, ell, sf2, sn2)
    m, s = _inputs(D, R, seed + 20, scale=0.01)
    m = X[rng.randint(n, size=R)].copy()
    return dict(X=X, ell=ell, sf2=sf2, beta=beta, iK=iK, mode=0, m=m, s=s)


def ard_mixed(n, D, E, R, seed=0):
    """ARD as training leaves it: per output a third of the dimensions irrelevant (ell = 1e3), a third short (0.1)"""
    X, Y, ell, sf2, sn2, rng = _base(n, D, E, seed)
    for a in range(E):
        perm = rng.permutation(D)
        ell[a, perm[:D // 3]] = 1e3
        ell[a, perm[D // 3:2 * (D // 3)]] = 0.1
    iK, beta = _factors(X, Y, ell, sf2, sn2)
    m, s = _inputs(D, R, seed + 20, scale=0.05)
    return dict(X=X, ell=ell, sf2=sf2, beta=beta, iK=iK, mode=0, m=m, s=s)


def wide_data(n, D, E, R, seed=0):
    """some dimensions (velocities) span +-10 with length-scales to match; m three length-scales outside the hull"""
    X, Y, ell, sf2, sn2, rng = _base(n, D, E, seed)
    wide = np.arange(D) % 2 == 1
    X = X.copy()
    X[:, wide] = 20.0 * X[:, wide] - 10.0
    ell[:, wide] *= 5.0
    iK, beta = _factors(X, _targets(X / np.where(wide, 5.0, 1.0), E, rng), ell, sf2, sn2)
    m, s = _inputs(D, R, seed + 20)
    T = np.where(wide, 5.0, 1.0)
    s = s * T[None, :, None] * T[None, None, :]                    # (a congruence: s stays positive definite)
    m[:, 0] = 1.0 + 3.0 * ell[:, 0].max()
    return dict(X=X, ell=ell, sf2=sf2, beta=beta, iK=iK, mode=0, m=m, s=s)


def _with_s(n, D, E, R, seed, make_s):
    d = benign(n, D, E, R, seed=seed)
    d["s"] = np.stack([make_s(np.random.RandomState(seed + 40 + r)) for r in range(R)])
    return d


def s_zero(n, D, E, R, seed=0):
    """s = 0 exactly (PILCO.compute_action): the moment match is the GP posterior at m"""
    return _with_s(n, D, E, R, seed, lambda rng: np.zeros((D, D)))


def s_tiny(n, D, E, R, seed=0):
    """s = 1e-14 I: Q = O(1e-14), log det R at rounding level"""
    return _with_s(n, D, E, R, seed, lambda rng: 1e-14 * np.eye(D))


def s_singular(n, D, E, R, seed=0):
    """the joint of a state and a deterministic linear policy, s = [[S, S W'], [W S, W S W']] (rank Ds < D): what every
    linear-policy rollout step feeds the dynamics"""
    Ds = max(1, D - max(1, D // 4))

    def make(rng):
        A = rng.rand(Ds, Ds)
        Sg, W = 0.3 * A @ A.T, rng.randn(D - Ds, Ds)
        return np.block([[Sg, Sg @ W.T], [W @ Sg, W @ Sg @ W.T]])
    return _with_s(n, D, E, R, seed, make)


def s_zero_coordinate(n, D, E, R, seed=0):
    """one coordinate known exactly: a zero row and column in s"""
    def make(rng):
        A = rng.rand(D, D)
        s = 0.3 * A @ A.T
        s[D // 2, :] = 0.0
        s[:, D // 2] = 0.0
        return s
    return _with_s(n, D, E, R, seed, make)


def s_huge(n, D, E, R, seed=0):
    """s = 1e4 I: the input is far wider than the data and every length-scale"""
    return _with_s(n, D, E, R, seed, lambda rng: 1e4 * np.eye(D))


def s_spread(n, D, E, R, seed=0):
    """eigenvalues of s spread over 1e-8 .. 1e4 in a random basis"""
    def make(rng):
        U = np.linalg.qr(rng.randn(D, D))[0]
        s = (U * 10.0 ** np.linspace(-8, 4, D)) @ U.T
        return 0.5 * (s + s.T)
    return _with_s(n, D, E, R, seed, make)


def scales(n, D, E, R, seed=0):
    """signal variances 1e-6 and 1e4 with noise 1e-6: |iK| ~ 1e6 and the trace term cancels heavily against beta beta'"""
    X, Y, ell, sf2, sn2, rng = _base(n, D, E, seed)
    sf2 = np.where(np.arange(E) % 2 == 0, 1e-6, 1e4)
    sn2 = 1e-6 * np.ones(E)
    iK, beta = _factors(X, Y * np.sqrt(sf2)[None, :], ell, sf2, sn2)
    m, s = _inputs(D, R, seed + 20)
    return dict(X=X, ell=ell, sf2=sf2, beta=beta, iK=iK, mode=0, m=m, s=s)


def fitc_factors(n, D, E, R, seed=0):
    """FITC factors over n inducing points (4 n data rows): iK is indefinite, not an inverse Gram matrix (computed by the
    fp64 port of the FITC factorisation)"""
    from oracle import python_port as pp
    Xd, Y, ell, sf2, sn2, rng = _base(4 * n, D, E, seed)
    Z = rng.rand(n, D)
    iK, beta = pp.fitc_factorizations(Xd, Z, Y, ell, sf2, sn2)
    m, s = _inputs(D, R, seed + 20)
    return dict(X=Z, ell=ell, sf2=sf2, beta=beta, iK=iK, mode=0, m=m, s=s)


REGIMES = dict(short_ell=short_ell, ard_mixed=ard_mixed, wide_data=wide_data, s_zero=s_zero, s_tiny=s_tiny,
               s_singular=s_singular, s_zero_coordinate=s_zero_coordinate, s_huge=s_huge, s_spread=s_spread,
               scales=scales, fitc_factors=fitc_factors)


# ---------------------------------------------------------------------------------------------------------------------
# single-element probes: beta_a = e_{i_a}, iK = 0, so T_ab = L'_ab[i_a, i_b] is ONE element of the n x n matrix
# ---------------------------------------------------------------------------------------------------------------------
def probe_indices(n, E=16):
    """E centre indices on the structural boundaries of the tile kernels at THIS n, most specific first: the last valid
    centre, the chunk boundary 511 | 512, one centre in each column tile of the last chunk's tail group (GM <= 4 tiles),
    the row-block boundary 63 | 64, first / last lane of octets 0, 1, 7, 8 (63 | 64 again) and 9, both octets of the
    odd-pass pairs {0, 1} and {8, 9}; then the remaining centres in order.  The first padded centre is never an index."""
    last_tile = (n - 1) // 8
    want = [n - 1]
    if n > 512:
        want += [511, 512]
    want += [8 * t + (3 * t) % 8 for t in range(last_tile - 1, max(last_tile - 4, -1), -1)]   # the other tiles of the tail
    want += [63, 64, 0, 7, 8, 15, 56, 71, 72, 79, 127, 128]
    idx = []
    for i in want + list(range(n)):
        if 0 <= i < n and i not in idx:
            idx.append(i)
    return idx[:E]


def probe(n, D, R, seed=0, E=16):
    """benign geometry, E outputs with distinct length-scales, one-hot beta at ``probe_indices`` and no inverse"""
    rng = np.random.RandomState(seed)
    X = rng.rand(n, D)
    ell, sf2 = 1.0 + rng.rand(E, D), 1.0 + rng.rand(E)
    idx = probe_indices(n, E)
    beta = np.zeros((E, n))
    beta[np.arange(E), idx] = 1.0
    m, s = _inputs(D, R, seed + 20)
    return dict(X=X, ell=ell, sf2=sf2, beta=beta, iK=None, mode=0, m=m, s=s, idx=idx)


def far_probe(n, D, seed=0, E=16):
    """length-scales of 0.03 around a point mass at centre 0, one-hot beta at centres spread from the nearest to the
    farthest: the probed elements run from O(1) down to exp(-3000), across the exp's clamp at 2^-1008"""
    rng = np.random.RandomState(seed)
    X = rng.rand(n, D)
    ell, sf2 = 0.03 * (1.0 + 0.2 * rng.rand(E, D)), np.ones(E)
    order = np.argsort(((X - X[0]) ** 2).sum(1))
    idx = [int(order[int(round(k))]) for k in np.linspace(0, n - 1, E)]
    beta = np.zeros((E, n))
    beta[np.arange(E), idx] = 1.0
    return dict(X=X, ell=ell, sf2=sf2, beta=beta, iK=None, mode=0, m=X[:1].copy(), s=1e-4 * np.eye(D)[None], idx=idx)
