"""Shared test helpers: seeded synthetic problems (SURVEY.md section 8d recipe), error metrics and the SASS of the
built library."""
import ctypes
import functools
import os
import re
import shutil
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CUOBJDUMP = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"


@functools.lru_cache(maxsize=None)
def _sass_functions():
    """[(mangled name, SASS text)] of every function of the built library, from one cuobjdump run per process.  A
    function's text ends at the next function or at the next module's Fatbin header, which holds the source path."""
    lib = os.path.join(ROOT, "pilco_b200", "libpilco_b200.so")
    out = subprocess.run([CUOBJDUMP, "-sass", lib], capture_output=True, text=True, timeout=600).stdout
    funcs, name, lines = [], None, []
    for line in out.splitlines() + ["Fatbin"]:
        m = re.match(r"\s*Function : (\S+)", line)
        if m or line.startswith("Fatbin"):
            if name:
                funcs.append((name, "\n".join(lines)))
            name, lines = (m.group(1) if m else None), []
        elif name:
            lines.append(line)
    return funcs


def sass(pattern):
    """{mangled name: SASS text} of every function whose name matches the regular expression ``pattern`` (a static
    kernel that several modules hold: the last module's copy)"""
    return {name: text for name, text in _sass_functions() if re.search(pattern, name)}


def sass_named(names):
    """{name: SASS text} of the kernels whose mangled names contain one of ``names`` (keyed by the first that does)"""
    return {next(k for k in names if k in m): text for m, text in sass("|".join(map(re.escape, names))).items()}


def relerr(a, b):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    return float(np.max(np.abs(a - b) / (np.abs(b) + 1e-300)))


def scaled_err(a, b):
    """max |a-b| / max|b|  (robust when individual entries are ~0)"""
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    return float(np.max(np.abs(a - b)) / (np.max(np.abs(b)) + 1e-300))


def make_gp_problem(n, D, E, seed=0, noise=1e-2):
    """X=rand(n,D), Y=sin(X)A+noise (test_predictions.py:19-21 recipe), benign fixed hyper-parameters."""
    rng = np.random.RandomState(seed)
    X = rng.rand(n, D)
    A = rng.rand(D, E)
    Y = np.sin(X).dot(A) + 1e-3 * (rng.rand(n, E) - 0.5)
    ell = 1.0 + rng.rand(E, D)
    sf2 = 1.0 + rng.rand(E)
    sn2 = noise * np.ones(E)
    return X, Y, ell, sf2, sn2


def make_input(D, seed=1, scale=1.0):
    rng = np.random.RandomState(seed)
    m = rng.rand(1, D)
    s = rng.rand(D, D)
    s = scale * s.dot(s.T)
    return m, s


def hyp_of(ell, sf2, sn2):
    """MATLAB log-hyper layout [D+2, E] (test_predictions.py:44-48)."""
    return np.log(np.hstack((ell, np.sqrt(sf2[:, None]), np.sqrt(sn2[:, None])))).T


def make_rollout_problem(N, Ds, U, bf, R, seed=0):
    """Seeded synthetic PILCO problem of a BASELINE.json config shape (SURVEY.md section 8d recipe, as bench.py builds the
    metric workload): dynamics data X=rand(N,D), state differences Y = 0.05 (sin(X) A + noise), fixed benign
    hyper-parameters; R RBF policies with bf centres.  Small state differences keep a 40-50 step rollout with
    untrained hyper-parameters finite (cf. tests/test_cascade.py:22)."""
    D = Ds + U
    rng = np.random.RandomState(seed)
    X = rng.rand(N, D)
    A = rng.rand(D, Ds)
    Y = 0.05 * (np.sin(X).dot(A) + 1e-3 * (rng.rand(N, Ds) - 0.5))
    ell = 1.0 + rng.rand(Ds, D)
    sf2 = 0.05 * (1.0 + rng.rand(Ds))
    sn2 = 1e-3 * np.ones(Ds)
    Xc, Yc, lc = [], [], []
    for r in range(R):
        rr = np.random.RandomState(seed + 1 + r)
        Xc.append(rr.randn(bf, Ds) * 0.5 + 0.5)
        Yc.append(0.1 * rr.randn(bf, U))
        lc.append(1.0 + 0.1 * rr.randn(U, Ds))
    return dict(X=X, Y=Y, ell=ell, sf2=sf2, sn2=sn2, Xc=np.stack(Xc), Yc=np.stack(Yc), lc=np.stack(lc),
                m0=X[0, :Ds].copy(), S0=0.1 * np.eye(Ds), W=np.eye(Ds), t=np.zeros(Ds), maxa=np.ones(U))


def oracle_rollout(P, r, H, dyn_fact=None, centres=None):
    """H-step cascade of restart r with the numpy port of the reference's Python path (oracle.python_port).
    ``dyn_fact`` = (iK, beta) to use instead of the exact-GP factorisation (FITC), with ``centres`` = Z."""
    from oracle import python_port as pp
    Ds = P["m0"].shape[0]
    iK, beta = dyn_fact if dyn_fact is not None else pp.calculate_factorizations(P["X"], P["Y"], P["ell"], P["sf2"], P["sn2"])
    C = P["X"] if centres is None else centres
    return pp.predict(P["m0"][None], P["S0"], H,
                      lambda m, s: pp.rbf_action(P["Xc"][r], P["Yc"][r], P["lc"][r], m, s, True, P["maxa"][None]),
                      lambda m, s: pp.predict_given_factorizations(C, P["ell"], P["sf2"], m, s, iK, beta),
                      lambda m, s: pp.exponential_reward(m, s, P["W"], P["t"][None]))


def _rel(g, ref):
    """the largest difference of the gradient dicts g and ref, relative to ref's largest entry"""
    scale = max(float(np.abs(r).max()) for r in ref.values())
    return max(float(np.abs(g[k].reshape(ref[k].shape) - ref[k]).max()) for k in ref) / scale


def _zscores(a, b=None, ref=None):
    """largest |mean| / standard error of a - b (paired draws) or of a against the constant ref"""
    worst = 0.0
    for k in a:
        d = np.stack(a[k]) - (np.stack(b[k]) if b is not None else ref[k])
        worst = max(worst, float(np.max(np.abs(d.mean(0)) / (d.std(0, ddof=1) / np.sqrt(d.shape[0])))))
    return worst


def _ref(x):
    """a ctypes reference to x, or NULL for None"""
    return ctypes.byref(x) if x is not None else None


def _round2(n):
    """n rounded up to even: the workspace slots' 16-byte alignment in doubles"""
    return n + (n & 1)


# ---- the host build of trig_math.cuh (tests/host_harness/trig_harness.cpp) -------------------------------------------
_dp = ctypes.POINTER(ctypes.c_double)


def trig_harness(so):
    """compile the host harness of the angular feature map's closed forms into the shared library ``so`` and load it"""
    subprocess.check_call(["g++", "-O1", "-shared", "-fPIC", "-x", "c++", "-o", so,
                           os.path.join(ROOT, "tests", "host_harness", "trig_harness.cpp")])
    lib = ctypes.CDLL(so)
    ip = ctypes.POINTER(ctypes.c_int)
    lib.trig_moments_host.argtypes = [ctypes.c_int, ctypes.c_int, ip] + [_dp] * 5
    lib.trig_vjp_host.argtypes = [ctypes.c_int, ctypes.c_int, ip] + [_dp] * 7
    lib.angles_layout.argtypes = [ctypes.POINTER(ctypes.c_size_t)]
    return lib


def _p(a):
    return np.ascontiguousarray(a, dtype=np.float64).ctypes.data_as(_dp)


def host_moments(lib, m, s, dims):
    Ds, A = len(m), len(dims)
    Dh = Ds + A
    M, S, C = np.zeros(Dh), np.zeros((Dh, Dh)), np.zeros((Ds, Dh))
    m, s = np.ascontiguousarray(m, dtype=np.float64), np.ascontiguousarray(s, dtype=np.float64)
    d = (ctypes.c_int * max(A, 1))(*dims)
    assert lib.trig_moments_host(Ds, A, d, _p(m), _p(s), M.ctypes.data_as(_dp), S.ctypes.data_as(_dp),
                                 C.ctypes.data_as(_dp)) == 0
    return M, S, C


def host_vjp(lib, m, s, dims, gM, gS, gC):
    Ds, A = len(m), len(dims)
    gm, gs = np.zeros(Ds), np.zeros((Ds, Ds))
    arrs = [np.ascontiguousarray(a, dtype=np.float64) for a in (m, s, gM, gS, gC)]
    d = (ctypes.c_int * max(A, 1))(*dims)
    assert lib.trig_vjp_host(Ds, A, d, *[a.ctypes.data_as(_dp) for a in arrs], gm.ctypes.data_as(_dp),
                             gs.ctypes.data_as(_dp)) == 0
    return gm, gs


def _trig_cases():
    rng = np.random.RandomState(7)
    out = []
    for Ds, dims in ((2, [0]), (4, [2]), (4, [1, 3]), (3, [2, 0, 1]), (6, [4, 1])):
        B = rng.randn(Ds, Ds)
        out.append(("random", rng.randn(Ds) * 2, 0.3 * B @ B.T, dims))
    out.append(("zero_cov", np.array([0.3, -2.0, 1.1]), np.zeros((3, 3)), [1, 2]))
    s = np.diag([0.2, 10.0, 0.5]); s[0, 2] = s[2, 0] = 0.1
    out.append(("saa_10", np.array([0.5, 1.0, -0.7]), s, [1]))
    L = np.array([[1.0, 0.0, 0.0], [0.999, 0.0447, 0.0], [0.2, 0.1, 0.5]])
    out.append(("correlated_angles", np.array([0.4, -1.3, 0.2]), 0.8 * L @ L.T, [0, 1]))
    v = rng.randn(4)
    out.append(("singular", rng.randn(4), np.outer(v, v), [0, 3]))
    return out


TRIG_CASES = _trig_cases()     # (name, m [Ds], s [Ds,Ds], angle dims)
