"""The GP factorisations and training objectives in extended precision, with the conditioning of every output.

A plain statement of what ``factorize.cu`` computes (``oracle/python_port.py`` states it in fp64) in ``np.longdouble``
-- the x87 80-bit format where numpy provides it (eps 1.08e-19) -- and, for directional derivatives, in
``np.clongdouble``: every function here is written without conjugation, so it is analytic in its inputs and
``Im f(theta + i h v) / h`` at h = 1e-30 is the derivative along v with no cancellation at all (complex step).

The building blocks are hand-written (numpy's ``linalg`` is fp64 only): the SE-ARD Gram matrix (``expl``), a Cholesky
factorisation by columns, the triangular inverse by rows and triangular solves, each vectorised over rows.

Besides the values every output comes with a CONDITION SCALE, computed in fp64 (it is only a bar): a device result is
judged by ``|error| / (eps64 * scale)``, O(1) to O(n) for a backward-stable fp64 computation however ill-conditioned
the Gram matrix, and large when a kernel loses bits a backward-stable algorithm would not lose.
  L     backward error |K - L L'| against |L| |L'|
  beta  normwise backward error |K beta - y|_inf / (| |K| |beta| |_inf + |y|_inf) (``beta_backward``)
  iK    |K^-1| |L| |L'| |K^-1|, entry by entry: the first-order effect of a backward error of the factorisation
  nlml  the sum of |terms| plus the factor scales propagated through the formula
"""
import numpy as np

LD = np.longdouble
CLD = np.clongdouble
EPS_LD = float(np.finfo(LD).eps)
EPS64 = float(np.finfo(np.float64).eps)
HAVE_EXTENDED = EPS_LD < 1e-18
NEED_EXTENDED = "np.longdouble is only 64 bits wide on this platform: no extended-precision oracle"
LOG2PI = np.log(2 * np.arccos(LD(-1)))
JITTER = 1e-6                    # FITC: Kmm + 1e-6 I (smgpr.py:27)


def _x(a, dtype=LD):
    return np.asarray(a, dtype=dtype)


# ---- building blocks ----------------------------------------------------------------------------------------------
def gram(A, B, ell, sf2):
    """sf2 exp(-0.5 sum_d ((a_d - b_d) / ell_d)^2) from the differences (no |a|^2 + |b|^2 - 2ab cancellation)"""
    dt = np.result_type(A, B, ell, sf2, LD)
    A, B, ell = _x(A, dt), _x(B, dt), _x(ell, dt)
    d2 = np.zeros((A.shape[0], B.shape[0]), dt)
    for d in range(A.shape[1]):
        t = (A[:, d][:, None] - B[:, d][None, :]) / ell[d]
        d2 = d2 + t * t
    return _x(sf2, dt) * np.exp(-d2 / 2)


def cholesky(A):
    """lower L with L L^T = A (no conjugation: analytic for complex A); raises LinAlgError at a pivot <= 0"""
    A = np.array(A)
    n = A.shape[0]
    L = np.zeros_like(A)
    for j in range(n):
        p = A[j, j] - L[j, :j] @ L[j, :j]
        if np.real(p) <= 0:
            raise np.linalg.LinAlgError("pivot %d not positive in the factorisation oracle" % j)
        L[j, j] = np.sqrt(p)
        L[j + 1:, j] = (A[j + 1:, j] - L[j + 1:, :j] @ L[j, :j]) / L[j, j]
    return L


def tri_inverse(L):
    """R = L^-1 of a lower-triangular L, by rows"""
    n = L.shape[0]
    R = np.zeros_like(L)
    for i in range(n):
        R[i, i] = 1 / L[i, i]
        R[i, :i] = -(L[i, :i] @ R[:i, :i]) * R[i, i]
    return R


def solve_lower(L, b):
    x = np.array(b, dtype=np.result_type(L, b))
    for i in range(L.shape[0]):
        x[i] = (x[i] - L[i, :i] @ x[:i]) / L[i, i]
    return x


def solve_upper_t(L, b):
    """x with L^T x = b"""
    x = np.array(b, dtype=np.result_type(L, b))
    for i in range(L.shape[0] - 1, -1, -1):
        x[i] = (x[i] - L[i + 1:, i] @ x[i + 1:]) / L[i, i]
    return x


def abs_prod_scale(L, M):
    """|M| |L| |L'| |M| in fp64 (the first-order effect on M = K^-1 of a backward error bounded by |L| |L'|)"""
    aL, aM = np.abs(np.asarray(L, np.float64)), np.abs(np.asarray(M, np.float64))
    return aM @ (aL @ (aL.T @ aM))


# ---- exact GP -----------------------------------------------------------------------------------------------------
def gp_factor(X, y, ell, sf2, sn2, dtype=LD):
    """One output of pilco_gp_factorize: dict(K, L, R, iK, beta, logdet) with K = Gram + sn2 I"""
    K = gram(_x(X, dtype), _x(X, dtype), _x(ell, dtype), _x(sf2, dtype))
    K = K + _x(sn2, dtype) * np.eye(K.shape[0], dtype=dtype)
    L = cholesky(K)
    R = tri_inverse(L)
    y = _x(y, dtype)
    return dict(K=K, L=L, R=R, iK=R.T @ R, beta=solve_upper_t(L, solve_lower(L, y)),
                logdet=2 * np.log(np.diagonal(L)).sum())


def gram_scale(X, ell, K):
    """|K| (1 + d2) in fp64: the conditioning of the Gram entries themselves -- exp(-d2 / 2) turns the rounding of the
    scaled squared distance d2 into a relative error of about d2 eps64, large where some ell_d is short"""
    X, ell = np.asarray(X, np.float64), np.asarray(ell, np.float64)
    d2 = sum(((X[:, d][:, None] - X[:, d][None, :]) / ell[d]) ** 2 for d in range(X.shape[1]))
    return np.abs(K.astype(np.float64)) * (1.0 + d2)


def gp_scales(f, X, ell):
    """fp64 condition scales of gp_factor's outputs: LL = |L| |L'| + |K| (1 + d2), the bar of a backward error of the
    factorisation including the Gram entries' own rounding, and iK = |K^-1| LL |K^-1| entry by entry"""
    aL = np.abs(f["L"].astype(np.float64))
    LL = aL @ aL.T + gram_scale(X, ell, f["K"])
    aM = np.abs(f["iK"].astype(np.float64))
    return dict(iK=aM @ (LL @ aM), LL=LL)


def beta_backward(K, beta_hat, y):
    """normwise backward error of a computed solution of K beta = y, residual in longdouble, K longdouble [n,n]"""
    b, y = _x(beta_hat), _x(y)
    r = K @ b - y
    den = (np.abs(K).astype(np.float64) @ np.abs(np.asarray(beta_hat, np.float64))).max() + float(np.abs(y).max())
    return float(np.abs(r).max()) / den


def beta_backward_chunked(X, ell, sf2, sn2, beta_hat, y, rows=256):
    """beta_backward with K built row block by row block (large n: K itself is never held)"""
    X, b, y = _x(X), _x(beta_hat), _x(y)
    ab = np.abs(np.asarray(beta_hat, np.float64))
    rmax, den = 0.0, 0.0
    for i0 in range(0, X.shape[0], rows):
        Kr = gram(X[i0:i0 + rows], X, ell, sf2)
        Kr[np.arange(Kr.shape[0]), i0 + np.arange(Kr.shape[0])] += _x(sn2)
        rmax = max(rmax, float(np.abs(Kr @ b - y[i0:i0 + rows]).max()))
        den = max(den, float((np.abs(Kr).astype(np.float64) @ ab).max()))
    return rmax / (den + float(np.abs(y).max()))


def dgram(X, ell, sf2, K0):
    """[D + 2] list of dK/dtheta for theta = (ell_1 .. ell_D, sf2, sn2) of one output (K0 = Gram without noise)"""
    X, ell = _x(X, K0.dtype), _x(ell, K0.dtype)
    out = []
    for d in range(X.shape[1]):
        t = (X[:, d][:, None] - X[:, d][None, :])
        out.append(K0 * t * t / ell[d] ** 3)
    out.append(K0 / _x(sf2, K0.dtype))
    out.append(np.eye(X.shape[0], dtype=K0.dtype))
    return out


def gp_nlml(X, y, ell, sf2, sn2, want_grad=True, want_scale=True):
    """-log N(y | 0, K + sn2 I) of one output, the closed-form gradient -0.5 tr((a a' - K^-1) dK/dtheta) over
    theta = (ell, sf2, sn2), and their condition scales -> dict(nlml, grad [D+2], c_nlml, c_grad [D+2])"""
    f = gp_factor(X, y, ell, sf2, sn2)
    n = f["K"].shape[0]
    y = _x(y)
    a = f["beta"]
    fit, half_ld = y @ a / 2, f["logdet"] / 2
    out = dict(nlml=fit + half_ld + n * LOG2PI / 2)
    if want_scale:
        sc = gp_scales(f, X, ell)
        a64, iK64 = np.abs(a.astype(np.float64)), np.abs(f["iK"].astype(np.float64))
        L64 = np.abs(f["L"].astype(np.float64))
        out["c_nlml"] = (float(np.abs(y @ a)) / 2 + float(np.abs(np.log(np.diagonal(L64))).sum()) + n * float(LOG2PI) / 2
                         + a64 @ sc["LL"] @ a64 / 2 + (iK64 * sc["LL"]).sum() / 2)
    if want_grad:
        K0 = f["K"] - _x(sn2) * np.eye(n, dtype=LD)
        W = np.outer(a, a) - f["iK"]
        dK = dgram(X, ell, sf2, K0)
        out["grad"] = np.array([-(W * g).sum() / 2 for g in dK], dtype=LD)
        if want_scale:
            sa = iK64 @ (sc["LL"] @ a64)                       # |K^-1| |L||L'| |alpha|: first-order error of alpha
            cW = np.abs(W.astype(np.float64)) + np.outer(sa, a64) + np.outer(a64, sa) + sc["iK"]
            gs = gram_scale(X, ell, np.ones_like(K0)) + 1.0         # dK/dtheta's own relative rounding, 1 + d2
            out["c_grad"] = np.array([(cW * np.abs(g.astype(np.float64)) * gs).sum() / 2 for g in dK])
    return out


def gp_nlml_cs(X, y, ell, sf2, sn2, v, h=1e-30):
    """d nlml / dt along theta + t v, v = (v_ell [D], v_sf2, v_sn2), by complex step in clongdouble"""
    D = len(ell)
    v = _x(v)
    ih = CLD(1j) * LD(h)
    ellc = _x(ell, CLD) + ih * v[:D]
    sf2c, sn2c = _x(sf2, CLD) + ih * v[D], _x(sn2, CLD) + ih * v[D + 1]
    f = gp_factor(_x(X, CLD), _x(y, CLD), ellc, sf2c, sn2c, dtype=CLD)
    val = _x(y, CLD) @ f["beta"] / 2 + f["logdet"] / 2
    return np.imag(val) / LD(h)


# ---- FITC ---------------------------------------------------------------------------------------------------------
def fitc_factor(X, Z, y, ell, sf2, sn2):
    """One output of pilco_fitc_factorize (smgpr.py:24-45 as oracle.python_port.fitc_factorizations states it)
    -> dict(iK, beta) and their fp64 condition scales c_iK, c_beta.  iK = Kmm^-1 - sn2 (L Am)^-T (L Am)^-1 cancels by
    design; its scale is the sum of both parts' absolute values, each with its own propagated scale."""
    X, Z, y, ell, sf2, sn2 = _x(X), _x(Z), _x(y), _x(ell), _x(sf2), _x(sn2)
    M = Z.shape[0]
    Kmm = gram(Z, Z, ell, sf2) + LD(JITTER) * np.eye(M, dtype=LD)
    Kmn = gram(Z, X, ell, sf2)
    L = cholesky(Kmm)
    Li = tri_inverse(L)
    V = Li @ Kmn
    G = np.sqrt(1 + (sf2 - (V * V).sum(0)) / sn2)
    V = V / G
    Am = cholesky(V @ V.T + sn2 * np.eye(M, dtype=LD))
    Ai = tri_inverse(Am)
    iAt = Ai @ Li
    beta = Li.T @ (Ai.T @ (Ai @ ((V / G) @ y)))
    P1, P2 = Li.T @ Li, iAt.T @ iAt
    A = L @ Am
    c1 = np.abs(P1.astype(np.float64)) + abs_prod_scale(L, P1)
    c2 = float(sn2) * (np.abs(P2.astype(np.float64)) + abs_prod_scale(A, P2))
    aA, aP2 = np.abs(A.astype(np.float64)), np.abs(P2.astype(np.float64))
    rhs = np.abs(Kmn.astype(np.float64)) @ (np.abs(y.astype(np.float64)) / (G.astype(np.float64) ** 2))
    c_beta = aP2 @ (aA @ (aA.T @ np.abs(beta.astype(np.float64))) + np.abs(L.astype(np.float64)) @
                    (np.abs(Li.astype(np.float64)) @ rhs))
    return dict(iK=P1 - sn2 * P2, beta=beta, c_iK=c1 + c2, c_beta=c_beta)


def fitc_bound(X, y, Z, ell, sf2, sn2, dtype=LD):
    """the collapsed FITC bound as oracle/fitc_staged.fitc_nlml states it (value only; analytic for complex inputs)
    -> (value, fp64 scale: sum of |terms| and the nu cancellation sf2 + sn2 - colsum(V o V) propagated)"""
    X, y, Z = _x(X, dtype), _x(y, dtype), _x(Z, dtype)
    ell, sf2, sn2 = _x(ell, dtype), _x(sf2, dtype), _x(sn2, dtype)
    N, M = X.shape[0], Z.shape[0]
    Kuf = gram(Z, X, ell, sf2)
    Luu = cholesky(gram(Z, Z, ell, sf2) + _x(JITTER, dtype) * np.eye(M, dtype=dtype))
    V = tri_inverse(Luu) @ Kuf
    nu = sf2 + sn2 - (V * V).sum(0)
    B = np.eye(M, dtype=dtype) + (V / nu) @ V.T
    L = cholesky(B)
    gamma = solve_lower(L, V @ (y / nu))
    terms = [(y * y / nu).sum() / 2, -(gamma @ gamma) / 2, np.log(nu).sum() / 2, np.log(np.diagonal(L)).sum(),
             N * LOG2PI / 2]
    val = sum(terms)
    if dtype is CLD:
        return val, None
    f64 = lambda a: np.abs(np.asarray(a, np.float64))
    cnu = f64(sf2) + f64(sn2) + (f64(V) ** 2).sum(0)            # |nu| before the cancellation
    dnu = (f64(y) ** 2 / f64(nu) ** 2 + 1 / f64(nu)) / 2        # |d value / d nu|
    aL = f64(L)
    Bi = f64(tri_inverse(L).T @ tri_inverse(L))
    scale = sum(float(abs(t)) for t in terms) + float((dnu * cnu).sum()) + float((Bi * (aL @ aL.T)).sum()) \
        + float(f64(gamma) @ f64(gamma))
    return val, scale


def fitc_bound_cs(X, y, Z, ell, sf2, sn2, v_ell, v_sf2, v_sn2, v_Z, h=1e-30):
    """d bound / dt along (ell, sf2, sn2, Z) + t (v_ell, v_sf2, v_sn2, v_Z) by complex step"""
    ih = CLD(1j) * LD(h)
    val, _ = fitc_bound(X, y, _x(Z, CLD) + ih * _x(v_Z), _x(ell, CLD) + ih * _x(v_ell), _x(sf2, CLD) + ih * LD(v_sf2),
                        _x(sn2, CLD) + ih * LD(v_sn2), dtype=CLD)
    return np.imag(val) / LD(h)


def max_ratio(err, scale):
    """max |err| / (eps64 * scale) over the entries"""
    err = np.abs(np.asarray(err, np.float64))
    return float(np.max(err / (EPS64 * np.maximum(np.asarray(scale, np.float64), 1e-300))))
