"""The SE-ARD moment match in extended precision, with the conditioning of every output entry.

A plain statement of DESIGN.md section 3 (the kernels' formulation, as ``oracle/staged.py`` states it in fp64) in
``np.longdouble`` -- the x87 80-bit format where numpy provides it (eps 1.08e-19).  The factors ``beta`` and ``iK`` are
INPUTS, so the moment match is tested apart from the factorisation and can be fed arbitrary factors (FITC's indefinite
``iK``, one-hot ``beta``).  The D x D solves and log-determinants are a hand-written elimination (numpy's ``linalg`` is
fp64 only); the n x n work is vectorised (``np.exp`` is ``expl`` on ``longdouble``).

Besides ``M, S, V`` every entry comes with its CONDITION SCALE, the sum of the absolute values of the terms it was
summed from: a device result is judged by ``|error| / (eps64 * scale)``, which is O(1) for a well-written fp64 kernel
whatever the cancellation in the sum, and grows when a kernel loses bits it did not have to lose.
"""
import numpy as np

LD = np.longdouble
EPS_LD = float(np.finfo(LD).eps)
EPS64 = float(np.finfo(np.float64).eps)
HAVE_EXTENDED = EPS_LD < 1e-18
NEED_EXTENDED = "np.longdouble is only 64 bits wide on this platform: no extended-precision oracle"


def _ld(a):
    return np.asarray(a, dtype=LD)


def solve_logdet(A, B):
    """X = A^-1 B and log det A (A with positive determinant) by Gaussian elimination with partial pivoting."""
    A = _ld(A).copy()
    X = _ld(B).copy()
    k = A.shape[0]
    logdet, sign = LD(0), 1
    for j in range(k):
        piv = j + int(np.argmax(np.abs(A[j:, j])))
        if piv != j:
            A[[j, piv]] = A[[piv, j]]
            X[[j, piv]] = X[[piv, j]]
            sign = -sign
        d = A[j, j]
        if d == 0:
            raise np.linalg.LinAlgError("singular matrix in the moment-match oracle")
        if d < 0:
            sign = -sign
        logdet = logdet + np.log(np.abs(d))
        f = A[j + 1:, j] / d
        A[j + 1:] = A[j + 1:] - f[:, None] * A[j][None, :]
        X[j + 1:] = X[j + 1:] - f[:, None] * X[j][None, :]
    if sign < 0:
        raise np.linalg.LinAlgError("negative determinant in the moment-match oracle")
    for j in range(k - 1, -1, -1):
        X[j] = (X[j] - A[j, j + 1:] @ X[j + 1:]) / A[j, j]
    return X, logdet


def pair_operands(zeta, p, lsf2, s, a, b):
    """A'[n], B[m], U'[n,:] of the pair (a, b): L'[n,m] = exp(A'[n] + B[m] + U'[n].zeta[m]) (unscaled exponents)."""
    delta = p[a] + p[b]
    Amat = s + np.diag(1 / delta)
    Y, ldA = solve_logdet(Amat, s)                       # Cm s
    Q = LD(0.5) * Y / delta[:, None]
    Q = (Q + Q.T) / 2
    logdetR = ldA + np.log(delta).sum()
    za, zb = zeta * p[a], zeta * p[b]
    k = lsf2[:, None] - (p[:, None, :] * zeta[None] ** 2).sum(-1) / 2
    Ap = k[a] + ((za @ Q) * za).sum(1) - logdetR / 2
    Bq = k[b] + ((zb @ Q) * zb).sum(1)
    Ua = 2 * (za @ Q) * p[b]
    return Ap, Bq, Ua


def moment_match(X, ell, sf2, beta, iK, m, s, mode=0, want_scale=True):
    """-> dict(M [E], S [E,E], V [D,E], and with ``want_scale`` cM, cS, cV: the condition scales), all longdouble.

    ``iK`` None or [E,n,n]: the trace term of the diagonal pairs (exact-GP mode with an inverse).  ``mode`` 1 adds 1e-6
    instead of sf2 on the diagonal of S (the RBF policy's fixed prior variance and noise cancel up to that)."""
    X, ell, sf2, beta, m, s = _ld(X), _ld(ell), _ld(sf2), _ld(beta), _ld(m).reshape(-1), _ld(s)
    E, D = ell.shape
    s = (s + s.T) / 2
    zeta = X - m[None, :]
    p = 1 / ell ** 2
    lsf2 = np.log(sf2)
    M, V = np.zeros(E, LD), np.zeros((D, E), LD)
    cM, cV = np.zeros(E, LD), np.zeros((D, E), LD)
    for a in range(E):
        A = s + np.diag(ell[a] ** 2)
        W, ldA = solve_logdet(A, np.eye(D))
        t = zeta @ W
        c = np.exp(lsf2[a] + np.log(ell[a] ** 2).sum() / 2 - ldA / 2)
        w = c * beta[a] * np.exp(-(zeta * t).sum(1) / 2)
        M[a] = w.sum()
        cM[a] = np.abs(w).sum()
        V[:, a] = (w[:, None] * t).sum(0)
        cV[:, a] = np.abs(w[:, None] * t).sum(0)
    S, cS = np.zeros((E, E), LD), np.zeros((E, E), LD)
    for b in range(E):
        for a in range(b + 1):
            Ap, Bq, Ua = pair_operands(zeta, p, lsf2, s, a, b)
            G = beta[a][:, None] * beta[b][None, :]
            if a == b and mode == 0 and iK is not None:
                G = G - _ld(iK[a])
            H = G * np.exp(Ap[:, None] + Bq[None, :] + Ua @ zeta.T)
            dg = (sf2[a] if mode == 0 else LD(1e-6)) if a == b else LD(0)
            S[a, b] = S[b, a] = H.sum() + dg - M[a] * M[b]
            cS[a, b] = cS[b, a] = np.abs(H).sum() + dg + np.abs(M[a] * M[b])
    out = dict(M=M, S=S, V=V)
    if want_scale:
        out.update(cM=cM, cS=cS, cV=cV)
    return out


def log_element(X, ell, sf2, m, s, a, b, i, j):
    """log L'_ab[i, j]: the exponent of ONE element of the n x n matrix of pair (a, b) (single-element probes)"""
    X, ell, sf2, m, s = _ld(X), _ld(ell), _ld(sf2), _ld(m).reshape(-1), _ld(s)
    s = (s + s.T) / 2
    Ap, Bq, Ua = pair_operands(X - m[None, :], 1 / ell ** 2, np.log(sf2), s, a, b)
    return Ap[i] + Bq[j] + Ua[i] @ (X[j] - m)


def contraction(out, gM, gS, gV):
    """<gM, M> + <gS, S> + <gV, V> and its condition scale (the same sum over the entries' condition scales)"""
    gM, gS, gV = _ld(gM), _ld(gS), _ld(gV)
    val = (gM * out["M"]).sum() + (gS * out["S"]).sum() + (gV * out["V"]).sum()
    scale = (np.abs(gM) * out["cM"]).sum() + (np.abs(gS) * out["cS"]).sum() + (np.abs(gV) * out["cV"]).sum()
    return val, scale


def directional_derivative(X, ell, sf2, beta, iK, m, s, dm, ds, gM, gS, gV, mode=0, h=None):
    """d/dt <g, (M, S, V)>(m + t dm, s + t ds) at t = 0 by central differences with one Richardson step, in longdouble:
    truncation O(h^4), round-off eps_ld / h -- about 1e-14 of the function's scale, with no autograd involved.
    ``ds`` symmetric; ``h`` defaults to 1e-4 of the shortest squared length-scale (at most 1e-4).  The formulas are analytic wherever s + diag(ell^2) and s + diag(1/(p_a + p_b)) are positive
    definite, so the steps may leave the PSD cone at a singular ``s`` (they never reach a device)."""
    m, s, dm, ds = _ld(m).reshape(-1), _ld(s), _ld(dm).reshape(-1), _ld(ds)
    if h is None:
        h = 1e-4 * min(1.0, float(np.min(np.asarray(ell, dtype=np.float64))) ** 2)

    def f(t):
        t = LD(t)
        return contraction(moment_match(X, ell, sf2, beta, iK, m + t * dm, s + t * ds, mode), gM, gS, gV)[0]

    def central(step):
        return (f(step) - f(-step)) / (2 * LD(step))
    return (4 * central(h / 2) - central(h)) / 3
