"""GPflow 2.1's predictive forms, transcribed in numpy (fp64) from their documented algebra, for the tests of
pilco_gp_predict.  They use the Cholesky forms GPflow computes with, independently of the (iK, beta) form the device
kernel contracts:

- ``gpr_predict_f``: gpflow.models.GPR.predict_f through ``base_conditional``: Lm = chol(K + sn2 I), A = Lm^-1 K_mn,
  var = k** - A'A, mean = (Lm^-T A)' y.
- ``fitc_predict_f``: gpflow.models.GPRFITC ``common_terms`` + ``predict_f``: Luu = chol(Kuu + 1e-6 I),
  V = Luu^-1 Kuf, nu = Kdiag - diag(V'V) + sn2, L = chol(I + V diag(1/nu) V'), gamma = L^-1 V (y / nu);
  w = Luu^-1 Kus, mean = w' L^-T gamma, var = k** - w'w + (L^-1 w)'(L^-1 w).

Single output: X [N,D], y [N], ell [D], sf2, sn2 scalars, Xs [T,D].  Returns mean [T] and var [T] or [T,T].
"""
import numpy as np
from scipy.linalg import solve_triangular


def se_ard(X1, X2, ell, sf2):
    d = (X1[:, None, :] - X2[None, :, :]) / ell
    return sf2 * np.exp(-0.5 * (d * d).sum(-1))


def gpr_predict_f(X, y, ell, sf2, sn2, Xs, full_cov=False):
    Kmm = se_ard(X, X, ell, sf2) + sn2 * np.eye(X.shape[0])
    Kmn = se_ard(X, Xs, ell, sf2)
    Lm = np.linalg.cholesky(Kmm)
    A = solve_triangular(Lm, Kmn, lower=True)
    var = se_ard(Xs, Xs, ell, sf2) - A.T @ A if full_cov else sf2 - (A * A).sum(0)
    A = solve_triangular(Lm.T, A, lower=False)
    return A.T @ y, var


def fitc_predict_f(X, Z, y, ell, sf2, sn2, Xs, full_cov=False):
    M = Z.shape[0]
    Luu = np.linalg.cholesky(se_ard(Z, Z, ell, sf2) + 1e-6 * np.eye(M))
    V = solve_triangular(Luu, se_ard(Z, X, ell, sf2), lower=True)
    nu = sf2 - (V * V).sum(0) + sn2
    L = np.linalg.cholesky(np.eye(M) + (V / nu) @ V.T)
    gamma = solve_triangular(L, V @ (y / nu), lower=True)
    w = solve_triangular(Luu, se_ard(Z, Xs, ell, sf2), lower=True)
    mean = w.T @ solve_triangular(L.T, gamma, lower=False)
    a = solve_triangular(L, w, lower=True)
    if full_cov:
        return mean, se_ard(Xs, Xs, ell, sf2) - w.T @ w + a.T @ a
    return mean, sf2 - (w * w).sum(0) + (a * a).sum(0)


def ik_beta_predict(C, ell, sf2, iK, beta, Xs):
    """The (iK, beta) form the device kernel implements: mean = k*' beta, var = sf2 - k*' iK k*."""
    Ks = se_ard(Xs, C, ell, sf2)
    return Ks @ beta, sf2 - ((Ks @ iK) * Ks).sum(1)
