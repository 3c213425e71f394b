"""GPflow 2.1's GPModel.predict_f_samples in numpy (fp64), given the standard normals, for the tests of
pilco_gp_predict_samples.  The posterior covariance is ``predict_oracle``'s Cholesky form (exact GPR or FITC, the
algebra GPflow computes with), then

  full_cov=True :  L = chol(cov + jitter I),  samples = mean + L eps      (GPflow's default_jitter() = 1e-6)
  full_cov=False:  samples = mean + sqrt(max(var, 0)) eps                   (no jitter)

Single output: X [N,D], y [N], ell [D], sf2, sn2 scalars, Xs [T,D], eps [S,T].  ``Z`` selects FITC.  Returns
samples [S,T], mean [T] and the covariance [T,T] (full_cov) or variance [T] that drew them.
"""
import numpy as np

from predict_oracle import fitc_predict_f, gpr_predict_f

DEFAULT_JITTER = 1e-6


def posterior(X, y, ell, sf2, sn2, Xs, full_cov=True, Z=None):
    if Z is None:
        return gpr_predict_f(X, y, ell, sf2, sn2, Xs, full_cov=full_cov)
    return fitc_predict_f(X, Z, y, ell, sf2, sn2, Xs, full_cov=full_cov)


def draw(mean, cov_or_var, eps, full_cov=True, jitter=DEFAULT_JITTER):
    """samples [S,T] = mean + L eps (full_cov) or mean + sqrt(max(var, 0)) eps, for eps [S,T]"""
    eps = np.asarray(eps, dtype=np.float64)
    if full_cov:
        L = np.linalg.cholesky(cov_or_var + jitter * np.eye(cov_or_var.shape[0]))
        return mean[None] + eps @ L.T
    return mean[None] + np.sqrt(np.maximum(cov_or_var, 0.0))[None] * eps


def predict_f_samples(X, y, ell, sf2, sn2, Xs, eps, full_cov=True, Z=None, jitter=DEFAULT_JITTER):
    mean, c = posterior(X, y, ell, sf2, sn2, Xs, full_cov=full_cov, Z=Z)
    return draw(mean, c, eps, full_cov=full_cov, jitter=jitter), mean, c


def ik_beta_posterior(C, ell, sf2, iK, beta, Xs, full_cov=True):
    """The same posterior in the (iK, beta) form the device contracts (mean = K* beta, cov = K** - K* iK K*'), with
    numpy's own iK: its difference from ``posterior`` is the oracle's own sensitivity to a reordered product."""
    from predict_oracle import se_ard
    Ks = se_ard(Xs, C, ell, sf2)
    if full_cov:
        return Ks @ beta, se_ard(Xs, Xs, ell, sf2) - Ks @ iK @ Ks.T
    return Ks @ beta, sf2 - ((Ks @ iK) * Ks).sum(1)
