"""Numpy statement of the consistent particle sampler (pilco_particles_rollout_consistent, DESIGN.md section 14) for
the tests: each particle follows ONE function per dynamics output drawn from the latent posterior
k_post(a, b) = k_e(a, b) - k(a, C) iK_e k(C, b), sampled sequentially along the particle's own inputs with the
semidefinite Cholesky rule (a pivot d2 <= TAU sf2_e leaves its column out of later substitutions).  Test
infrastructure only; vectorised over particles and outputs."""
import numpy as np

from pilco_b200 import _lib
from particle_oracle import policy_action, reward_value, se_k

TAU = 1e-10


def _posterior(dyn, A, B):
    """latent posterior covariance k_post(A, B) per output -> [E, |A|, |B|]"""
    C, ell, sf2, iK = (dyn[k] for k in ("C", "ell", "sf2", "iK"))
    n = C.shape[0]
    out = []
    for e in range(ell.shape[0]):
        Ka, Kb = se_k(A, C, ell[e], sf2[e]), se_k(B, C, ell[e], sf2[e])
        out.append(se_k(A, B, ell[e], sf2[e]) - Ka @ iK[e][:n, :n] @ Kb.T)
    return np.stack(out)


def _posterior_pairs(dyn, A, B, swap=False):
    """k_post(A_p, B_p) of row-wise pairs A, B [P,D] -> [P,E]; ``swap``: the quadratic form as k_A (iK k_B) instead of
    (k_A iK) k_B, the same value with other roundings"""
    C, ell, sf2, iK = (dyn[k] for k in ("C", "ell", "sf2", "iK"))
    n = C.shape[0]
    out = []
    for e in range(ell.shape[0]):
        Ka, Kb = se_k(A, C, ell[e], sf2[e]), se_k(B, C, ell[e], sf2[e])
        d = (A - B) / ell[e][None, :]
        q = (Ka * (Kb @ iK[e][:n, :n])).sum(1) if swap else ((Ka @ iK[e][:n, :n]) * Kb).sum(1)
        out.append(sf2[e] * np.exp(-0.5 * (d * d).sum(-1)) - q)
    return np.stack(out, 1)


def _mean(dyn, A):
    C, ell, sf2, beta = (dyn[k] for k in ("C", "ell", "sf2", "beta"))
    return np.stack([se_k(A, C, ell[e], sf2[e]) @ beta[e] for e in range(ell.shape[0])], 1)


class FunctionSample:
    """The running state of one draw per (particle, output): the visited inputs and the packed factor rows.
    ``step(Xt, eps_t)`` -> f(Xt) [P,E] given the draws at the earlier inputs."""

    def __init__(self, dyn, P, swap=False):
        self.dyn, self.P, self.swap = dyn, P, swap
        self.E = dyn["ell"].shape[0]
        self.X = []              # visited inputs, each [P,D]
        self.L = []              # rows l [P,E,s] of the factor, below the diagonal
        self.piv = []            # pivots [P,E] (0: degenerate column)
        self.eps = []            # the normals [P,E] of the earlier steps

    def step(self, Xt, eps_t):
        dyn, P, E, t = self.dyn, self.P, self.E, len(self.X)
        sf2 = np.asarray(dyn["sf2"]).reshape(1, E)
        mu = _mean(dyn, Xt)
        var = _posterior_pairs(dyn, Xt, Xt, self.swap)      # [P,E]
        l = np.zeros((P, E, t))
        for s in range(t):                                  # forward substitution, one column at a time
            c = _posterior_pairs(dyn, Xt, self.X[s], self.swap)
            sub = (self.L[s] * l[:, :, :s]).sum(-1) if s else 0.0
            piv = self.piv[s]
            l[:, :, s] = np.where(piv > 0.0, (c - sub) / np.where(piv > 0.0, piv, 1.0), 0.0)
        d2 = var - (l * l).sum(-1)
        f = mu + np.sqrt(np.maximum(d2, 0.0)) * eps_t
        if t:
            f = f + (l * np.stack(self.eps, -1)).sum(-1)
        self.X.append(Xt.copy()); self.L.append(l); self.eps.append(eps_t.copy())
        self.piv.append(np.where(d2 > TAU * sf2, np.sqrt(np.maximum(d2, 0.0)), 0.0))
        return f


def joint_draw(dyn, Xs, eps):
    """f at the fixed inputs Xs [T,D] from the normals eps [T,E] as mu + chol(K_post) eps, per output (K_post positive
    definite) -> [T,E]"""
    K = _posterior(dyn, Xs, Xs)
    mu = _mean(dyn, Xs)
    return mu + np.stack([np.linalg.cholesky(K[e]) @ eps[:, e] for e in range(K.shape[0])], 1)


def consistent_rollout(dyn, pol, terms, x0, eps, mult_mu=0.0, swap=False):
    """-> traj [P,H+1,Ds], act [P,H,U], step_reward [P,H], step_risk [P,H], ret [P] of the consistent sampler with
    the caller's x0 [P,Ds] and normals eps [P,H,Ds] (eps[:, t] is the step-t normal of every output).  ``swap``
    reorders the posterior's sums: the difference of the two is the sampler's own sensitivity to rounding"""
    P, H, Ds = eps.shape
    x = np.asarray(x0, dtype=np.float64).copy()
    fs = FunctionSample(dyn, P, swap)
    traj, act, rew, risk = [x], [], np.zeros((P, H)), np.zeros((P, H))
    for t in range(H):
        for term in terms:
            v = float(term.get("coef", 1.0)) * reward_value(term, x)
            if int(term.get("channel", _lib.CHANNEL_ADD)) == _lib.CHANNEL_MULT:
                risk[:, t] += v
            else:
                rew[:, t] += v
        u = policy_action(pol, x)
        act.append(u)
        x = x + fs.step(np.hstack([x, u]), eps[:, t])
        traj.append(x)
    ret = rew.sum(1)
    if any(int(t.get("channel", 0)) == _lib.CHANNEL_MULT for t in terms):
        ret = ret + mult_mu * (1.0 - np.prod(1.0 - risk, axis=1))
    U = act[0].shape[1] if act else 0
    return (np.stack(traj, 1), np.stack(act, 1) if act else np.zeros((P, 0, U)), rew, risk, ret)
