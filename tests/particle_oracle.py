"""Numpy statement of the particle rollout (pilco_particles_rollout, DESIGN.md section 11) for the tests: P particles
from the caller's x0 [P,Ds], driven by the caller's standard normals eps [P,H,Ds], through a factorised dynamics GP
(centres C, ell, sf2, iK, beta) under a linear or RBF policy, with the reward terms evaluated at each particle's
pre-step state.  Test infrastructure only; vectorised over particles."""
import numpy as np

from pilco_b200 import _lib

RBF_VAR = 1e-6          # output variance of the deterministic-GP (RBF) policy at a point, as compute_action sees it


def se_k(Xs, C, ell, sf2):
    """sf2 exp(-0.5 |(x - c)/ell|^2) in the direct difference form -> [T, n]"""
    d = (Xs[:, None, :] - C[None, :, :]) / ell[None, None, :]
    return sf2 * np.exp(-0.5 * (d * d).sum(-1))


def gp_latent(dyn, Xs):
    """posterior mean and latent variance [T,E] of the factorised model dyn = dict(C, ell, sf2, iK, beta)"""
    C, ell, sf2, iK, beta = (dyn[k] for k in ("C", "ell", "sf2", "iK", "beta"))
    n = C.shape[0]
    M, V = [], []
    for e in range(ell.shape[0]):
        K = se_k(Xs, C, ell[e], sf2[e])
        M.append(K @ beta[e])
        V.append(sf2[e] - ((K @ iK[e][:n, :n]) * K).sum(1))
    return np.stack(M, 1), np.stack(V, 1)


def policy_action(pol, x):
    """squashed action [P,U]; pol = dict(kind, squash, maxa, W, b) (linear) or dict(kind, squash, maxa, C, ell, sf2,
    beta) (RBF: the deterministic GP's mean, its output variance RBF_VAR enters the squash as in compute_action)"""
    if pol["kind"] == _lib.POLICY_LINEAR:
        u, var = x @ np.asarray(pol["W"]).T + np.asarray(pol["b"]).reshape(1, -1), 0.0
    else:
        u = np.stack([se_k(x, pol["C"], pol["ell"][j], pol["sf2"][j]) @ pol["beta"][j]
                      for j in range(pol["ell"].shape[0])], 1)
        var = RBF_VAR
    if pol.get("squash", True):
        u = np.asarray(pol["maxa"]).reshape(1, -1) * np.exp(-0.5 * var) * np.sin(u)
    return u


def box_point(prm, x):
    nd, inside = int(prm[0]), prm[1] != 0.0
    ok = np.ones(x.shape[0], dtype=bool)
    for k in range(nd):
        v = x[:, int(prm[3 + 3 * k])]
        ok &= (prm[4 + 3 * k] < v) & (v < prm[5 + 3 * k])
    return (ok == inside).astype(np.float64)


def reward_value(term, x):
    """one reward term (engine dict: kind, W, t) at the points x [P,Ds] -> [P]"""
    W = np.asarray(term["W"], dtype=np.float64)
    if term["kind"] == _lib.REWARD_BOX:
        return box_point(W, x)
    if term["kind"] == _lib.REWARD_LINEAR:
        return x @ W.reshape(-1)
    d = x - np.asarray(term["t"], dtype=np.float64).reshape(1, -1)
    return np.exp(-0.5 * np.einsum("pi,ij,pj->p", d, W.reshape(d.shape[1], d.shape[1]), d))


def particle_rollout(dyn, pol, terms, x0, eps, mult_mu=0.0):
    """-> traj [P,H+1,Ds], act [P,H,U], step_reward [P,H], step_risk [P,H], ret [P]"""
    P, H, Ds = eps.shape
    x = np.asarray(x0, dtype=np.float64).copy()
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
        mu, var = gp_latent(dyn, np.hstack([x, u]))
        x = x + mu + np.sqrt(np.maximum(var, 0.0)) * eps[:, t]
        traj.append(x)
    ret = rew.sum(1)
    if any(int(t.get("channel", 0)) == _lib.CHANNEL_MULT for t in terms):
        ret = ret + mult_mu * (1.0 - np.prod(1.0 - risk, axis=1))
    U = act[0].shape[1] if act else 0
    return (np.stack(traj, 1), np.stack(act, 1) if act else np.zeros((P, 0, U)), rew, risk, ret)


def moment_check(samples, mean, cov, nse=5.0):
    """largest deviation, in standard errors estimated from the samples, of the sample mean and covariance of
    samples [P,Ds] from (mean [Ds], cov [Ds,Ds])"""
    P = samples.shape[0]
    xm = samples.mean(0)
    z = samples - xm
    worst = np.max(np.abs(xm - mean) / (samples.std(0) / np.sqrt(P)))
    for i in range(samples.shape[1]):
        for j in range(i + 1):
            zz = z[:, i] * z[:, j]
            worst = max(worst, abs(zz.mean() - cov[i, j]) / (zz.std() / np.sqrt(P)))
    return float(worst)
