"""Torch statement of the particle rollout's score-function gradient (pilco_particles_rollout_score_grad, DESIGN.md
section 16) for the tests.  Given a rollout's trajectories, x0 and eps (the device's, or tests/particle_oracle.py's), the
surrogate

    (1/P) sum_p sum_{t < H-1} w_pt log N(y_pt; mu(x~_t(theta)), var(x~_t(theta))),   y = mu(theta0) + s(theta0) eps

is differentiated w.r.t. the policy parameters with w, x_t and y held fixed.  Its gradient at theta0 is that of
sum w (eps / s0 mu(theta) + (eps^2 - 1) / (2 var0) var(theta)) (0 where var0 <= 0), which is what is formed here: the
log density itself would cancel y - mu.  The RBF policy's beta goes through the Cholesky solve, as
tests/particle_grad_oracle.py's.  Test infrastructure only."""
import numpy as np
import torch

from pilco_b200 import _lib
from particle_oracle import RBF_VAR, reward_value
from particle_grad_oracle import _se, rbf_beta

F64 = torch.float64


def weights(terms, traj, mult_mu=0.0, baseline=True):
    """w [P, H-1]: the return-to-go G_pt of every transition t < H-1 from the reward terms at traj [P,H+1,Ds], minus
    the leave-one-out mean of the other particles' G_qt when ``baseline`` (and P > 1)"""
    traj = np.asarray(traj, dtype=np.float64)
    P, H = traj.shape[0], traj.shape[1] - 1
    rew, risk = np.zeros((P, H)), np.zeros((P, H))
    for t in range(H):
        for term in terms:
            v = float(term.get("coef", 1.0)) * reward_value(term, traj[:, t])
            if int(term.get("channel", _lib.CHANNEL_ADD)) == _lib.CHANNEL_MULT:
                risk[:, t] += v
            else:
                rew[:, t] += v
    mult = any(int(term.get("channel", 0)) == _lib.CHANNEL_MULT for term in terms)
    G = np.zeros((P, max(H - 1, 0)))
    for t in range(H - 1):
        G[:, t] = rew[:, t + 1:].sum(1)
        if mult:
            G[:, t] += mult_mu * np.prod(1.0 - risk[:, :t + 1], 1) * (1.0 - np.prod(1.0 - risk[:, t + 1:], 1))
    if baseline and P > 1:
        G = G - (G.sum(0, keepdims=True) - G) / (P - 1)
    return G


def score_grad(dyn, pol, terms, traj, eps, mult_mu=0.0, baseline=True):
    """the score-function gradient of the mean return over the rollout (traj [P,H+1,Ds], eps [P,H,Ds]).
    dyn = dict(C, ell, sf2, iK, beta) (numpy); pol = dict(kind, squash, maxa, W, b) or dict(kind, squash, maxa, Xc, Yc,
    ell, sf2, sn2), as particle_grad_oracle.value_and_grad.  -> {'W','b'} or {'X','Y','ell'} numpy arrays"""
    traj, eps = np.asarray(traj, dtype=np.float64), np.asarray(eps, dtype=np.float64)
    P, H, Ds = eps.shape
    t = lambda a: torch.as_tensor(np.asarray(a, dtype=np.float64))
    if pol["kind"] == _lib.POLICY_LINEAR:
        prm = {"W": t(pol["W"]).clone().requires_grad_(), "b": t(pol["b"]).reshape(-1).clone().requires_grad_()}
        act = lambda x: x @ prm["W"].T + prm["b"][None]
        su = 0.0
    else:
        prm = {k: t(pol[s]).clone().requires_grad_() for k, s in (("X", "Xc"), ("Y", "Yc"), ("ell", "ell"))}
        beta = rbf_beta(prm["X"], prm["Y"], prm["ell"], pol["sf2"], pol["sn2"])
        act = lambda x: torch.stack([_se(x, prm["X"], prm["ell"][j], float(pol["sf2"][j])) @ beta[j]
                                     for j in range(beta.shape[0])], 1)
        su = RBF_VAR
    keys = list(prm)
    if H < 2:                                   # the last transition carries no reward: nothing to differentiate
        return {k: np.zeros(prm[k].shape) for k in keys}
    w = t(weights(terms, traj, mult_mu, baseline))
    maxa = t(pol["maxa"]).reshape(1, -1)
    C, ell, sf2, iK, bd = (t(dyn[k]) for k in ("C", "ell", "sf2", "iK", "beta"))
    n = C.shape[0]
    sur = torch.zeros((), dtype=F64)
    for s in range(H - 1):
        x = t(traj[:, s])
        u = act(x)
        if pol.get("squash", True):
            u = maxa * np.exp(-0.5 * su) * torch.sin(u)
        xt = torch.cat([x, u], 1)
        e = t(eps[:, s])
        for k in range(Ds):
            K = _se(xt, C, ell[k], sf2[k])
            mu = K @ bd[k]
            var = sf2[k] - ((K @ iK[k][:n, :n]) * K).sum(1)
            v0 = var.detach()
            pos = v0 > 0.0
            safe = torch.where(pos, v0, torch.ones_like(v0))
            a = torch.where(pos, e[:, k] / torch.sqrt(safe), torch.zeros_like(v0))
            b = torch.where(pos, (e[:, k] * e[:, k] - 1.0) / (2.0 * safe), torch.zeros_like(v0))
            sur = sur + (w[:, s] * (a * mu + b * var)).sum()
    grads = torch.autograd.grad(sur / P, [prm[k] for k in keys], allow_unused=True)
    return {k: (np.zeros(prm[k].shape) if g is None else g.numpy()) for k, g in zip(keys, grads)}
