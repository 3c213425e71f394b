"""Torch autograd statement of the particle rollout's pathwise gradient (pilco_particles_rollout_grad, DESIGN.md
section 12) for the tests: tests/particle_oracle.py transcribed to torch, differentiated w.r.t. the policy parameters
at fixed x0 and eps.  The RBF policy's beta = (K + sn2 I)^-1 Yc goes through a Cholesky solve, so the gradient
w.r.t. the centres, targets and lengthscales includes the factorisation, as the device's does.  Also the closed form
of the predict VJP (pilco_gp_predict_vjp) in numpy.  Test infrastructure only."""
import numpy as np
import torch

from pilco_b200 import _lib
from particle_oracle import RBF_VAR, box_point, se_k

F64 = torch.float64


def _se(Xs, C, ell, sf2):
    d = (Xs[:, None, :] - C[None, :, :]) / ell[None, None, :]
    return sf2 * torch.exp(-0.5 * (d * d).sum(-1))


def rbf_beta(Xc, Yc, ell, sf2, sn2):
    """beta [U,bf] = (K_j + sn2_j I)^-1 Yc[:, j] through a Cholesky solve (torch or numpy inputs, torch out)"""
    Xc, Yc, ell = (torch.as_tensor(a, dtype=F64) for a in (Xc, Yc, ell))
    bf = Xc.shape[0]
    out = []
    for j in range(Yc.shape[1]):
        K = _se(Xc, Xc, ell[j], float(sf2[j])) + float(sn2[j]) * torch.eye(bf, dtype=F64)
        out.append(torch.cholesky_solve(Yc[:, j:j + 1], torch.linalg.cholesky(K))[:, 0])
    return torch.stack(out, 0)


def rbf_pol_np(Xc, Yc, ell, maxa, sf2=None, sn2=None, squash=True):
    """the numpy oracle's RBF policy dict for the parameters (Xc [bf,Ds], Yc [bf,U], ell [U,Ds])"""
    U = Yc.shape[1]
    sf2 = np.ones(U) if sf2 is None else sf2
    sn2 = 1e-4 * np.ones(U) if sn2 is None else sn2
    return dict(kind=_lib.POLICY_RBF, squash=squash, maxa=maxa, C=Xc, ell=ell, sf2=sf2,
                beta=rbf_beta(Xc, Yc, ell, sf2, sn2).numpy())


def _reward(term, x):
    W = torch.as_tensor(np.asarray(term["W"], dtype=np.float64))
    if term["kind"] == _lib.REWARD_BOX:            # flat almost everywhere: value only
        return torch.as_tensor(box_point(W.numpy(), x.detach().numpy()))
    if term["kind"] == _lib.REWARD_LINEAR:
        return x @ W.reshape(-1)
    d = x - torch.as_tensor(np.asarray(term["t"], dtype=np.float64)).reshape(1, -1)
    Ds = d.shape[1]
    return torch.exp(-0.5 * torch.einsum("pi,ij,pj->p", d, W.reshape(Ds, Ds), d))


def value_and_grad(dyn, pol, terms, x0, eps, mult_mu=0.0):
    """value = mean particle return and its gradient w.r.t. the policy parameters at fixed x0, eps.
    dyn = dict(C, ell, sf2, iK, beta) (numpy); pol = dict(kind, squash, maxa, W, b) or dict(kind, squash, maxa, Xc, Yc,
    ell, sf2, sn2).  -> (value, {'W','b'} or {'X','Y','ell'} numpy arrays)"""
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
    maxa = t(pol["maxa"]).reshape(1, -1)
    C, ell, sf2, iK, bd = (t(dyn[k]) for k in ("C", "ell", "sf2", "iK", "beta"))
    n = C.shape[0]
    x, e = t(x0), t(eps)
    rew, risks = torch.zeros(P, dtype=F64), []
    for s in range(H):
        risk = torch.zeros(P, dtype=F64)
        for term in terms:
            v = float(term.get("coef", 1.0)) * _reward(term, x)
            if int(term.get("channel", _lib.CHANNEL_ADD)) == _lib.CHANNEL_MULT:
                risk = risk + v
            else:
                rew = rew + v
        risks.append(risk)
        u = act(x)
        if pol.get("squash", True):
            u = maxa * np.exp(-0.5 * su) * torch.sin(u)
        xt = torch.cat([x, u], 1)
        mu, var = [], []
        for k in range(ell.shape[0]):
            K = _se(xt, C, ell[k], sf2[k])
            mu.append(K @ bd[k])
            var.append(sf2[k] - ((K @ iK[k][:n, :n]) * K).sum(1))
        x = x + torch.stack(mu, 1) + torch.sqrt(torch.clamp(torch.stack(var, 1), min=0.0)) * e[:, s]
    ret = rew
    if any(int(term.get("channel", 0)) == _lib.CHANNEL_MULT for term in terms) and H > 0:
        ret = ret + mult_mu * (1.0 - torch.prod(1.0 - torch.stack(risks, 1), 1))
    value = ret.mean()
    keys = list(prm)
    if not value.requires_grad:                 # H = 0: the return does not depend on the policy
        return float(value), {k: np.zeros(prm[k].shape) for k in keys}
    grads = torch.autograd.grad(value, [prm[k] for k in keys], allow_unused=True)
    return float(value.detach()), {k: (np.zeros(prm[k].shape) if g is None else g.numpy()) for k, g in zip(keys, grads)}


def predict_vjp(dyn, Xs, gmean, gvar):
    """closed form of pilco_gp_predict_vjp in numpy -> (gXs [T,D], scale [T,D]: the sum of |terms|, with |iK| k for w)"""
    C, ell, sf2, iK, beta = (dyn[k] for k in ("C", "ell", "sf2", "iK", "beta"))
    n = C.shape[0]
    g, scale = np.zeros(Xs.shape), np.zeros(Xs.shape)
    diff = C[None, :, :] - Xs[:, None, :]                         # [T,n,D]
    for e in range(ell.shape[0]):
        K = se_k(Xs, C, ell[e], sf2[e])
        w = K @ iK[e][:n, :n]
        c = K * (gmean[:, e:e + 1] * beta[e][None] - 2.0 * gvar[:, e:e + 1] * w)
        g += (c[:, :, None] * diff).sum(1) / ell[e] ** 2
        # the rounding of w = iK k is bounded by sum |iK| k, not by |w|: that enters the scale
        ca = K * (np.abs(gmean[:, e:e + 1] * beta[e][None]) + 2.0 * np.abs(gvar[:, e:e + 1]) * (K @ np.abs(iK[e][:n, :n])))
        scale += (ca[:, :, None] * np.abs(diff)).sum(1) / ell[e] ** 2
    return g, scale
