"""Torch statement of the particle rollouts' policy gradients for the tests: tests/particle_oracle.py transcribed to
torch and differentiated w.r.t. the policy parameters at fixed x0 and eps.

  * ``value_and_grad``: the step-wise sampler's pathwise gradient (pilco_particles_rollout_grad, DESIGN.md section 12);
  * ``consistent_value_and_grad``: the consistent sampler's (pilco_particles_rollout_consistent_grad, section 15), with
    the same pivot mask and the tau rule in reverse (a degenerate step's own noise is held constant), and the explicit
    numpy statement of its reverse steps 1-6 at a fixed input sequence (``reverse_steps``);
  * ``score_grad``: the score-function gradient (pilco_particles_rollout_score_grad, section 16) plus the joint terms'
    direct dependence on the policy (section 18).

The RBF policy's beta = (K + sn2 I)^-1 Yc goes through a Cholesky solve, so the gradient w.r.t. the centres, targets and
lengthscales includes the factorisation, as the device's does.  Also the closed form of the predict VJP
(pilco_gp_predict_vjp) in numpy.  Test infrastructure only."""
import numpy as np
import torch

from pilco_b200 import _lib
import particle_oracle as po

F64 = torch.float64
T = lambda a: torch.as_tensor(np.asarray(a, dtype=np.float64))


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


def policy(pol):
    """(parameters with requires_grad, x -> squashed action) of pol = dict(kind, squash, maxa, W, b) or dict(kind,
    squash, maxa, Xc, Yc, ell, sf2, sn2); the parameters are {'W','b'} or {'X','Y','ell'}"""
    if pol["kind"] == _lib.POLICY_LINEAR:
        prm = {"W": T(pol["W"]).clone().requires_grad_(), "b": T(pol["b"]).reshape(-1).clone().requires_grad_()}
        raw, su = (lambda x: x @ prm["W"].T + prm["b"][None]), 0.0
    else:
        prm = {k: T(pol[s]).clone().requires_grad_() for k, s in (("X", "Xc"), ("Y", "Yc"), ("ell", "ell"))}
        beta = rbf_beta(prm["X"], prm["Y"], prm["ell"], pol["sf2"], pol["sn2"])
        raw = lambda x: torch.stack([_se(x, prm["X"], prm["ell"][j], float(pol["sf2"][j])) @ beta[j]
                                     for j in range(beta.shape[0])], 1)
        su = po.RBF_VAR
    maxa = T(pol["maxa"]).reshape(1, -1)
    act = (lambda x: maxa * np.exp(-0.5 * su) * torch.sin(raw(x))) if pol.get("squash", True) else raw
    return prm, act


def point_value(term, x, u):
    """particle_oracle.point_value in torch (box terms: value only, flat almost everywhere)"""
    W = T(term["W"])
    if term["kind"] == _lib.REWARD_BOX:
        return T(po.box_point(W.numpy(), x.detach().numpy()))
    z = torch.cat([x, u], 1) if po.is_joint(term) else x
    if term["kind"] in (_lib.REWARD_LINEAR, _lib.REWARD_LINEAR_SA):
        return z @ W.reshape(-1)
    d = z - T(term["t"]).reshape(1, -1)
    return torch.exp(-0.5 * torch.einsum("pi,ij,pj->p", d, W.reshape(d.shape[1], d.shape[1]), d))


def gp_latent(dyn, xt):
    """particle_oracle.gp_latent in torch -> mean, latent variance [T,E]"""
    C, ell, sf2, iK, bd = (T(dyn[k]) for k in ("C", "ell", "sf2", "iK", "beta"))
    n = C.shape[0]
    mu, var = [], []
    for k in range(ell.shape[0]):
        K = _se(xt, C, ell[k], sf2[k])
        mu.append(K @ bd[k])
        var.append(sf2[k] - ((K @ iK[k][:n, :n]) * K).sum(1))
    return torch.stack(mu, 1), torch.stack(var, 1)


class TorchFunctionSample:
    """particle_oracle.FunctionSample in torch: step(Xt [P,D], eps_t [P,E]) -> (mean' [P,E], var' [P,E])"""

    def __init__(self, dyn, swap=False):
        self.dyn = dyn
        self.C, self.ell, self.sf2, self.iK = (T(dyn[k]) for k in ("C", "ell", "sf2", "iK"))
        self.n, self.E, self.swap = self.C.shape[0], self.ell.shape[0], swap
        self.X, self.L, self.piv, self.eps = [], [], [], []
        self.min_ratio = np.inf                 # the smallest pivot d2 / (TAU sf2) kept by the mask

    def _pairs(self, A, B):
        out = []
        for e in range(self.E):
            Ka, Kb = _se(A, self.C, self.ell[e], self.sf2[e]), _se(B, self.C, self.ell[e], self.sf2[e])
            iK = self.iK[e][:self.n, :self.n]
            q = (Ka * (Kb @ iK)).sum(1) if self.swap else ((Ka @ iK) * Kb).sum(1)
            d = (A - B) / self.ell[e][None, :]
            out.append(self.sf2[e] * torch.exp(-0.5 * (d * d).sum(-1)) - q)
        return torch.stack(out, 1)

    def step(self, Xt, eps_t):
        mu = gp_latent(self.dyn, Xt)[0]
        var = self._pairs(Xt, Xt)
        cols = []
        for s in range(len(self.X)):
            c = self._pairs(Xt, self.X[s])
            if s:
                c = c - (self.L[s] * torch.stack(cols, -1)).sum(-1)
            piv = self.piv[s]
            cols.append(torch.where(piv > 0.0, c / torch.where(piv > 0.0, piv, torch.ones_like(piv)), torch.zeros_like(c)))
        l = torch.stack(cols, -1) if cols else torch.zeros(Xt.shape[0], self.E, 0, dtype=F64)
        d2 = var - (l * l).sum(-1)
        mask = d2.detach() > po.TAU * self.sf2[None]
        if mask.any():
            self.min_ratio = min(self.min_ratio, float((d2.detach()[mask] / (po.TAU * self.sf2[None].expand_as(d2)[mask])).min()))
        vp = torch.clamp(d2, min=0.0)
        vp = torch.where(mask, vp, vp.detach())                 # the tau rule: a degenerate step's own noise is constant
        mean = mu + ((l * torch.stack(self.eps, -1)).sum(-1) if self.eps else 0.0)
        self.X.append(Xt); self.L.append(l); self.eps.append(eps_t)
        self.piv.append(torch.where(mask, torch.sqrt(torch.where(mask, d2, torch.ones_like(d2))), torch.zeros_like(d2)))
        return mean, vp


def _grads(value, prm):
    keys = list(prm)
    if not value.requires_grad:                 # e.g. H = 0: nothing depends on the policy
        return {k: np.zeros(prm[k].shape) for k in keys}
    g = torch.autograd.grad(value, [prm[k] for k in keys], allow_unused=True)
    return {k: (np.zeros(prm[k].shape) if gi is None else gi.numpy()) for k, gi in zip(keys, g)}


def _pathwise(pol, terms, x0, eps, mult_mu, transition):
    """mean particle return and its gradient; ``transition([x, u], eps_t)`` -> (mean, var) of the step's increment"""
    P, H, Ds = eps.shape
    prm, act = policy(pol)
    x, e = T(x0), T(eps)
    rews, risks = [], []
    for s in range(H):
        u = act(x)
        r, k = po.step_values(terms, lambda term: point_value(term, x, u), torch.zeros(P, dtype=F64))
        rews.append(r); risks.append(k)
        mean, var = transition(torch.cat([x, u], 1), e[:, s])
        x = x + mean + torch.sqrt(var) * e[:, s]
    stack = lambda v: torch.stack(v, 1) if H else torch.zeros((P, 0), dtype=F64)
    value = po.particle_return(terms, stack(rews), stack(risks), mult_mu).mean()
    return float(value.detach()), _grads(value, prm)


def value_and_grad(dyn, pol, terms, x0, eps, mult_mu=0.0):
    """value = mean return of the step-wise sampler and its gradient w.r.t. the policy parameters at fixed x0, eps.
    dyn = dict(C, ell, sf2, iK, beta) (numpy); pol as ``policy`` takes it.  -> (value, {'W','b'} or {'X','Y','ell'})"""
    def transition(xt, e):
        mu, var = gp_latent(dyn, xt)
        return mu, torch.clamp(var, min=0.0)
    return _pathwise(pol, terms, x0, eps, mult_mu, transition)


def consistent_value_and_grad(dyn, pol, terms, x0, eps, mult_mu=0.0, swap=False):
    """``value_and_grad`` of the consistent sampler -> (value, grads, smallest kept pivot d2 / (TAU sf2))"""
    fs = TorchFunctionSample(dyn, swap)
    return _pathwise(pol, terms, x0, eps, mult_mu, fs.step) + (fs.min_ratio,)


def score_grad(dyn, pol, terms, traj, eps, mult_mu=0.0, baseline=True, direct=True, transitions=True):
    """The score-function gradient of the mean return over the rollout (traj [P,H+1,Ds], eps [P,H,Ds]; the device's,
    or particle_oracle's), pol as ``policy`` takes it.  With ``transitions`` the surrogate

        (1/P) sum_p sum_{t < H-1} w_pt log N(y_pt; mu(x~_t(theta)), var(x~_t(theta))),   y = mu(theta0) + s(theta0) eps

    is differentiated with w (``weights``), x_t and y held fixed: its gradient at theta0 is that of
    sum w (eps / s0 mu(theta) + (eps^2 - 1) / (2 var0) var(theta)) (0 where var0 <= 0), which is what is formed here.
    With ``direct``, the joint terms' own dependence on the parameters through u_t = pi(x_t) at fixed states,
    (1/P) sum_p sum_{t<H} a_kt v_k([x_pt, pi(x_pt)]), is added.  -> {'W','b'} or {'X','Y','ell'} numpy arrays"""
    traj, eps = np.asarray(traj, dtype=np.float64), np.asarray(eps, dtype=np.float64)
    P, H, Ds = eps.shape
    prm, act = policy(pol)
    if H == 0:
        return _grads(torch.zeros(()), prm)
    xs = [T(traj[:, s]) for s in range(H)]
    us = [act(x) for x in xs]
    rew, risk = po.path_rewards(terms, traj, np.stack([u.detach().numpy() for u in us], 1))
    G = po.weights(terms, rew, risk, mult_mu, baseline)
    mult = any(po.is_mult(t) for t in terms)
    sur = torch.zeros((), dtype=F64)
    for s, (x, u) in enumerate(zip(xs, us)):
        if transitions and s < H - 1:
            mu, var = gp_latent(dyn, torch.cat([x, u], 1))
            v0, e = var.detach(), T(eps[:, s])
            pos = v0 > 0.0
            safe = torch.where(pos, v0, torch.ones_like(v0))
            a = torch.where(pos, e / torch.sqrt(safe), torch.zeros_like(v0))
            b = torch.where(pos, (e * e - 1.0) / (2.0 * safe), torch.zeros_like(v0))
            sur = sur + (T(G[:, s])[:, None] * (a * mu + b * var)).sum()
        if direct:
            wm = mult_mu * np.prod(np.delete(1.0 - risk, s, axis=1), axis=1) if mult else np.zeros(P)
            for term in terms:
                if po.is_joint(term):
                    w = float(term.get("coef", 1.0)) * (T(wm) if po.is_mult(term) else 1.0)
                    sur = sur + (w * point_value(term, x, u)).sum()
    return _grads(sur / P, prm)


def fixed_inputs_objective(dyn, Xs, eps, mbar, vbar):
    """sum_t sum_e mbar_te mean'_te + vbar_te var'_te of ONE particle's draw at the fixed inputs Xs [T,D] (torch,
    differentiable in Xs), with the tau rule of consistent_value_and_grad"""
    fs = TorchFunctionSample(dyn)
    tot = 0.0
    for t in range(Xs.shape[0]):
        mean, vp = fs.step(Xs[t:t + 1], torch.as_tensor(eps[t:t + 1]))
        tot = tot + (torch.as_tensor(mbar[t]) * mean[0]).sum() + (torch.as_tensor(vbar[t]) * vp[0]).sum()
    return tot


def reverse_steps(dyn, Xs, eps, mbar, vbar):
    """d/dXs of fixed_inputs_objective by DESIGN.md section 15's steps 1-6, written out: Xs [T,D], eps, mbar, vbar [T,E]
    -> gX [T,D]"""
    C, ell, sf2, iK, beta = (dyn[k] for k in ("C", "ell", "sf2", "iK", "beta"))
    n, (T_, D), E = C.shape[0], Xs.shape, ell.shape[0]
    gX = np.zeros((T_, D))
    for e in range(E):
        K = po.se_k(Xs, C, ell[e], sf2[e])                         # K*_t rows [T,n]
        iKe = iK[e][:n, :n]
        kx = po.se_k(Xs, Xs, ell[e], sf2[e])                       # k_e(x~_t, x~_s)
        kp = kx - K @ iKe @ K.T                                    # the posterior covariance
        Lm, piv = np.zeros((T_, T_)), np.zeros(T_)
        for t in range(T_):                                        # the forward: rows l_t. and pivots
            for s in range(t):
                if piv[s] > 0.0:
                    Lm[t, s] = (kp[t, s] - Lm[s, :s] @ Lm[t, :s]) / piv[s]
            d2 = kp[t, t] - Lm[t, :t] @ Lm[t, :t]
            piv[t] = np.sqrt(d2) if d2 > po.TAU * sf2[e] else 0.0
        Lam, G = np.zeros((T_, T_)), np.zeros((T_, T_))
        for t in range(T_ - 1, -1, -1):
            db = vbar[t, e] + Lam[t, t] / (2.0 * piv[t]) if piv[t] > 0.0 else 0.0              # 1
            lb = Lam[t, :t] + mbar[t, e] * eps[:t, e] - 2.0 * db * Lm[t, :t]                   # 3
            for s in range(t - 1, -1, -1):                                                      # 4
                c = lb[s] / piv[s] if piv[s] > 0.0 else 0.0
                Lam[s, s] -= c * Lm[t, s]
                lb[:s] -= c * Lm[s, :s]
                Lam[s, :s] -= c * Lm[t, :s]
                G[t, s] = G[s, t] = c                                                           # 5
            others = np.arange(T_) != t                                                         # 6
            a = -2.0 * db * K[t] - G[t, others] @ K[others]
            cn = K[t] * (mbar[t, e] * beta[e] + a @ iKe)
            direct = ((G[t, others] * kx[t, others])[:, None] * (Xs[others] - Xs[t])).sum(0)
            gX[t] += ((cn[:, None] * (C - Xs[t])).sum(0) + direct) / ell[e] ** 2
    return gX


def predict_vjp(dyn, Xs, gmean, gvar):
    """closed form of pilco_gp_predict_vjp in numpy -> (gXs [T,D], scale [T,D]: the sum of |terms|, with |iK| k for w)"""
    C, ell, sf2, iK, beta = (dyn[k] for k in ("C", "ell", "sf2", "iK", "beta"))
    n = C.shape[0]
    g, scale = np.zeros(Xs.shape), np.zeros(Xs.shape)
    diff = C[None, :, :] - Xs[:, None, :]                         # [T,n,D]
    for e in range(ell.shape[0]):
        K = po.se_k(Xs, C, ell[e], sf2[e])
        w = K @ iK[e][:n, :n]
        c = K * (gmean[:, e:e + 1] * beta[e][None] - 2.0 * gvar[:, e:e + 1] * w)
        g += (c[:, :, None] * diff).sum(1) / ell[e] ** 2
        # the rounding of w = iK k is bounded by sum |iK| k, not by |w|: that enters the scale
        ca = K * (np.abs(gmean[:, e:e + 1] * beta[e][None]) + 2.0 * np.abs(gvar[:, e:e + 1]) * (K @ np.abs(iK[e][:n, :n])))
        scale += (ca[:, :, None] * np.abs(diff)).sum(1) / ell[e] ** 2
    return g, scale
