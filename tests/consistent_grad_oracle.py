"""Oracles of the consistent sampler's pathwise gradient (pilco_particles_rollout_consistent_grad, DESIGN.md section 15)
for the tests: tests/consistent_oracle.py transcribed to torch and differentiated w.r.t. the policy parameters at fixed
x0 and eps, with the same pivot mask and the tau rule in reverse (a degenerate step's own noise is held constant);
and the explicit numpy statement of the reverse steps 1-6 at a fixed input sequence.  Test infrastructure only."""
import numpy as np
import torch

from pilco_b200 import _lib
from consistent_oracle import TAU
from particle_grad_oracle import F64, _reward, _se, rbf_beta
from particle_oracle import RBF_VAR, se_k


class _TorchFunctionSample:
    """consistent_oracle.FunctionSample in torch: step(Xt [P,D], eps_t [P,E]) -> (mean' [P,E], var' [P,E])"""

    def __init__(self, dyn, swap=False):
        t = lambda a: torch.as_tensor(np.asarray(a, dtype=np.float64))
        self.C, self.ell, self.sf2, self.iK, self.beta = (t(dyn[k]) for k in ("C", "ell", "sf2", "iK", "beta"))
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
        mu = torch.stack([_se(Xt, self.C, self.ell[e], self.sf2[e]) @ self.beta[e] for e in range(self.E)], 1)
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
        mask = d2.detach() > TAU * self.sf2[None]
        if mask.any():
            self.min_ratio = min(self.min_ratio, float((d2.detach()[mask] / (TAU * self.sf2[None].expand_as(d2)[mask])).min()))
        vp = torch.clamp(d2, min=0.0)
        vp = torch.where(mask, vp, vp.detach())                 # the tau rule: a degenerate step's own noise is constant
        mean = mu + ((l * torch.stack(self.eps, -1)).sum(-1) if self.eps else 0.0)
        self.X.append(Xt); self.L.append(l); self.eps.append(eps_t)
        self.piv.append(torch.where(mask, torch.sqrt(torch.where(mask, d2, torch.ones_like(d2))), torch.zeros_like(d2)))
        return mean, vp


def value_and_grad(dyn, pol, terms, x0, eps, mult_mu=0.0, swap=False):
    """value = mean return of the consistent sampler and its gradient w.r.t. the policy parameters at fixed x0, eps;
    arguments as particle_grad_oracle.value_and_grad.  -> (value, grads, smallest kept pivot d2 / (TAU sf2))"""
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
    fs = _TorchFunctionSample(dyn, swap)
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
        mean, vp = fs.step(torch.cat([x, u], 1), e[:, s])
        x = x + mean + torch.sqrt(vp) * e[:, s]
    ret = rew
    if any(int(term.get("channel", 0)) == _lib.CHANNEL_MULT for term in terms) and H > 0:
        ret = ret + mult_mu * (1.0 - torch.prod(1.0 - torch.stack(risks, 1), 1))
    value = ret.mean()
    keys = list(prm)
    if not value.requires_grad:
        return float(value), {k: np.zeros(prm[k].shape) for k in keys}, fs.min_ratio
    grads = torch.autograd.grad(value, [prm[k] for k in keys], allow_unused=True)
    return (float(value.detach()), {k: (np.zeros(prm[k].shape) if g is None else g.numpy()) for k, g in zip(keys, grads)},
            fs.min_ratio)


def fixed_inputs_objective(dyn, Xs, eps, mbar, vbar):
    """sum_t sum_e mbar_te mean'_te + vbar_te var'_te of ONE particle's draw at the fixed inputs Xs [T,D] (torch,
    differentiable in Xs), with the tau rule of value_and_grad"""
    fs = _TorchFunctionSample(dyn)
    tot = 0.0
    for t in range(Xs.shape[0]):
        mean, vp = fs.step(Xs[t:t + 1], torch.as_tensor(eps[t:t + 1]))
        tot = tot + (torch.as_tensor(mbar[t]) * mean[0]).sum() + (torch.as_tensor(vbar[t]) * vp[0]).sum()
    return tot


def reverse_steps(dyn, Xs, eps, mbar, vbar):
    """d/dXs of fixed_inputs_objective by DESIGN.md section 15's steps 1-6, written out: Xs [T,D], eps, mbar, vbar [T,E]
    -> gX [T,D]"""
    C, ell, sf2, iK, beta = (dyn[k] for k in ("C", "ell", "sf2", "iK", "beta"))
    n, (T, D), E = C.shape[0], Xs.shape, ell.shape[0]
    gX = np.zeros((T, D))
    for e in range(E):
        K = se_k(Xs, C, ell[e], sf2[e])                            # K*_t rows [T,n]
        iKe = iK[e][:n, :n]
        kx = se_k(Xs, Xs, ell[e], sf2[e])                          # k_e(x~_t, x~_s)
        kp = kx - K @ iKe @ K.T                                    # the posterior covariance
        Lm, piv = np.zeros((T, T)), np.zeros(T)
        for t in range(T):                                         # the forward: rows l_t. and pivots
            for s in range(t):
                if piv[s] > 0.0:
                    Lm[t, s] = (kp[t, s] - Lm[s, :s] @ Lm[t, :s]) / piv[s]
            d2 = kp[t, t] - Lm[t, :t] @ Lm[t, :t]
            piv[t] = np.sqrt(d2) if d2 > TAU * sf2[e] else 0.0
        Lam, G = np.zeros((T, T)), np.zeros((T, T))
        for t in range(T - 1, -1, -1):
            db = vbar[t, e] + Lam[t, t] / (2.0 * piv[t]) if piv[t] > 0.0 else 0.0              # 1
            lb = Lam[t, :t] + mbar[t, e] * eps[:t, e] - 2.0 * db * Lm[t, :t]                   # 3
            for s in range(t - 1, -1, -1):                                                      # 4
                c = lb[s] / piv[s] if piv[s] > 0.0 else 0.0
                Lam[s, s] -= c * Lm[t, s]
                lb[:s] -= c * Lm[s, :s]
                Lam[s, :s] -= c * Lm[t, :s]
                G[t, s] = G[s, t] = c                                                           # 5
            others = np.arange(T) != t                                                          # 6
            a = -2.0 * db * K[t] - G[t, others] @ K[others]
            cn = K[t] * (mbar[t, e] * beta[e] + a @ iKe)
            direct = ((G[t, others] * kx[t, others])[:, None] * (Xs[others] - Xs[t])).sum(0)
            gX[t] += ((cn[:, None] * (C - Xs[t])).sum(0) + direct) / ell[e] ** 2
    return gX
