"""Torch statement of the Gaussian-resampled particle rollout for the tests (pilco_particles_resampled_*, DESIGN.md
section 26): tests/particle_oracle.py's step-wise sampler with the refit at every step t >= 1,

  x'_t = x_{t-1} + mu + sqrt(max(var, 0)) eps_{t-1},  mu^_t, S^_t = the sample mean and unbiased covariance of x'_t,
  x_t  = mu^_t + chol(S^_t) xi_{t-1}

with ``chol`` a Python-loop Cholesky that applies the device's degenerate-column rule (resample_math.cuh), so autograd
differentiates the factor as executed.  Test infrastructure only."""
import numpy as np
import torch

import particle_grad_oracle as pgo
import particle_oracle as po

F64 = torch.float64
TAU = 1e-12


def chol(S):
    """the column-by-column factor of S's lower triangle (torch, differentiable); a column whose pivot d_j <= TAU S_jj
    (or S_jj <= 0) is zero"""
    n = S.shape[0]
    zero = S.new_zeros(())
    L = [[zero] * n for _ in range(n)]
    for j in range(n):
        d = S[j, j]
        for k in range(j):
            d = d - L[j][k] * L[j][k]
        sjj, dv = float(S[j, j].detach()), float(d.detach())
        if not (sjj > 0.0 and dv > TAU * sjj):
            continue
        piv = torch.sqrt(d)
        L[j][j] = piv
        for i in range(j + 1, n):
            s = S[i, j]
            for k in range(j):
                s = s - L[i][k] * L[j][k]
            L[i][j] = s / piv
    return torch.stack([torch.stack(row) for row in L])


def chol_np(S):
    return chol(torch.as_tensor(np.asarray(S, dtype=np.float64))).numpy()


def chol_bwd_np(S, Lb):
    """d <Lb, chol(S)> / d S on S's lower triangle (its upper triangle is 0), by autograd"""
    St = torch.as_tensor(np.asarray(S, dtype=np.float64)).clone().requires_grad_()
    L = chol(St)
    if not L.requires_grad:
        return np.zeros_like(np.asarray(S, dtype=np.float64))
    g, = torch.autograd.grad((L * torch.as_tensor(np.asarray(Lb, dtype=np.float64))).sum(), St, allow_unused=True)
    return np.zeros_like(np.asarray(S, dtype=np.float64)) if g is None else np.tril(g.numpy())


def _moments(x):
    m = x.mean(0)
    c = x - m[None]
    return m, c.T @ c / (x.shape[0] - 1)


def rollout(dyn, pol, terms, x0, eps, xi, mult_mu=0.0):
    """-> dict(traj [P,H+1,Ds], act, rew, risk, ret, step_mean [H+1,Ds], step_cov [H+1,Ds,Ds], xp [H,P,Ds], value,
    grad) of one restart; grad = d value / d the policy parameters ({'W','b'} or {'X','Y','ell'}), value = mean
    return, x0, eps and xi held fixed"""
    P, H, Ds = eps.shape
    prm, act = pgo.policy(pol)
    x, e, z = pgo.T(x0), pgo.T(eps), pgo.T(xi)
    traj, acts, rews, risks, xps = [x], [], [], [], []
    m, S = _moments(x)
    means, covs = [m], [S]
    for t in range(H):
        u = act(x)
        r, k = po.step_values(terms, lambda term: pgo.point_value(term, x, u), torch.zeros(P, dtype=F64))
        rews.append(r); risks.append(k); acts.append(u)
        mu, var = pgo.gp_latent(dyn, torch.cat([x, u], 1))
        xp = x + mu + torch.sqrt(torch.clamp(var, min=0.0)) * e[:, t]
        m, S = _moments(xp)
        x = m[None] + z[:, t] @ chol(S).T
        traj.append(x); xps.append(xp); means.append(m); covs.append(S)
    stack = lambda v: torch.stack(v, 1) if H else torch.zeros((P, 0), dtype=F64)
    rew, risk = stack(rews), stack(risks)
    ret = po.particle_return(terms, rew, risk, mult_mu)
    value = ret.mean()
    grad = pgo._grads(value, prm)
    nd = lambda v: v.detach().numpy()
    return dict(traj=nd(torch.stack(traj, 1)), act=nd(torch.stack(acts, 1)) if H else np.zeros((P, 0, 0)),
                rew=nd(rew), risk=nd(risk), ret=nd(ret), step_mean=nd(torch.stack(means)),
                step_cov=nd(torch.stack(covs)), xp=nd(torch.stack(xps)) if H else np.zeros((0, P, Ds)),
                value=float(value.detach()), grad=grad)
