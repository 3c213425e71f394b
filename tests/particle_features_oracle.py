"""Function samples from random-feature draws with an exact data update (DESIGN.md section 30) in the shared particle
oracles, tests/particle_oracle.py (numpy) and tests/particle_grad_oracle.py (torch), without a copy of their step loops:
the draws give the transition x + f_p(x~) that both loops take.

    omega_ei = zeta_ei / ell_e,  phi_e(x) = sqrt(sf2_e / F) [cos(omega_e x); sin(omega_e x)]
    v_pe = beta_e - iK_e (Phi_e(X) w_pe + sqrt(sn2_e) eps_pe),  f_pe(x~) = phi_e(x~)' w_pe + k_e(x~, X) v_pe

dyn = dict(C, ell, sf2, iK, beta) as the shared oracles take it.  Test infrastructure only."""
import numpy as np
import torch

import particle_grad_oracle as pgo
import particle_oracle as po


def draw(dyn, sn2, zeta, w, eps_y):
    """(omega [E,F,D], v [P,E,n]) of the normals zeta [E,F,D], w [P,E,2F], eps_y [P,E,n]"""
    C, ell, sf2, iK, beta = (dyn[k] for k in ("C", "ell", "sf2", "iK", "beta"))
    n, E = C.shape[0], ell.shape[0]
    omega = zeta / ell[:, None, :]
    v = np.empty((w.shape[0], E, n))
    for e in range(E):
        Phi = features(C, omega[e], sf2[e])                                    # [n, 2F]
        R = w[:, e] @ Phi.T + np.sqrt(sn2[e]) * eps_y[:, e]                      # [P, n]
        v[:, e] = beta[e][None] - R @ iK[e][:n, :n].T
    return omega, v


def features(x, omega_e, sf2_e):
    """phi_e at the rows of x (numpy) -> [T, 2F]"""
    a = x @ omega_e.T
    return np.sqrt(sf2_e / omega_e.shape[0]) * np.hstack([np.cos(a), np.sin(a)])


def evaluate(dyn, omega, w, v, xt):
    """f_p(x~_p) [P,E] at one input per particle (numpy)"""
    C, ell, sf2 = dyn["C"], dyn["ell"], dyn["sf2"]
    out = np.empty((xt.shape[0], ell.shape[0]))
    for e in range(ell.shape[0]):
        out[:, e] = (features(xt, omega[e], sf2[e]) * w[:, e]).sum(1) + \
            (po.se_k(xt, C, ell[e], sf2[e]) * v[:, e]).sum(1)
    return out


def evaluate_torch(dyn, omega, w, v, xt):
    """``evaluate`` with xt a torch tensor (differentiable in xt)"""
    C, ell, sf2 = (pgo.T(dyn[k]) for k in ("C", "ell", "sf2"))
    om, w, v = pgo.T(omega), pgo.T(w), pgo.T(v)
    F = om.shape[1]
    cols = []
    for e in range(ell.shape[0]):
        a = xt @ om[e].T
        phi = torch.sqrt(sf2[e] / F) * torch.cat([torch.cos(a), torch.sin(a)], 1)
        d = (xt[:, None, :] - C[None]) / ell[e][None, None, :]
        k = sf2[e] * torch.exp(-0.5 * (d * d).sum(-1))
        cols.append((phi * w[:, e]).sum(1) + (k * v[:, e]).sum(1))
    return torch.stack(cols, 1)


def rollout(dyn, omega, w, v, pol, terms, x0, H, mult_mu=0.0, angle_dims=None, nu=None, var=None):
    """traj, act, step_reward, step_risk, ret of the feature sampler (numpy, the shared step loop)"""
    P, E = w.shape[0], dyn["ell"].shape[0]
    eps = np.zeros((P, H, E))
    return po._rollout(pol, terms, x0, eps, mult_mu, lambda x, xt, e: x + evaluate(dyn, omega, w, v, xt), angle_dims,
                       nu, var)


def value_and_grad(dyn, omega, w, v, pol, terms, x0, H, mult_mu=0.0, angle_dims=None, nu=None, var=None, b=None):
    """value = mean return of the feature sampler and its torch-autograd gradient w.r.t. the policy parameters (the
    shared pathwise loop) -> (value, grads, hist)"""
    P, E = w.shape[0], dyn["ell"].shape[0]
    eps = np.zeros((P, H, E))
    return pgo._pathwise(pol, terms, x0, eps, mult_mu, lambda x, xt, e: x + evaluate_torch(dyn, omega, w, v, xt),
                         angle_dims, nu, var, b)


def conditional_variance(dyn, sn2, omega, xs):
    """Var[f_e(x~) | omega] [T,E] of the sampler at the rows of xs given the frequencies:
    |phi(x~) - k_x~X iK Phi(X)|^2 + sn2 |iK k_Xx~|^2"""
    C, ell, sf2, iK = (dyn[k] for k in ("C", "ell", "sf2", "iK"))
    n = C.shape[0]
    out = np.empty((xs.shape[0], ell.shape[0]))
    for e in range(ell.shape[0]):
        k = po.se_k(xs, C, ell[e], sf2[e])                                       # [T, n]
        A = k @ iK[e][:n, :n]
        r = features(xs, omega[e], sf2[e]) - A @ features(C, omega[e], sf2[e])
        out[:, e] = (r * r).sum(1) + sn2[e] * (A * A).sum(1)
    return out
