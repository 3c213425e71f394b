"""Torch statement of PILCO's exploration objective in the particle rollouts (DESIGN.md section 24) for the tests:
tests/particle_noise_oracle.py's pathwise value with the sample spread of each step's reward added,

    value = mean_p ret_p + b sum_t sigma_t,   sigma_t^2 = sum_k c_k^2 Var_p[r_kpt]   (ADD terms, unbiased variance)
    sigma_t = sqrt(sigma_t^2) if sigma_t^2 > 1e-12, else 0 (constant)

with the state terms at the raw x_t and the joint terms at [phi(x_t), u_t].  At b = 0 the value and gradient are the
noise oracle's bitwise (the same graph: the bonus is not added).  Test infrastructure only."""
import numpy as np
import torch

import particle_angles_oracle as pao
import particle_grad_oracle as pgo
import particle_noise_oracle as pno
import particle_oracle as po

F64 = torch.float64
FLOOR = 1e-12


def _additive(terms):
    return [t for t in terms if not po.is_mult(t) and t["kind"] != 2]


def step_var(terms, value, P):
    """sigma_t^2 of one step (torch): sum_k c_k^2 torch.var(r_k, unbiased=True) over the additive terms, in term order"""
    var = torch.zeros((), dtype=F64)
    for term in _additive(terms):
        c = float(term.get("coef", 1.0))
        var = var + c * c * torch.var(value(term), unbiased=True)
    return var


def sigma(var):
    """section 21's floor: sqrt above 1e-12, else a constant 0"""
    return torch.sqrt(var) if float(var.detach()) > FLOOR else torch.zeros((), dtype=F64)


def _pathwise(pol, terms, x0, eps, nu, v, mult_mu, transition, angle_dims, b):
    P, H, E = eps.shape
    sv = pno._scale(v)
    prm, act = pgo.policy(pol)
    x, e = pgo.T(x0), pgo.T(eps)
    n = pgo.T(nu) if sv is not None else None
    rews, risks, svar = [], [], []
    for s in range(H):
        xf = pao.feature_map_torch(x, angle_dims)
        zf = xf if sv is None else pao.feature_map_torch(pno.measurement(x, n[:, s], sv), angle_dims)
        u = act(zf)
        val = lambda term: pgo.point_value(term, xf if po.is_joint(term) else x, u)
        r, k = po.step_values(terms, val, torch.zeros(P, dtype=F64))
        rews.append(r); risks.append(k)
        svar.append(step_var(terms, val, P))
        mean, var = transition(torch.cat([xf, u], 1), e[:, s])
        x = x + mean + torch.sqrt(var) * e[:, s]
    stack = lambda w: torch.stack(w, 1) if H else torch.zeros((P, 0), dtype=F64)
    value = po.particle_return(terms, stack(rews), stack(risks), mult_mu).mean()
    if b != 0.0 and H:
        bonus = torch.zeros((), dtype=F64)
        for sv2 in svar:
            bonus = bonus + sigma(sv2)
        value = value + b * bonus
    sv_np = np.array([float(s.detach()) for s in svar])
    return float(value.detach()), pgo._grads(value, prm), sv_np


def value_and_grad(dyn, pol, terms, x0, eps, nu=None, v=None, mult_mu=0.0, angle_dims=None, b=0.0):
    """pno.value_and_grad with the exploration bonus -> (value, grads, step_var [H])"""
    def transition(xt, e):
        mu, var = pgo.gp_latent(dyn, xt)
        return mu, torch.clamp(var, min=0.0)
    return _pathwise(pol, terms, x0, eps, nu, v, mult_mu, transition, angle_dims, b)


def consistent_value_and_grad(dyn, pol, terms, x0, eps, nu=None, v=None, mult_mu=0.0, angle_dims=None, b=0.0,
                              swap=False):
    """pno.consistent_value_and_grad with the exploration bonus -> (value, grads, step_var [H])"""
    fs = pgo.TorchFunctionSample(dyn, swap)
    return _pathwise(pol, terms, x0, eps, nu, v, mult_mu, fs.step, angle_dims, b)


def sample_moments(terms, traj, act, angle_dims=None):
    """(mean [H], var [H]) of the step rewards over the particles of traj [P,H+1,E], act [P,H,U] (numpy): mean_t =
    sum_k c_k mean_p r_kpt and var_t = sum_k c_k^2 Var_p[r_kpt] (ddof 1) over the additive terms"""
    P, H = act.shape[:2]
    mean, var = np.zeros(H), np.zeros(H)
    for t in range(H):
        x, xf = traj[:, t], pao.feature_map(traj[:, t], angle_dims)
        for term in _additive(terms):
            c = float(term.get("coef", 1.0))
            r = po.point_value(term, xf if po.is_joint(term) else x, act[:, t])
            mean[t] += c * r.mean()
            var[t] += c * c * r.var(ddof=1)
    return mean, var
