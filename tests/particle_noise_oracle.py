"""Numpy and torch statement of the particle rollouts with measurement noise at the policy's input (DESIGN.md section
23) for the tests: tests/particle_angles_oracle.py with the policy reading the measurement

    z_t = x_t + sqrt(v) o nu_t,   u_t = pi(phi(z_t)),   x~_t = [phi(x_t), u_t]

(nu [P,H,E] standard normals, v [E] variances).  The state, the state terms, the joint terms' phi(x) and the GP's
outputs are those of the angle oracle.  With v None or all zero the measurement is x itself (the same object, so the
autograd graph is the angle oracle's too) and every function computes bitwise what the angle oracle computes.  Test
infrastructure only."""
import numpy as np
import torch

import particle_angles_oracle as pao
import particle_grad_oracle as pgo
import particle_oracle as po

F64 = torch.float64


def _scale(v):
    """sqrt(v) [E], or None for no noise (v None or all zero)"""
    if v is None:
        return None
    v = np.asarray(v, dtype=np.float64).reshape(-1)
    return np.sqrt(v) if np.any(v != 0.0) else None


def measurement(x, nu_t, sv):
    """z = x + sqrt(v) o nu (numpy or torch); x itself without noise"""
    if sv is None:
        return x
    return x + (pgo.T(sv)[None] * nu_t if torch.is_tensor(x) else sv[None] * nu_t)


# ---- forward (numpy) --------------------------------------------------------------------------------------------------
def _rollout(pol, terms, x0, eps, nu, v, mult_mu, transition, angle_dims):
    """the step loop: u_t = pi(phi(z_t)), ``transition(x, [phi(x), u], eps_t)`` -> the next state"""
    P, H, E = eps.shape
    sv = _scale(v)
    x = np.asarray(x0, dtype=np.float64).copy()
    traj, act = [x], []
    for t in range(H):
        xf = pao.feature_map(x, angle_dims)
        zf = xf if sv is None else pao.feature_map(measurement(x, nu[:, t], sv), angle_dims)
        u = po.policy_action(pol, zf)
        x = transition(x, np.hstack([xf, u]), eps[:, t])
        traj.append(x); act.append(u)
    traj, act = np.stack(traj, 1), np.stack(act, 1) if H else np.zeros((P, 0, 0))
    rew, risk = pao.path_rewards(terms, traj, act, angle_dims)
    return traj, act, rew, risk, po.particle_return(terms, rew, risk, mult_mu)


def particle_rollout(dyn, pol, terms, x0, eps, nu, v, mult_mu=0.0, angle_dims=None):
    """pao.particle_rollout with the noisy measurement -> traj [P,H+1,E], act [P,H,U], step_reward, step_risk, ret"""
    def transition(x, xt, e):
        mu, var = po.gp_latent(dyn, xt)
        return x + mu + np.sqrt(np.maximum(var, 0.0)) * e
    return _rollout(pol, terms, x0, eps, nu, v, mult_mu, transition, angle_dims)


def consistent_rollout(dyn, pol, terms, x0, eps, nu, v, mult_mu=0.0, swap=False, angle_dims=None):
    """pao.consistent_rollout with the noisy measurement: the draw conditions on the particle's earlier [phi(x), u]"""
    fs = po.FunctionSample(dyn, eps.shape[0], swap)
    return _rollout(pol, terms, x0, eps, nu, v, mult_mu, lambda x, xt, e: x + fs.step(xt, e), angle_dims)


# ---- gradients (torch autograd) ---------------------------------------------------------------------------------------
def _pathwise(pol, terms, x0, eps, nu, v, mult_mu, transition, angle_dims):
    """pao._pathwise with the noisy measurement: mean particle return and its gradient w.r.t. the policy parameters"""
    P, H, E = eps.shape
    sv = _scale(v)
    prm, act = pgo.policy(pol)
    x, e = pgo.T(x0), pgo.T(eps)
    n = pgo.T(nu) if sv is not None else None
    rews, risks = [], []
    for s in range(H):
        xf = pao.feature_map_torch(x, angle_dims)
        zf = xf if sv is None else pao.feature_map_torch(measurement(x, n[:, s], sv), angle_dims)
        u = act(zf)
        r, k = po.step_values(terms, lambda term: pgo.point_value(term, xf if po.is_joint(term) else x, u),
                              torch.zeros(P, dtype=F64))
        rews.append(r); risks.append(k)
        mean, var = transition(torch.cat([xf, u], 1), e[:, s])
        x = x + mean + torch.sqrt(var) * e[:, s]
    stack = lambda w: torch.stack(w, 1) if H else torch.zeros((P, 0), dtype=F64)
    value = po.particle_return(terms, stack(rews), stack(risks), mult_mu).mean()
    return float(value.detach()), pgo._grads(value, prm)


def value_and_grad(dyn, pol, terms, x0, eps, nu, v, mult_mu=0.0, angle_dims=None):
    """pao.value_and_grad with the noisy measurement -> (value, {'W','b'} or {'X','Y','ell'}) in the policy's layout"""
    def transition(xt, e):
        mu, var = pgo.gp_latent(dyn, xt)
        return mu, torch.clamp(var, min=0.0)
    return _pathwise(pol, terms, x0, eps, nu, v, mult_mu, transition, angle_dims)


def consistent_value_and_grad(dyn, pol, terms, x0, eps, nu, v, mult_mu=0.0, swap=False, angle_dims=None):
    """pao.consistent_value_and_grad with the noisy measurement -> (value, grads, smallest kept pivot ratio)"""
    fs = pgo.TorchFunctionSample(dyn, swap)
    return _pathwise(pol, terms, x0, eps, nu, v, mult_mu, fs.step, angle_dims) + (fs.min_ratio,)


def score_grad(dyn, pol, terms, traj, eps, nu, v, mult_mu=0.0, baseline=True, direct=True, angle_dims=None):
    """pao.score_grad with the noisy measurement: the transitions' log-densities at [phi(x_t), pi(phi(z_t))] with x_t,
    x_{t+1} and nu held fixed, weighted by the return-to-go, plus the joint terms' direct dependence on the parameters
    through u_t -> {'W','b'} or {'X','Y','ell'}"""
    traj, eps = np.asarray(traj, dtype=np.float64), np.asarray(eps, dtype=np.float64)
    P, H, E = eps.shape
    sv = _scale(v)
    prm, act = pgo.policy(pol)
    if H == 0:
        return pgo._grads(torch.zeros(()), prm)
    xs = [pao.feature_map_torch(pgo.T(traj[:, s]), angle_dims) for s in range(H)]
    zs = xs if sv is None else [pao.feature_map_torch(pgo.T(measurement(traj[:, s], nu[:, s], sv)), angle_dims)
                                for s in range(H)]
    us = [act(z) for z in zs]
    rew, risk = pao.path_rewards(terms, traj, np.stack([u.detach().numpy() for u in us], 1), angle_dims)
    G = po.weights(terms, rew, risk, mult_mu, baseline)
    mult = any(po.is_mult(t) for t in terms)
    sur = torch.zeros((), dtype=F64)
    for s, (x, u) in enumerate(zip(xs, us)):
        if s < H - 1:
            mu, var = pgo.gp_latent(dyn, torch.cat([x, u], 1))
            v0, e = var.detach(), pgo.T(eps[:, s])
            pos = v0 > 0.0
            safe = torch.where(pos, v0, torch.ones_like(v0))
            a = torch.where(pos, e / torch.sqrt(safe), torch.zeros_like(v0))
            b = torch.where(pos, (e * e - 1.0) / (2.0 * safe), torch.zeros_like(v0))
            sur = sur + (pgo.T(G[:, s])[:, None] * (a * mu + b * var)).sum()
        if direct:
            wm = mult_mu * np.prod(np.delete(1.0 - risk, s, axis=1), axis=1) if mult else np.zeros(P)
            for term in terms:
                if po.is_joint(term):
                    w = float(term.get("coef", 1.0)) * (pgo.T(wm) if po.is_mult(term) else 1.0)
                    sur = sur + (w * pgo.point_value(term, x, u)).sum()
    return pgo._grads(sur / P, prm)
