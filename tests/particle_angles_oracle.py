"""Numpy and torch statement of the particle rollouts with angular state dimensions (DESIGN.md section 20) for the tests:
tests/particle_oracle.py and tests/particle_grad_oracle.py with the feature map

    phi(x) = [x_j, j not an angle, increasing j] ++ [sin x_a, cos x_a for a in angle_dims order]

applied where the policy, the transition and the joint terms read the state; the state, the state terms and the GP's
outputs stay raw.  phi is written here (numpy and torch), independently of the engine's.  Every function is built from
the two oracles' own pieces (policy, GP posterior, function sample, reward values, return), so with ``angle_dims``
None or empty it computes what they compute.  Test infrastructure only."""
import numpy as np
import torch

import particle_grad_oracle as pgo
import particle_oracle as po

F64 = torch.float64


def feature_map(x, angle_dims=None):
    """phi(x) along the last axis (numpy).  None or empty: x itself (the same object)"""
    if not angle_dims:
        return x
    dims = [int(a) for a in angle_dims]
    keep = [j for j in range(x.shape[-1]) if j not in dims]
    parts = [x[..., keep]]
    for a in dims:
        parts += [np.sin(x[..., a:a + 1]), np.cos(x[..., a:a + 1])]
    return np.concatenate(parts, -1)


def feature_map_torch(x, angle_dims=None):
    """``feature_map`` in torch (x [P,Ds]).  None or empty: x itself"""
    if not angle_dims:
        return x
    dims = [int(a) for a in angle_dims]
    keep = [j for j in range(x.shape[1]) if j not in dims]
    parts = [x[:, keep]]
    for a in dims:
        parts += [torch.sin(x[:, a:a + 1]), torch.cos(x[:, a:a + 1])]
    return torch.cat(parts, 1)


# ---- forward (numpy) --------------------------------------------------------------------------------------------------
def path_rewards(terms, traj, act, angle_dims=None):
    """po.path_rewards with the joint terms at [phi(x_t), u_t] and the state terms at the raw x_t"""
    P, H = act.shape[:2]
    rew, risk = np.zeros((P, H)), np.zeros((P, H))
    for t in range(H):
        x, xf = traj[:, t], feature_map(traj[:, t], angle_dims)
        rew[:, t], risk[:, t] = po.step_values(
            terms, lambda term: po.point_value(term, xf if po.is_joint(term) else x, act[:, t]), np.zeros(P))
    return rew, risk


def _rollout(pol, terms, x0, eps, mult_mu, transition, angle_dims):
    """the step loop: u_t = pi(phi(x_t)), ``transition(x, [phi(x), u], eps_t)`` -> the next state"""
    P, H, Ds = eps.shape
    x = np.asarray(x0, dtype=np.float64).copy()
    traj, act = [x], []
    for t in range(H):
        xf = feature_map(x, angle_dims)
        u = po.policy_action(pol, xf)
        x = transition(x, np.hstack([xf, u]), eps[:, t])
        traj.append(x); act.append(u)
    traj, act = np.stack(traj, 1), np.stack(act, 1) if H else np.zeros((P, 0, 0))
    rew, risk = path_rewards(terms, traj, act, angle_dims)
    return traj, act, rew, risk, po.particle_return(terms, rew, risk, mult_mu)


def particle_rollout(dyn, pol, terms, x0, eps, mult_mu=0.0, angle_dims=None):
    """po.particle_rollout with angles -> traj [P,H+1,Ds], act [P,H,U], step_reward, step_risk [P,H], ret [P]"""
    def transition(x, xt, e):
        mu, var = po.gp_latent(dyn, xt)
        return x + mu + np.sqrt(np.maximum(var, 0.0)) * e
    return _rollout(pol, terms, x0, eps, mult_mu, transition, angle_dims)


def consistent_rollout(dyn, pol, terms, x0, eps, mult_mu=0.0, swap=False, angle_dims=None):
    """po.consistent_rollout with angles: the function draw conditions on the particle's earlier [phi(x), u]"""
    fs = po.FunctionSample(dyn, eps.shape[0], swap)
    return _rollout(pol, terms, x0, eps, mult_mu, lambda x, xt, e: x + fs.step(xt, e), angle_dims)


# ---- gradients (torch autograd) ---------------------------------------------------------------------------------------
def _pathwise(pol, terms, x0, eps, mult_mu, transition, angle_dims):
    """pgo._pathwise with angles: mean particle return and its gradient w.r.t. the policy parameters"""
    P, H, Ds = eps.shape
    prm, act = pgo.policy(pol)
    x, e = pgo.T(x0), pgo.T(eps)
    rews, risks = [], []
    for s in range(H):
        xf = feature_map_torch(x, angle_dims)
        u = act(xf)
        r, k = po.step_values(terms, lambda term: pgo.point_value(term, xf if po.is_joint(term) else x, u),
                              torch.zeros(P, dtype=F64))
        rews.append(r); risks.append(k)
        mean, var = transition(torch.cat([xf, u], 1), e[:, s])
        x = x + mean + torch.sqrt(var) * e[:, s]
    stack = lambda v: torch.stack(v, 1) if H else torch.zeros((P, 0), dtype=F64)
    value = po.particle_return(terms, stack(rews), stack(risks), mult_mu).mean()
    return float(value.detach()), pgo._grads(value, prm)


def value_and_grad(dyn, pol, terms, x0, eps, mult_mu=0.0, angle_dims=None):
    """pgo.value_and_grad with angles -> (value, {'W','b'} or {'X','Y','ell'}) in the policy's Dh layout"""
    def transition(xt, e):
        mu, var = pgo.gp_latent(dyn, xt)
        return mu, torch.clamp(var, min=0.0)
    return _pathwise(pol, terms, x0, eps, mult_mu, transition, angle_dims)


def consistent_value_and_grad(dyn, pol, terms, x0, eps, mult_mu=0.0, swap=False, angle_dims=None):
    """pgo.consistent_value_and_grad with angles -> (value, grads, smallest kept pivot d2 / (TAU sf2))"""
    fs = pgo.TorchFunctionSample(dyn, swap)
    return _pathwise(pol, terms, x0, eps, mult_mu, fs.step, angle_dims) + (fs.min_ratio,)


def score_grad(dyn, pol, terms, traj, eps, mult_mu=0.0, baseline=True, direct=True, angle_dims=None):
    """pgo.score_grad with angles: the transitions' log-densities at [phi(x_t), pi(phi(x_t))] with x_t, x_{t+1} held
    fixed, weighted by the return-to-go (po.weights of the rewards of ``path_rewards``), plus the joint terms' direct
    dependence on the parameters through u_t -> {'W','b'} or {'X','Y','ell'}"""
    traj, eps = np.asarray(traj, dtype=np.float64), np.asarray(eps, dtype=np.float64)
    P, H, Ds = eps.shape
    prm, act = pgo.policy(pol)
    if H == 0:
        return pgo._grads(torch.zeros(()), prm)
    xs = [feature_map_torch(pgo.T(traj[:, s]), angle_dims) for s in range(H)]
    us = [act(x) for x in xs]
    rew, risk = path_rewards(terms, traj, np.stack([u.detach().numpy() for u in us], 1), angle_dims)
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
