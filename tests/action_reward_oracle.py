"""Oracles for reward terms on the joint state-action Gaussian (PILCO_REWARD_EXP_SA / PILCO_REWARD_LINEAR_SA, DESIGN.md
section 18), for the tests:

  * ``mm_rollout``: the moment-matching cascade in torch fp64 from oracle/torch_port.py's pieces, with every reward
    kind and both channels, joint terms evaluated at the joint Gaussian handed to the dynamics model; autograd gives
    the gradient oracle of pilco_rollout_backward;
  * ``particle_rollout`` (numpy), ``value_and_grad`` (torch autograd, pathwise) and ``score_grad`` (torch autograd of
    the score surrogate plus the joint terms' direct dependence on the policy) on top of tests/particle_oracle.py,
    particle_grad_oracle.py and score_grad_oracle.py, with joint terms evaluated at the point [x_t, u_t].

Within a step the particle paths accumulate the state terms first, then the joint terms, each in term order.
Test infrastructure only."""
import numpy as np
import torch

from pilco_b200 import _lib
from oracle import torch_port as tp, safe_port as sp
import particle_oracle as po
from particle_grad_oracle import _se, rbf_beta

F64 = torch.float64
T = lambda a: torch.as_tensor(np.asarray(a, dtype=np.float64))
JOINT = (_lib.REWARD_EXP_SA, _lib.REWARD_LINEAR_SA)
_EXP = (_lib.REWARD_EXP, _lib.REWARD_EXP_SA)


def is_joint(term):
    return term["kind"] in JOINT


def _is_mult(term):
    return int(term.get("channel", _lib.CHANNEL_ADD)) == _lib.CHANNEL_MULT


def _ordered(terms):
    """the particle paths' accumulation order: state terms, then joint terms"""
    return [t for t in terms if not is_joint(t)] + [t for t in terms if is_joint(t)]


# ---- moment matching ------------------------------------------------------------------------------------------------
def term_moment(term, m, s):
    """expected value of one term under N(m [1,d], s [d,d]) (torch scalar); d = Ds, or D for a joint term"""
    W = T(term["W"])
    if term["kind"] in _EXP:
        return tp.exponential_reward(m, s, W, T(term["t"]).reshape(1, -1))[0, 0]
    if term["kind"] == _lib.REWARD_BOX:
        prm = np.asarray(term["W"], dtype=np.float64)
        nd = int(prm[0])
        return sp.box_risk_torch(m, s, [int(prm[3 + 3 * k]) for k in range(nd)], [prm[4 + 3 * k] for k in range(nd)],
                                 [prm[5 + 3 * k] for k in range(nd)], sfac=prm[2], inside=prm[1] != 0.0)
    return (m @ W.reshape(-1, 1))[0, 0]


def mm_rollout(dyn_fn, action_fn, terms, m0, S0, H, mult_mu=0.0):
    """H steps of pilco.py:118-153 with the reward terms: dyn_fn(m, s) -> (M, S, V), action_fn(m_x, s_x) -> (m_u, s_u,
    c_xu).  -> dict(traj_m [H+1,Ds], traj_S [H+1,Ds,Ds], step_reward [H], step_risk [H], reward) of torch values"""
    m_x, s_x = m0.reshape(1, -1), S0
    tm, tS, rews, risks = [m_x[0]], [s_x], [], []
    for _ in range(H):
        m_u, s_u, c_xu = action_fn(m_x, s_x)
        m = torch.cat([m_x, m_u], dim=1)
        s1 = torch.cat([s_x, s_x @ c_xu], dim=1)
        s = torch.cat([s1, torch.cat([(s_x @ c_xu).T, s_u], dim=1)], dim=0)
        rew, risk = torch.zeros((), dtype=F64), torch.zeros((), dtype=F64)
        for term in terms:
            v = float(term.get("coef", 1.0)) * (term_moment(term, m, s) if is_joint(term) else term_moment(term, m_x, s_x))
            if _is_mult(term):
                risk = risk + v
            else:
                rew = rew + v
        rews.append(rew); risks.append(risk)
        M_dx, S_dx, C_dx = dyn_fn(m, s)
        m_x, s_x = M_dx + m_x, S_dx + s_x + s1 @ C_dx + C_dx.T @ s1.T
        tm.append(m_x[0]); tS.append(s_x)
    total = sum(rews) if rews else torch.zeros((), dtype=F64)
    if H > 0 and any(_is_mult(t) for t in terms):
        total = total + mult_mu * (1.0 - torch.prod(1.0 - torch.stack(risks)))
    z = torch.zeros(0, dtype=F64)
    return dict(traj_m=torch.stack(tm), traj_S=torch.stack(tS), step_reward=torch.stack(rews) if rews else z,
                step_risk=torch.stack(risks) if risks else z, reward=total)


def mm_problem_rollout(kind, params, X, Y, ell, sf2, sn2, maxa, terms, m0, S0, H, mult_mu=0.0, squash=True,
                       dyn_fact=None, centres=None):
    """``mm_rollout`` for an exact-GP dynamics model (or the given factorisation over ``centres``: FITC) under a linear
    (params = W, b) or RBF (params = Xc, Yc, ell) policy; params may require grad"""
    iK, beta = dyn_fact if dyn_fact is not None else tp.calculate_factorizations(T(X), T(Y), T(ell), T(sf2), T(sn2))
    C = T(X) if centres is None else T(centres)
    dyn = lambda m, s: tp.predict_given_factorizations(C, T(ell), T(sf2), m, s, iK, beta)
    ma = T(maxa)[None] if squash else None
    if kind == "linear":
        act = lambda m, s: tp.linear_action(params[0], params[1][None], m, s, ma)
    else:
        act = lambda m, s: tp.rbf_action(params[0], params[1], params[2], m, s, ma)
    return mm_rollout(dyn, act, terms, m0 if torch.is_tensor(m0) else T(m0), S0 if torch.is_tensor(S0) else T(S0), H, mult_mu)


# ---- particles ------------------------------------------------------------------------------------------------------
def point_value(term, x, u):
    """one term at the points x [P,Ds], u [P,U] (numpy) -> [P]"""
    if not is_joint(term):
        return po.reward_value(term, x)
    z = np.hstack([x, u])
    W = np.asarray(term["W"], dtype=np.float64)
    if term["kind"] == _lib.REWARD_LINEAR_SA:
        return z @ W.reshape(-1)
    d = z - np.asarray(term["t"], dtype=np.float64).reshape(1, -1)
    return np.exp(-0.5 * np.einsum("pi,ij,pj->p", d, W, d))


def particle_rollout(dyn, pol, terms, x0, eps, mult_mu=0.0):
    """tests/particle_oracle.py's particle_rollout with joint terms -> traj, act, step_reward, step_risk, ret"""
    P, H, Ds = eps.shape
    x = np.asarray(x0, dtype=np.float64).copy()
    traj, act, rew, risk = [x], [], np.zeros((P, H)), np.zeros((P, H))
    for t in range(H):
        u = po.policy_action(pol, x)
        for term in _ordered(terms):
            v = float(term.get("coef", 1.0)) * point_value(term, x, u)
            (risk if _is_mult(term) else rew)[:, t] += v
        act.append(u)
        mu, var = po.gp_latent(dyn, np.hstack([x, u]))
        x = x + mu + np.sqrt(np.maximum(var, 0.0)) * eps[:, t]
        traj.append(x)
    ret = rew.sum(1)
    if any(_is_mult(t) for t in terms):
        ret = ret + mult_mu * (1.0 - np.prod(1.0 - risk, axis=1))
    U = act[0].shape[1] if act else 0
    return np.stack(traj, 1), np.stack(act, 1) if act else np.zeros((P, 0, U)), rew, risk, ret


def _point_value_t(term, x, u):
    """torch ``point_value`` (box terms: value only, flat almost everywhere)"""
    W = T(term["W"])
    if term["kind"] == _lib.REWARD_BOX:
        return T(po.box_point(W.numpy(), x.detach().numpy()))
    z = torch.cat([x, u], 1) if is_joint(term) else x
    if term["kind"] in (_lib.REWARD_LINEAR, _lib.REWARD_LINEAR_SA):
        return z @ W.reshape(-1)
    d = z - T(term["t"]).reshape(1, -1)
    return torch.exp(-0.5 * torch.einsum("pi,ij,pj->p", d, W.reshape(d.shape[1], d.shape[1]), d))


def _policy_t(pol):
    """(parameters with requires_grad, x -> squashed action) as particle_grad_oracle.value_and_grad builds them"""
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


def _gp_t(dyn, xt):
    C, ell, sf2, iK, bd = (T(dyn[k]) for k in ("C", "ell", "sf2", "iK", "beta"))
    n = C.shape[0]
    mu, var = [], []
    for k in range(ell.shape[0]):
        K = _se(xt, C, ell[k], sf2[k])
        mu.append(K @ bd[k])
        var.append(sf2[k] - ((K @ iK[k][:n, :n]) * K).sum(1))
    return torch.stack(mu, 1), torch.stack(var, 1)


def _grads(value, prm):
    keys = list(prm)
    if not value.requires_grad:
        return {k: np.zeros(prm[k].shape) for k in keys}
    g = torch.autograd.grad(value, [prm[k] for k in keys], allow_unused=True)
    return {k: (np.zeros(prm[k].shape) if gi is None else gi.numpy()) for k, gi in zip(keys, g)}


def value_and_grad(dyn, pol, terms, x0, eps, mult_mu=0.0):
    """mean particle return and its pathwise gradient w.r.t. the policy parameters at fixed x0, eps (pol as
    particle_grad_oracle.value_and_grad takes it) -> (value, {'W','b'} or {'X','Y','ell'})"""
    P, H, Ds = eps.shape
    prm, act = _policy_t(pol)
    x, e = T(x0), T(eps)
    rew, risks = torch.zeros(P, dtype=F64), []
    for s in range(H):
        u = act(x)
        risk = torch.zeros(P, dtype=F64)
        for term in _ordered(terms):
            v = float(term.get("coef", 1.0)) * _point_value_t(term, x, u)
            if _is_mult(term):
                risk = risk + v
            else:
                rew = rew + v
        risks.append(risk)
        mu, var = _gp_t(dyn, torch.cat([x, u], 1))
        x = x + mu + torch.sqrt(torch.clamp(var, min=0.0)) * e[:, s]
    ret = rew
    if H > 0 and any(_is_mult(t) for t in terms):
        ret = ret + mult_mu * (1.0 - torch.prod(1.0 - torch.stack(risks, 1), 1))
    value = ret.mean()
    return float(value.detach()), _grads(value, prm)


def score_grad(dyn, pol_np, pol, terms, traj, eps, mult_mu=0.0, direct=True, transitions=True):
    """The score-function gradient with joint terms over the rollout (traj [P,H+1,Ds], eps [P,H,Ds]): the transition
    part of tests/score_grad_oracle.py with return-to-go weights that contain the joint terms, plus (``direct``) the
    joint terms' own dependence on the parameters through u_t = pi(x_t) at fixed states,
    (1/P) sum_p sum_{t<H} a_kt v_k([x_pt, pi(x_pt)]).  ``pol_np``: the numpy oracle's policy dict (for the weights)."""
    traj, eps = np.asarray(traj, dtype=np.float64), np.asarray(eps, dtype=np.float64)
    P, H, Ds = eps.shape
    rew, risk = np.zeros((P, H)), np.zeros((P, H))
    for t in range(H):
        u = po.policy_action(pol_np, traj[:, t])
        for term in _ordered(terms):
            (risk if _is_mult(term) else rew)[:, t] += float(term.get("coef", 1.0)) * point_value(term, traj[:, t], u)
    mult = any(_is_mult(t) for t in terms)
    G = np.zeros((P, max(H - 1, 0)))
    for t in range(H - 1):
        G[:, t] = rew[:, t + 1:].sum(1)
        if mult:
            G[:, t] += mult_mu * np.prod(1.0 - risk[:, :t + 1], 1) * (1.0 - np.prod(1.0 - risk[:, t + 1:], 1))
    if P > 1:
        G = G - (G.sum(0, keepdims=True) - G) / (P - 1)
    prm, act = _policy_t(pol)
    sur = torch.zeros((), dtype=F64)
    for s in range(H):
        x = T(traj[:, s])
        u = act(x)
        if transitions and s < H - 1:
            mu, var = _gp_t(dyn, torch.cat([x, u], 1))
            v0, e = var.detach(), T(eps[:, s])
            pos = v0 > 0.0
            safe = torch.where(pos, v0, torch.ones_like(v0))
            a = torch.where(pos, e / torch.sqrt(safe), torch.zeros_like(v0))
            b = torch.where(pos, (e * e - 1.0) / (2.0 * safe), torch.zeros_like(v0))
            sur = sur + (T(G[:, s])[:, None] * (a * mu + b * var)).sum()
        if direct:
            wm = mult_mu * np.prod(np.delete(1.0 - risk, s, axis=1), axis=1) if mult else np.zeros(P)
            for term in terms:
                if is_joint(term):
                    w = float(term.get("coef", 1.0)) * (T(wm) if _is_mult(term) else 1.0)
                    sur = sur + (w * _point_value_t(term, x, u)).sum()
    return _grads(sur / P, prm)
