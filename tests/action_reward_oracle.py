"""Moment-matching oracle for reward terms on the joint state-action Gaussian (PILCO_REWARD_EXP_SA /
PILCO_REWARD_LINEAR_SA, DESIGN.md section 18), for the tests: ``mm_rollout`` is the moment-matching cascade in torch
fp64 from oracle/torch_port.py's pieces, with every reward kind and both channels, joint terms evaluated at the joint
Gaussian handed to the dynamics model; autograd gives the gradient oracle of pilco_rollout_backward.  The particle
oracles with joint terms are tests/particle_oracle.py and particle_grad_oracle.py.  Test infrastructure only."""
import numpy as np
import torch

from pilco_b200 import _lib
from oracle import torch_port as tp, safe_port as sp
import particle_oracle as po
from particle_grad_oracle import F64, T


def term_moment(term, m, s):
    """expected value of one term under N(m [1,d], s [d,d]) (torch scalar); d = Ds, or D for a joint term"""
    W = T(term["W"])
    if term["kind"] in (_lib.REWARD_EXP, _lib.REWARD_EXP_SA):
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
        rew, risk = po.step_values(terms, lambda t: term_moment(t, m, s) if po.is_joint(t) else term_moment(t, m_x, s_x),
                                   torch.zeros((), dtype=F64))
        rews.append(rew); risks.append(risk)
        M_dx, S_dx, C_dx = dyn_fn(m, s)
        m_x, s_x = M_dx + m_x, S_dx + s_x + s1 @ C_dx + C_dx.T @ s1.T
        tm.append(m_x[0]); tS.append(s_x)
    z = torch.zeros(0, dtype=F64)
    step_reward, step_risk = (torch.stack(v) if v else z for v in (rews, risks))
    return dict(traj_m=torch.stack(tm), traj_S=torch.stack(tS), step_reward=step_reward, step_risk=step_risk,
                reward=po.particle_return(terms, step_reward[None], step_risk[None], mult_mu)[0])


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
