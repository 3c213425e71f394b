"""Torch statement of the moment-matching rollout with measurement noise at the policy's input
(pilco_rollout_noisy_*, DESIGN.md section 22): propagate.m with its noise lines active.  Per step the policy is
moment-matched at phi's moments under N(m, S + diag(v)) (phi = identity without angles), the dynamics receive
[phi(x), u] with phi's moments under N(m, S) and cov(phi(x), u) = S^_x V_u (q = S(j,i) C: the true S, the noisy C), and
the glue uses cov(x, [phi, u]) = S C^_x [I, V_u].  Rewards and the exploration bonus are those of
tests/exploration_oracle.py.  With v = 0 every value is bitwise that oracle's.  Autograd through it is the gradient
oracle.  Test infrastructure only."""
import torch

import action_reward_oracle as aro
import angles_oracle as ao
import exploration_oracle as eo
import particle_oracle as po
from oracle import torch_port as tp

F64 = torch.float64
T = eo.T


def noisy_rollout(dyn_fn, action_fn, terms, m0, S0, H, b, v, mult_mu=0.0, angle_dims=None):
    """``eo.explore_rollout`` with the measurement noise variances v [Ds] at the policy's input"""
    v = v if torch.is_tensor(v) else T(v)
    m_x, s_x = m0.reshape(1, -1), S0
    tm, tS, rews, risks, vars_ = [m_x[0]], [s_x], [], [], []
    zero = torch.zeros((), dtype=F64)
    for _ in range(H):
        s_z = s_x + torch.diag(v)                     # the measurement z = x + nu
        if angle_dims:
            mh, Sh, Ch = ao.trig_moments(m_x[0], s_x, angle_dims)
            mh = mh[None]
            mz, Sz, _ = ao.trig_moments(m_x[0], s_z, angle_dims)
            mz = mz[None]
        else:
            mh, Sh = m_x, s_x
            mz, Sz = m_x, s_z
        m_u, s_u, c_xu = action_fn(mz, Sz)
        m = torch.cat([mh, m_u], dim=1)
        s = torch.cat([torch.cat([Sh, Sh @ c_xu], dim=1), torch.cat([(Sh @ c_xu).T, s_u], dim=1)], dim=0)
        at = lambda t: (m, s) if po.is_joint(t) else (m_x, s_x)
        rew, risk = po.step_values(terms, lambda t: aro.term_moment(t, *at(t)), zero)
        var = zero
        for term in [t for t in terms if not po.is_joint(t)] + [t for t in terms if po.is_joint(t)]:
            if not po.is_mult(term):
                var = var + float(term.get("coef", 1.0)) ** 2 * eo.term_var(term, *at(term))
        rews.append(rew); risks.append(risk); vars_.append(var)
        M_dx, S_dx, C_dx = dyn_fn(m, s)
        if angle_dims:
            Q = s_x @ Ch
            K = torch.cat([Q, Q @ c_xu], dim=1) @ C_dx
        else:
            K = torch.cat([s_x, s_x @ c_xu], dim=1) @ C_dx
        m_x, s_x = M_dx + m_x, S_dx + s_x + K + K.T
        tm.append(m_x[0]); tS.append(s_x)
    z = torch.zeros(0, dtype=F64)
    step_reward, step_risk, step_var = (torch.stack(x) if x else z for x in (rews, risks, vars_))
    bonus = step_reward + b * eo.sigma(step_var)
    return dict(traj_m=torch.stack(tm), traj_S=torch.stack(tS), step_reward=step_reward, step_risk=step_risk,
                step_var=step_var, reward=po.particle_return(terms, bonus[None], step_risk[None], mult_mu)[0])


def problem_rollout(kind, params, X, Y, ell, sf2, sn2, maxa, terms, m0, S0, H, b, v, mult_mu=0.0, angle_dims=None):
    """``noisy_rollout`` for an exact-GP dynamics model under a linear (params = W, b) or RBF (params = Xc, Yc, ell)
    policy, squashed unless maxa is None; params, m0 and S0 may be torch leaves that require grad"""
    iK, beta = tp.calculate_factorizations(T(X), T(Y), T(ell), T(sf2), T(sn2))
    dyn = lambda m, s: tp.predict_given_factorizations(T(X), T(ell), T(sf2), m, s, iK, beta)
    ma = None if maxa is None else T(maxa)[None]
    if kind == "linear":
        act = lambda m, s: tp.linear_action(params[0], params[1].reshape(1, -1), m, s, ma)
    else:
        act = lambda m, s: tp.rbf_action(params[0], params[1], params[2], m, s, ma)
    m0 = m0 if torch.is_tensor(m0) else T(m0)
    S0 = S0 if torch.is_tensor(S0) else T(S0)
    return noisy_rollout(dyn, act, terms, m0, S0, H, b, v, mult_mu, angle_dims)
