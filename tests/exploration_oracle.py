"""Oracle of the exploration objective (pilco_rollout_explore_*, DESIGN.md section 21), for the tests.

numpy: the variance of one reward term and its VJP in closed form -- the f-scaled exponential moment r_f (r_1 the mean,
r_2 the second moment) with d r_f/dm = -f r_f w_f, d r_f/dS = (f/2) r_f (f w_f w_f' - W (I + f S W)^-1), and the linear
term's W' S W -- which the golden fixture of reward.m (tests/golden/reward_var.npz) checks.

torch: the moment-matching cascade (oracle/torch_port.py's pieces, the angular feature map of tests/angles_oracle.py)
with each step's reward variance sigma_t^2 = sum_k c_k^2 Var[r_k] over the additive terms and the objective
sum_t (E[r_t] + b sigma_t) (+ the multiplicative channel's term); autograd through it is the gradient oracle.
Test infrastructure only."""
import numpy as np
import torch

from pilco_b200 import _lib
from oracle import torch_port as tp
import action_reward_oracle as aro
import angles_oracle as ao
import particle_oracle as po

F64 = torch.float64
VAR_FLOOR = 1e-12
T = lambda a: torch.tensor(np.asarray(a), dtype=F64)


# ---- numpy closed forms --------------------------------------------------------------------------------------------
def exp_moment_vjp(m, s, W, t, f):
    """r_f and its derivatives (d/dm [D], d/dS [D,D], the symmetric form) at x ~ N(m, s)"""
    D = len(m)
    A = np.eye(D) + f * s @ W
    B = W @ np.linalg.inv(A)
    v = m - t
    w = B @ v
    r = np.exp(-0.5 * f * v @ w) / np.sqrt(np.linalg.det(A))
    return r, -f * r * w, 0.5 * f * r * (f * np.outer(w, w) - 0.5 * (B + B.T))


def exp_var_vjp(m, s, W, t):
    """Var = r_2 - r_1^2 of an exponential term and its derivatives (d/dm, d/dS)"""
    r1, dm1, dS1 = exp_moment_vjp(m, s, W, t, 1.0)
    r2, dm2, dS2 = exp_moment_vjp(m, s, W, t, 2.0)
    return r2 - r1 * r1, dm2 - 2.0 * r1 * dm1, dS2 - 2.0 * r1 * dS1


def linear_var_vjp(m, s, W):
    """Var = W' S W of a linear term and its derivatives (d/dm = 0, d/dS = W W')"""
    return W @ s @ W, np.zeros_like(m), np.outer(W, W)


# ---- torch cascade -------------------------------------------------------------------------------------------------
def term_var(term, m, s):
    """Var of one additive term under N(m [1,d], s [d,d]) (torch scalar): r_2 - r_1^2 (r_2 is the mean of the term with
    2 W), or W' s W"""
    W = T(term["W"])
    if term["kind"] in (_lib.REWARD_EXP, _lib.REWARD_EXP_SA):
        t = T(term["t"]).reshape(1, -1)
        r1 = tp.exponential_reward(m, s, W, t)[0, 0]
        return tp.exponential_reward(m, s, 2.0 * W, t)[0, 0] - r1 * r1
    if term["kind"] in (_lib.REWARD_LINEAR, _lib.REWARD_LINEAR_SA):
        return W @ s @ W
    raise ValueError("no variance closed form for reward kind %d" % term["kind"])


def sigma(var):
    """sqrt(var) above the floor, else 0 with zero gradient"""
    big = var > VAR_FLOOR
    return torch.where(big, torch.sqrt(torch.where(big, var, torch.ones_like(var))), torch.zeros_like(var))


def explore_rollout(dyn_fn, action_fn, terms, m0, S0, H, b, mult_mu=0.0, angle_dims=None):
    """H steps of the cascade (with phi in front of the policy and the dynamics when ``angle_dims``): dyn_fn(m, s) ->
    (M, S, V) on the joint [phi(x), u], action_fn(m, s) -> (m_u, s_u, c) on phi(x).  State terms at the raw (m_t, S_t),
    joint terms at the joint Gaussian.  -> dict(traj_m, traj_S, step_reward, step_risk, step_var [H], reward)"""
    m_x, s_x = m0.reshape(1, -1), S0
    tm, tS, rews, risks, vars_ = [m_x[0]], [s_x], [], [], []
    zero = torch.zeros((), dtype=F64)
    for _ in range(H):
        if angle_dims:
            mh, Sh, Ch = ao.trig_moments(m_x[0], s_x, angle_dims)
            mh = mh[None]
        else:
            mh, Sh = m_x, s_x
        m_u, s_u, c_xu = action_fn(mh, Sh)
        m = torch.cat([mh, m_u], dim=1)
        s = torch.cat([torch.cat([Sh, Sh @ c_xu], dim=1), torch.cat([(Sh @ c_xu).T, s_u], dim=1)], dim=0)
        at = lambda t: (m, s) if po.is_joint(t) else (m_x, s_x)
        rew, risk = po.step_values(terms, lambda t: aro.term_moment(t, *at(t)), zero)
        var = zero
        for term in [t for t in terms if not po.is_joint(t)] + [t for t in terms if po.is_joint(t)]:
            if not po.is_mult(term):
                var = var + float(term.get("coef", 1.0)) ** 2 * term_var(term, *at(term))
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
    step_reward, step_risk, step_var = (torch.stack(v) if v else z for v in (rews, risks, vars_))
    bonus = step_reward + b * sigma(step_var)
    return dict(traj_m=torch.stack(tm), traj_S=torch.stack(tS), step_reward=step_reward, step_risk=step_risk,
                step_var=step_var, reward=po.particle_return(terms, bonus[None], step_risk[None], mult_mu)[0])


def problem_rollout(kind, params, X, Y, ell, sf2, sn2, maxa, terms, m0, S0, H, b, mult_mu=0.0, angle_dims=None):
    """``explore_rollout`` for an exact-GP dynamics model under a squashed linear (params = W, b) or RBF (params = Xc,
    Yc, ell) policy; params, m0 and S0 may be torch leaves that require grad"""
    iK, beta = tp.calculate_factorizations(T(X), T(Y), T(ell), T(sf2), T(sn2))
    dyn = lambda m, s: tp.predict_given_factorizations(T(X), T(ell), T(sf2), m, s, iK, beta)
    ma = T(maxa)[None]
    if kind == "linear":
        act = lambda m, s: tp.linear_action(params[0], params[1].reshape(1, -1), m, s, ma)
    else:
        act = lambda m, s: tp.rbf_action(params[0], params[1], params[2], m, s, ma)
    m0 = m0 if torch.is_tensor(m0) else T(m0)
    S0 = S0 if torch.is_tensor(S0) else T(S0)
    return explore_rollout(dyn, act, terms, m0, S0, H, b, mult_mu, angle_dims)
