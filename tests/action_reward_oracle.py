"""Torch statement of the moment-matching rollout for the tests: ``mm_rollout`` is the cascade of propagate.m in fp64
from oracle/torch_port.py's pieces, with every reward kind and both channels, and the optional features of the device's
rollout:

  * joint terms (PILCO_REWARD_EXP_SA / LINEAR_SA, DESIGN.md section 18) at the joint Gaussian handed to the dynamics
    model, state terms at the state Gaussian N(m_t, S_t);
  * angular state dimensions ``angle_dims`` (section 20): phi's moments (tests/angles_oracle.py) in front of the policy
    and the dynamics;
  * measurement noise ``v`` at the policy's input (section 22): the policy is moment-matched at phi's moments under
    N(m, S + diag(v)), the dynamics receive [phi(x), u] with phi's moments under N(m, S) and cov(phi(x), u) = S^_x V_u
    (the true S, the noisy C);
  * the exploration objective ``b`` (section 21): each step's reward variance sigma_t^2 = sum_k c_k^2 Var[r_k] over the
    additive terms and the objective sum_t (E[r_t] + b sigma_t) (+ the multiplicative channel's term);
  * any policy as an ``action_fn``, the time-varying linear policy (section 27) among them (``step_action``).

Without them (angle_dims None, v None, b = 0) it is the plain cascade.  Autograd through it is the gradient oracle of
pilco_rollout_backward.  ``problem_rollout`` builds the cascade of an exact GP, FITC or a given factorisation under a
linear, RBF or scheduled linear policy.  The particle oracles are tests/particle_oracle.py and particle_grad_oracle.py.
Test infrastructure only."""
import numpy as np
import torch

from pilco_b200 import _lib
from oracle import torch_port as tp, safe_port as sp
import angles_oracle as ao
import particle_oracle as po
from particle_grad_oracle import F64, T

VAR_FLOOR = 1e-12


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


def _features(m_x, s_x, angle_dims):
    """phi's moments (m [1,Dh], S [Dh,Dh], inv(s) cov(x, phi) [Ds,Dh] or None for phi = identity)"""
    if not angle_dims:
        return m_x, s_x, None
    M, S, C = ao.trig_moments(m_x[0], s_x, angle_dims)
    return M[None], S, C


def mm_rollout(dyn_fn, action_fn, terms, m0, S0, H, mult_mu=0.0, angle_dims=None, v=None, b=0.0):
    """H steps of the cascade from N(m0, S0): dyn_fn(m, s) -> (M, S, V) on the joint [phi(x), u], action_fn(m, s) ->
    (m_u, s_u, c) on phi(z), called once per step in step order; v: measurement-noise variances [Ds] or None.
    -> dict(traj_m [H+1,Ds], traj_S [H+1,Ds,Ds], step_reward [H], step_risk [H], step_var [H], reward) (torch)"""
    m_x, s_x = (m0 if torch.is_tensor(m0) else T(m0)).reshape(1, -1), S0 if torch.is_tensor(S0) else T(S0)
    v = None if v is None else v if torch.is_tensor(v) else T(v)
    tm, tS, rews, risks, vars_ = [m_x[0]], [s_x], [], [], []
    zero = torch.zeros((), dtype=F64)
    for _ in range(H):
        s_z = s_x if v is None else s_x + torch.diag(v)     # the measurement z = x + nu
        mh, Sh, Ch = _features(m_x, s_x, angle_dims)
        mz, Sz = (mh, Sh) if v is None else _features(m_x, s_z, angle_dims)[:2]
        m_u, s_u, c_xu = action_fn(mz, Sz)
        m = torch.cat([mh, m_u], dim=1)
        s = torch.cat([torch.cat([Sh, Sh @ c_xu], dim=1), torch.cat([(Sh @ c_xu).T, s_u], dim=1)], dim=0)
        at = lambda t: (m, s) if po.is_joint(t) else (m_x, s_x)
        rew, risk = po.step_values(terms, lambda t: term_moment(t, *at(t)), zero)
        var = zero
        for term in po.in_step_order(po.additive(terms)):
            var = var + float(term.get("coef", 1.0)) ** 2 * term_var(term, *at(term))
        rews.append(rew); risks.append(risk); vars_.append(var)
        M_dx, S_dx, C_dx = dyn_fn(m, s)
        Q = s_x if Ch is None else s_x @ Ch                 # cov(x, phi) inv(S^)
        K = torch.cat([Q, Q @ c_xu], dim=1) @ C_dx          # cov(x, [phi, u]) C_dx
        m_x, s_x = M_dx + m_x, S_dx + s_x + K + K.T
        tm.append(m_x[0]); tS.append(s_x)
    z = torch.zeros(0, dtype=F64)
    step_reward, step_risk, step_var = (torch.stack(x) if x else z for x in (rews, risks, vars_))
    bonus = step_reward + b * sigma(step_var)
    return dict(traj_m=torch.stack(tm), traj_S=torch.stack(tS), step_reward=step_reward, step_risk=step_risk,
                step_var=step_var, reward=po.particle_return(terms, bonus[None], step_risk[None], mult_mu)[0])


def dynamics(X, Y, ell, sf2, sn2, Z=None, fact=None):
    """the dynamics moment match of an exact GP, of FITC over the inducing points Z, or of the given factorisation
    fact = (iK, beta) over the centres Z (X when Z is None)"""
    if fact is not None:
        iK, beta = fact
    elif Z is None:
        iK, beta = tp.calculate_factorizations(T(X), T(Y), T(ell), T(sf2), T(sn2))
    else:
        iK, beta = tp.fitc_factorizations(T(X), T(Z), T(Y), T(ell), T(sf2), T(sn2))
    C = T(X) if Z is None else T(Z)
    return lambda m, s: tp.predict_given_factorizations(C, T(ell), T(sf2), m, s, iK, beta)


def step_action(Ws, bs, maxa):
    """the time-varying linear policy as an action function: call k applies sq(Ws[k] x + bs[k]); Ws [>=H,U,Dh], bs
    [>=H,U] (tensors); maxa [U], or None for no squash"""
    ma = None if maxa is None else T(maxa)[None]
    step = [0]

    def act(m, s):
        t = step[0]
        step[0] += 1
        return tp.linear_action(Ws[t], bs[t].reshape(1, -1), m, s, ma)
    return act


def problem_rollout(kind, params, X, Y, ell, sf2, sn2, maxa, terms, m0, S0, H, mult_mu=0.0, angle_dims=None, v=None,
                    b=0.0, Z=None, fact=None):
    """``mm_rollout`` for the ``dynamics`` of (X, Y, ell, sf2, sn2, Z, fact) under a linear (kind "linear", params = W,
    b), RBF ("rbf", params = Xc, Yc, ell) or scheduled linear ("schedule", params = Ws, bs) policy, squashed unless maxa
    is None; params, m0 and S0 may be torch leaves that require grad"""
    if kind == "schedule":
        act = step_action(params[0], params[1], maxa)
    else:
        ma = None if maxa is None else T(maxa)[None]
        if kind == "linear":
            act = lambda m, s: tp.linear_action(params[0], params[1].reshape(1, -1), m, s, ma)
        else:
            act = lambda m, s: tp.rbf_action(params[0], params[1], params[2], m, s, ma)
    return mm_rollout(dynamics(X, Y, ell, sf2, sn2, Z, fact), act, terms, m0, S0, H, mult_mu, angle_dims, v, b)
