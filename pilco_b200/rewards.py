"""Rewards (drop-in for pilco/rewards.py).  ``ExponentialReward`` moments run on the device
(``pilco_exp_reward``); ``LinearReward``/``CombinedRewards`` are linear maps of the state moments.

Beyond the reference: ``ExponentialStateActionReward`` / ``LinearStateActionReward`` are functions of the joint
[x_t, u_t] of the state and the applied (squashed) action, evaluated inside the device rollout at the joint Gaussian
the dynamics model receives (reward kinds ``PILCO_REWARD_EXP_SA`` / ``PILCO_REWARD_LINEAR_SA``); ``action_cost`` builds
the usual saturating control-effort cost from them."""
import numpy as np

from . import engine, _lib
from .params import Parameter, host


class ExponentialReward:
    """exp(-(x-t)^T W (x-t)/2) under x~N(m,s) (rewards.py:7-51; reward.m)."""

    def __init__(self, state_dim, W=None, t=None):
        self.state_dim = state_dim
        self.W = Parameter(np.reshape(W, (state_dim, state_dim)) if W is not None else np.eye(state_dim), trainable=False)
        self.t = Parameter(np.reshape(t, (1, state_dim)) if t is not None else np.zeros((1, state_dim)), trainable=False)

    def compute_reward(self, m, s):
        k = self.state_dim
        m = np.asarray(m, dtype=np.float64).reshape(1, k)
        s = np.asarray(s, dtype=np.float64).reshape(1, k, k)
        mu, sR = engine.exp_reward(np.asarray(self.W), np.asarray(self.t).reshape(k), m, s, variance=True)
        return host(mu).reshape(1, 1), host(sR).reshape(1, 1)

    def terms(self, coef=1.0, channel=_lib.CHANNEL_ADD):
        return [dict(kind=_lib.REWARD_EXP, coef=float(coef), channel=channel, W=np.asarray(self.W),
                     t=np.asarray(self.t).reshape(self.state_dim))]


class LinearReward:
    """W^T x (rewards.py:53-61)."""

    def __init__(self, state_dim, W):
        self.state_dim = state_dim
        self.W = Parameter(np.reshape(W, (state_dim, 1)), trainable=False)

    def compute_reward(self, m, s):
        W = np.asarray(self.W)
        m = np.asarray(m, dtype=np.float64).reshape(1, self.state_dim)
        s = np.asarray(s, dtype=np.float64).reshape(self.state_dim, self.state_dim)
        return m @ W, W.T @ s @ W

    def terms(self, coef=1.0, channel=_lib.CHANNEL_ADD):
        return [dict(kind=_lib.REWARD_LINEAR, coef=float(coef), channel=channel,
                     W=np.asarray(self.W).reshape(self.state_dim), t=None)]


def _joint_moments(reward, m, s):
    """joint moments ([1,D], [D,D]) for a state-action reward's compute_reward; state moments alone are an error"""
    D = reward.state_dim + reward.control_dim
    m, s = np.asarray(m, dtype=np.float64), np.asarray(s, dtype=np.float64)
    if m.size != D or s.size != D * D:
        raise ValueError("%s.compute_reward needs the joint moments of state and action, m [1,%d] and s [%d,%d] "
                         "(state_dim=%d + control_dim=%d), got %s and %s: a reward on the action cannot be evaluated "
                         "on state moments alone; PILCO.predict evaluates it inside the rollout"
                         % (type(reward).__name__, D, D, D, reward.state_dim, reward.control_dim, m.shape, s.shape))
    return m.reshape(1, D), s.reshape(D, D)


class ExponentialStateActionReward:
    """exp(-(z-t)^T W (z-t)/2) under z = [x, u] ~ N(m, s), the joint of the state and the applied (squashed) action:
    W [D,D] (default I), t [1,D] (default 0), D = state_dim + control_dim.  In a rollout, step t's term is evaluated at
    the joint Gaussian handed to the dynamics model at step t; the final state has no action and no such term."""

    def __init__(self, state_dim, control_dim, W=None, t=None):
        self.state_dim, self.control_dim = int(state_dim), int(control_dim)
        D = self.state_dim + self.control_dim
        self.W = Parameter(np.reshape(W, (D, D)) if W is not None else np.eye(D), trainable=False)
        self.t = Parameter(np.reshape(t, (1, D)) if t is not None else np.zeros((1, D)), trainable=False)

    def compute_reward(self, m, s):
        """joint moments m [1,D], s [D,D] -> ([1,1], [1,1]) (pilco_exp_reward at dimension D)"""
        m, s = _joint_moments(self, m, s)
        D = m.shape[1]
        mu, sR = engine.exp_reward(np.asarray(self.W), np.asarray(self.t).reshape(D), m, s[None], variance=True)
        return host(mu).reshape(1, 1), host(sR).reshape(1, 1)

    def terms(self, coef=1.0, channel=_lib.CHANNEL_ADD):
        D = self.state_dim + self.control_dim
        return [dict(kind=_lib.REWARD_EXP_SA, coef=float(coef), channel=channel, W=np.asarray(self.W),
                     t=np.asarray(self.t).reshape(D), state_dim=self.state_dim, control_dim=self.control_dim)]


class LinearStateActionReward:
    """W^T [x, u]: W [D,1], D = state_dim + control_dim (see ``ExponentialStateActionReward`` for the semantics)."""

    def __init__(self, state_dim, control_dim, W):
        self.state_dim, self.control_dim = int(state_dim), int(control_dim)
        self.W = Parameter(np.reshape(W, (self.state_dim + self.control_dim, 1)), trainable=False)

    def compute_reward(self, m, s):
        m, s = _joint_moments(self, m, s)
        W = np.asarray(self.W)
        return m @ W, W.T @ s @ W

    def terms(self, coef=1.0, channel=_lib.CHANNEL_ADD):
        return [dict(kind=_lib.REWARD_LINEAR_SA, coef=float(coef), channel=channel,
                     W=np.asarray(self.W).reshape(self.state_dim + self.control_dim), t=None,
                     state_dim=self.state_dim, control_dim=self.control_dim)]


def action_cost(state_dim, control_dim, Q=None):
    """The saturating quadratic control-effort term exp(-u^T Q u / 2) (Q [U,U], default I) as an
    ``ExponentialStateActionReward`` with W = blockdiag(0, Q), t = 0.  With a positive coefficient c in
    ``CombinedRewards`` it is the cost -c (1 - exp(-u^T Q u / 2)) up to the constant c, which does not move the optimum:

        CombinedRewards(Ds, [ExponentialReward(Ds, t=target), action_cost(Ds, U, Q)], coefs=[1.0, 0.1])"""
    Ds, U = int(state_dim), int(control_dim)
    W = np.zeros((Ds + U, Ds + U))
    W[Ds:, Ds:] = np.eye(U) if Q is None else np.reshape(np.asarray(Q, dtype=np.float64), (U, U))
    return ExponentialStateActionReward(Ds, U, W=W)


class CombinedRewards:
    """Weighted sum of rewards (rewards.py:64-81)."""

    def __init__(self, state_dim, rewards=[], coefs=None):
        self.state_dim = state_dim
        self.base_rewards = rewards
        self.coefs = Parameter(coefs if coefs is not None else np.ones(len(rewards)), trainable=False)

    def compute_reward(self, m, s):
        total_mean, total_cov = 0, 0
        for reward, coef in zip(self.base_rewards, np.asarray(self.coefs)):
            mu, cov = reward.compute_reward(m, s)
            total_mean = total_mean + coef * np.asarray(mu)
            total_cov = total_cov + coef ** 2 * np.asarray(cov)
        return total_mean, total_cov

    def terms(self, coef=1.0, channel=_lib.CHANNEL_ADD):
        out = []
        for reward, c in zip(self.base_rewards, np.asarray(self.coefs)):
            out.extend(reward.terms(coef * float(c), channel))
        return out
