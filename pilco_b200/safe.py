"""Safe-PILCO extension (drop-in for safe_pilco_extension/{rewards_safe,safe_pilco}.py).

The risk rewards are closed-form box probabilities evaluated on the device (``pilco_box_risk``; inside the
rollout as reward kind ``PILCO_REWARD_BOX``); ``SafePILCO`` adds the multiplicative accumulator of
``SafePILCO.predict`` (safe_pilco.py:29-50) as a second reward channel of the same device cascade, so the
policy gradient comes from the same hand-derived reverse sweep."""
import numpy as np

from . import engine, _lib
from .models.pilco import PILCO
from .params import Parameter, host

_INF = float("inf")


class _BoxRisk:
    """P(low_k < x[dim_k] < high_k for all k), x[dim] ~ Normal(loc=m[dim], scale=sfac*s[dim,dim]) independent."""

    def _box(self):
        """-> (dims, lows, highs, sfac, inside)"""
        raise NotImplementedError

    def prm(self):
        dims, lows, highs, sfac, inside = self._box()
        out = [float(len(dims)), 1.0 if inside else 0.0, float(sfac)]
        for d, lo, hi in zip(dims, lows, highs):
            out += [float(d), float(lo), float(hi)]
        return np.asarray(out)

    def compute_reward(self, m, s):
        m = np.asarray(m, dtype=np.float64).reshape(1, -1)
        k = m.shape[1]
        s = np.asarray(s, dtype=np.float64).reshape(1, k, k)
        risk = engine.box_risk(self.prm(), m, s)
        return host(risk)[0], 0.0001 * np.ones(1)          # rewards_safe.py:25,58

    def terms(self, coef=1.0, channel=_lib.CHANNEL_ADD):
        return [dict(kind=_lib.REWARD_BOX, coef=float(coef), channel=channel, W=self.prm(), t=None)]


class RiskOfCollision(_BoxRisk):
    """rewards_safe.py:13-25: state dims 0 and 2, scale = 2*diag(s)."""

    def __init__(self, state_dim, low, high):
        self.state_dim = state_dim
        self.low = np.asarray(low, dtype=np.float64).reshape(-1)
        self.high = np.asarray(high, dtype=np.float64).reshape(-1)

    def _box(self):
        return (0, 2), self.low[:2], self.high[:2], 2.0, True


class SingleConstraint(_BoxRisk):
    """rewards_safe.py:27-58: one dimension, optional bounds (a bound that is None -- or, as in the reference's
    truthiness tests at :47,:50, zero -- is absent), ``inside=False`` returns the complement."""

    def __init__(self, dim, high=None, low=None, inside=True):
        if high is None and low is None:
            raise Exception("At least one of bounds (high,low) has to be defined")
        self.high = False if high is None else high
        self.low = False if low is None else low
        self.dim = int(dim)
        self.inside = bool(inside)

    def _box(self):
        if not self.high:
            lo, hi = self.low, _INF
        elif not self.low:
            lo, hi = -_INF, self.high
        else:
            lo, hi = self.low, self.high
        return (self.dim,), (lo,), (hi,), 1.0, self.inside


class ObjectiveFunction:
    """reward - mu * risk (rewards_safe.py:60-73)."""

    def __init__(self, reward_f, risk_f, mu=1.0):
        self.reward_f = reward_f
        self.risk_f = risk_f
        self.mu = Parameter(mu, trainable=False)

    def compute_reward(self, m, s):
        reward, var = self.reward_f.compute_reward(m, s)
        risk, _ = self.risk_f.compute_reward(m, s)
        return reward - float(self.mu) * risk, var

    def terms(self, coef=1.0, channel=_lib.CHANNEL_ADD):
        return self.reward_f.terms(coef, channel) + self.risk_f.terms(-coef * float(self.mu), channel)


class SafePILCO(PILCO):
    """safe_pilco.py:17-50: total = sum_t reward_add(x_t) + mu * (1 - prod_t (1 - reward_mult(x_t)))."""

    def __init__(self, data, num_induced_points=None, horizon=30, controller=None,
                 reward_add=None, reward_mult=None, m_init=None, S_init=None, name=None, mu=5.0, *, exploration=0.0,
                 measurement_noise=None):
        """``exploration``: PILCO's (the additive reward's sigma_t enters; the risk terms do not).
        ``measurement_noise``: PILCO's (the risk terms, like the reward, see the true state)"""
        super(SafePILCO, self).__init__(data, num_induced_points=num_induced_points, horizon=horizon,
                                        controller=controller, reward=reward_add, m_init=m_init, S_init=S_init,
                                        exploration=exploration, measurement_noise=measurement_noise)
        if reward_mult is None:
            raise Exception("have to define multiplicative reward")
        self.mu = Parameter(mu, trainable=False)
        self.reward_mult = reward_mult

    def reward_spec(self):
        return self.reward.terms() + self.reward_mult.terms(1.0, _lib.CHANNEL_MULT), float(self.mu)
