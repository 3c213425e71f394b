"""Closed forms of the exploration objective's reward variance (pilco_rollout_explore_*, DESIGN.md section 21) for the
tests, in numpy: the variance of one reward term and its VJP -- the f-scaled exponential moment r_f (r_1 the mean, r_2
the second moment) with d r_f/dm = -f r_f w_f, d r_f/dS = (f/2) r_f (f w_f w_f' - W (I + f S W)^-1), and the linear
term's W' S W -- which the golden fixture of reward.m (tests/golden/reward_var.npz) checks.  The torch cascade with the
variance is tests/action_reward_oracle.py.  Test infrastructure only."""
import numpy as np


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
