"""numpy oracle of the cross-entropy method's update (pilco_cem_update, pilco_cem_draw; DESIGN.md section 31), in the
device's order of operations: the rank order, the elites' mean and biased variance summed in rank order, the smoothed
sampling distribution, the best so far, the clipped draw and the trace row.  Every step is a product, a sum, a division
or a square root rounded once, so a faithful implementation matches it bit for bit."""
import numpy as np


def rank(value):
    """the rank order of value [K]: descending, NaN last, ties (and NaNs) to the lower index"""
    v = np.asarray(value, dtype=np.float64)
    key = lambda i: (bool(np.isnan(v[i])), 0.0 if np.isnan(v[i]) else -v[i], i)
    return np.array(sorted(range(v.shape[0]), key=key), dtype=np.int64)


def clip(x, lo, hi):
    """clip(x, lo, hi) with NaN kept"""
    x = np.asarray(x, dtype=np.float64)
    return np.where(x < lo, lo, np.where(x > hi, hi, x))


def draw(mean, std, xi, lo, hi):
    """candidates [K,H,U]: row 0 clip(mean), row k >= 1 clip(mean + std xi_k)"""
    out = clip(mean[None] + std[None] * xi, lo, hi)
    out[0] = clip(mean, lo, hi)
    return out


def update(cand, value, mean, std, ke, alpha, lo, hi, best_value, best, xi=None):
    """one iteration over cand [K,H,U] with value [K] -> dict(order, elites, mean, std, best_value, best, trace [2],
    cand: the next candidates (xi [K,H,U] given) or cand itself)"""
    cand, value = np.asarray(cand, dtype=np.float64), np.asarray(value, dtype=np.float64)
    order = rank(value)
    el = order[:ke]
    s = np.zeros_like(mean)
    for q in el:
        s = s + cand[q]
    m = s / ke
    s2 = np.zeros_like(mean)
    for q in el:
        d = cand[q] - m
        s2 = s2 + d * d
    v = s2 / ke
    beta = 1.0 - alpha
    new_mean = alpha * mean + beta * m
    new_std = np.sqrt(alpha * (std * std) + beta * v)
    top, tv = value[order[0]], 0.0
    for q in el:
        tv = tv + value[q]
    if top > best_value:
        best_value, best = top, cand[order[0]].copy()
    nxt = draw(new_mean, new_std, xi, lo, hi) if xi is not None else cand
    return dict(order=order, elites=el, mean=new_mean, std=new_std, best_value=best_value, best=best,
                trace=np.array([top, tv / ke]), cand=nxt)
