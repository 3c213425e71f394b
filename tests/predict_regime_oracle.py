"""The predict family (pilco_gp_predict, its full covariance and its VJP, DESIGN.md sections 10 and 12) and one step of
the consistent sampler's conditioning (DESIGN.md section 14) in extended precision, each output with its condition
scale.

The statements of the process are the shared oracles' (tests/particle_oracle.py for the posterior and the sequential
semidefinite Cholesky, tests/particle_grad_oracle.py for the VJP), run here on ``np.longdouble`` arrays -- the x87
80-bit format where numpy provides it (eps 1.08e-19), as tests/mm_oracle.py.  The factors ``beta`` and ``iK`` are
INPUTS: any factors define the predictor exactly, so the kernels are tested apart from the factorisation.

A device result is judged by ``|error| / (eps64 * scale)``, the scale being the sum of the absolute values of the terms
the entry is summed from (for the conditioning, a first-order running bound of the same kind carried through the
substitution: ``Conditioning``).  The ratio is O(1) for a well-written fp64 kernel whatever the cancellation, and grows
when a kernel loses bits it did not have to lose.
"""
import numpy as np

import mm_oracle as mo
import particle_grad_oracle as pgo
import particle_oracle as po

LD, EPS64 = mo.LD, mo.EPS64
HAVE_EXTENDED, NEED_EXTENDED = mo.HAVE_EXTENDED, mo.NEED_EXTENDED
TINY = LD(1e-300)                       # keeps a zero scale from dividing


def ld_model(C, ell, sf2, beta, iK):
    """the oracles' dyn dict in longdouble (iK cut to n x n)"""
    n = np.shape(C)[0]
    return dict(C=mo._ld(C), ell=mo._ld(ell), sf2=mo._ld(sf2).reshape(-1), beta=mo._ld(beta),
                iK=mo._ld(np.asarray(iK)[:, :n, :n]))


def predict(dyn, Xs, e0=0, ne=None):
    """-> dict(mean, var [T,ne], cmean = sum |k beta|, cvar = sf2 + sum |k_i iK_ij k_j|), longdouble"""
    C, ell, sf2, iK, beta = (dyn[k] for k in ("C", "ell", "sf2", "iK", "beta"))
    Xs = mo._ld(Xs)
    ne = ell.shape[0] - e0 if ne is None else ne
    out = dict(mean=[], var=[], cmean=[], cvar=[])
    for e in range(e0, e0 + ne):
        K = po.se_k(Xs, C, ell[e], sf2[e])
        out["mean"].append(K @ beta[e])
        out["var"].append(sf2[e] - ((K @ iK[e]) * K).sum(1))
        out["cmean"].append(K @ np.abs(beta[e]))
        out["cvar"].append(sf2[e] + ((K @ np.abs(iK[e])) * K).sum(1))
    return {k: np.stack(v, 1) for k, v in out.items()}


def full_cov(dyn, Xs, e):
    """-> (cov [T,T], scale [T,T]) of output e: k(x, x') - k(x, C) iK k(C, x'), and k(x, x') + |k| |iK| |k|'"""
    C, ell, sf2, iK = (dyn[k] for k in ("C", "ell", "sf2", "iK"))
    Xs = mo._ld(Xs)
    K, Kss = po.se_k(Xs, C, ell[e], sf2[e]), po.se_k(Xs, Xs, ell[e], sf2[e])
    return Kss - K @ iK[e] @ K.T, Kss + K @ np.abs(iK[e]) @ K.T


def predict_vjp(dyn, Xs, gmean, gvar):
    """gx = sum_e ell_e^-2 sum_n c_en (c_n - x) and its scale: particle_grad_oracle.predict_vjp in longdouble"""
    return pgo.predict_vjp(dyn, mo._ld(Xs), mo._ld(gmean), mo._ld(gvar))


class Conditioning(po.FunctionSample):
    """particle_oracle.FunctionSample (the sequential semidefinite Cholesky with the tau rule) with, per step and
    output, the condition scales of what the step closes with and the margin of its tau decision.

    The scales are a first-order bound on the rounding of an fp64 evaluation in units of eps64, carried through the
    substitution: c_ts = k(x_t, x_s) - k_t iK k_s has scale k(x_t, x_s) + |k_t| |iK| k_s; l_ts = (c_ts - sum_r
    l_sr l_tr) / piv_s has (sc c_ts + sum_r (|l_sr| sc l_tr + sc l_sr |l_tr|) + |l_ts| sc piv_s) / piv_s; d2 = var -
    sum_s l_ts^2 has sf2 + |k_t| |iK| k_t + 2 sum_s |l_ts| sc l_ts; piv_t = sqrt(d2) has sc d2 / (2 piv_t).  Carried
    over many steps through small pivots this bound grows far beyond the rounding a device shows, so a tau decision's
    margin is taken against the step's own sums: |d2 - TAU sf2| / (eps64 (sf2 + |k_t| |iK| k_t + sum_s l_ts^2)).
    Below about 10 the decision is rounding noise, and a device may decide the other way.  ``step`` records, each
    [P,E]: ``mean``, ``var`` (d2), ``piv`` (the base class's lists), and ``sc_mean``, ``sc_var``, ``margin``."""

    def __init__(self, dyn, P):
        super().__init__(dyn, P)
        self.AK = []                     # |K*| |iK| rows [E,P,n] of every step
        self.sc_l = []                   # scales of the factor rows [P,E,s]
        self.sc_piv = []
        self.sc_mean, self.sc_var, self.margin = [], [], []

    def step(self, Xt, eps_t):
        f = super().step(mo._ld(Xt), mo._ld(eps_t))
        dyn, t, E = self.dyn, len(self.X) - 1, self.E
        ell, sf2, iK, beta = dyn["ell"], dyn["sf2"], dyn["iK"], dyn["beta"]
        K, l, d2, piv = self.K[t], self.L[t], self.var[t], self.piv[t]
        self.AK.append(np.stack([K[e] @ np.abs(iK[e]) for e in range(E)]))
        AK = self.AK[t]

        def kx(s):                       # k_e(x~_t, x~_s) [P,E]
            out = []
            for e in range(E):
                d = (self.X[t] - self.X[s]) / ell[e][None, :]
                out.append(sf2[e] * np.exp(-0.5 * (d * d).sum(-1)))
            return np.stack(out, 1)
        sc_l = np.zeros(l.shape, dtype=LD)
        for s in range(t):
            sc_c = kx(s) + np.stack([(AK[e] * self.K[s][e]).sum(1) for e in range(E)], 1)
            sub = ((np.abs(self.L[s]) * sc_l[:, :, :s] + self.sc_l[s] * np.abs(l[:, :, :s])).sum(-1)) if s else 0.0
            ps = self.piv[s]
            sc_l[:, :, s] = np.where(ps > 0, (sc_c + sub + np.abs(l[:, :, s]) * self.sc_piv[s])
                                     / np.where(ps > 0, ps, 1), 0)
        sc_d2 = (sf2[None, :] + np.stack([(AK[e] * K[e]).sum(1) for e in range(E)], 1)
                 + 2 * (np.abs(l) * sc_l).sum(-1))
        sc_mean = np.stack([K[e] @ np.abs(beta[e]) for e in range(E)], 1)
        if t:                            # + sum_s |eps_s| (sc l_ts + |l_ts|)
            sc_mean = sc_mean + (np.abs(np.stack(self.eps[:t], -1)) * (sc_l + np.abs(l))).sum(-1)
        self.sc_l.append(sc_l)
        self.sc_piv.append(np.where(piv > 0, sc_d2 / (2 * np.where(piv > 0, piv, 1)), 0))
        self.sc_mean.append(sc_mean)
        self.sc_var.append(sc_d2)
        own = sf2[None, :] + np.stack([(AK[e] * K[e]).sum(1) for e in range(E)], 1) + (l * l).sum(-1)
        self.margin.append(np.abs(d2 - po.TAU * sf2[None, :]) / (EPS64 * own))
        return f


def increment_scale(cond, t, eps_t):
    """the scale of f_t = mean' + sqrt(max(d2, 0)) eps_t: sc mean' + |eps_t| times the rounding scale of the square
    root (sc d2 / (2 sqrt d2), or sqrt(sc d2 / eps64) where d2 is within the rounding of zero)"""
    d2, sc = np.maximum(cond.var[t], 0), cond.sc_var[t]
    root = np.minimum(sc / (2 * np.sqrt(np.maximum(d2, TINY))), np.sqrt(sc / EPS64))
    return cond.sc_mean[t] + np.abs(mo._ld(eps_t)) * root


def teacher_forced(dyn, xt, eps):
    """one particle batch's conditioning at the given inputs xt [P,H,D] with the step normals eps [P,H,E] -> the
    Conditioning object after H steps (its per-step lists are [P,E] each)"""
    cond = Conditioning(dyn, xt.shape[0])
    for t in range(xt.shape[1]):
        cond.step(xt[:, t], eps[:, t])
    return cond


def increment_ratios(dyn, traj, act, eps, margin=10.0):
    """every step's increment x_{t+1} - x_t of a consistent rollout (traj [P,H+1,E], act [P,H,U], fp64) against
    mean' + sqrt(max(var', 0)) eps_t of the conditioning at its own inputs [x_t, u_t], one step at a time: no error is
    carried from step to step.  The scale adds |x_t| + |x_{t+1}| for the rounding of the state update.  A (particle,
    output) pair is left out from the first step whose tau decision has a margin below ``margin`` on.
    -> (worst ratio over the entries kept, share of entries left out, smallest margin)"""
    H = act.shape[1]
    cond = teacher_forced(dyn, np.concatenate([traj[:, :H], act], -1), eps)
    keep = np.ones((eps.shape[0], eps.shape[2]), dtype=bool)
    worst, left_out = 0.0, 0
    for t in range(H):
        keep &= cond.margin[t] >= margin
        want = cond.mean[t] + np.sqrt(np.maximum(cond.var[t], 0)) * mo._ld(eps[:, t])
        sc = increment_scale(cond, t, eps[:, t]) + np.abs(traj[:, t]) + np.abs(traj[:, t + 1])
        r = np.abs((traj[:, t + 1] - traj[:, t]).astype(LD) - want) / (EPS64 * sc)
        worst = max(worst, float(r[keep].max(initial=0.0)))
        left_out += int((~keep).sum())
    return worst, left_out / (H * keep.size) if H else 0.0, float(min(m.min() for m in cond.margin))
