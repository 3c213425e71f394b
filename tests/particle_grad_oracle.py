"""Torch statement of the particle rollouts' policy gradients for the tests: tests/particle_oracle.py transcribed to
torch and differentiated w.r.t. the policy parameters at fixed x0 and eps, with the same optional features (angles
``angle_dims``, measurement noise ``nu``, ``v``) and, for the pathwise gradients, the exploration bonus ``b``.

  * ``value_and_grad``: the step-wise sampler's pathwise gradient (pilco_particles_rollout_grad, DESIGN.md section 12);
  * ``consistent_value_and_grad``: the consistent sampler's (pilco_particles_rollout_consistent_grad, section 15), with
    the same pivot mask and the tau rule in reverse (a degenerate step's own noise is held constant), and the explicit
    numpy statement of its reverse steps 1-6 at a fixed input sequence (``reverse_steps``);
  * ``resampled_rollout``: the Gaussian-resampled sampler (pilco_particles_resampled_*, section 26), the step-wise
    transition followed by the refit x_t = mu^_t + chol(S^_t) xi_{t-1} to the sample moments of the pre-fit particles;
  * ``score_grad``: the score-function gradient (pilco_particles_rollout_score_grad, section 16, and over consistent
    function samples with ``consistent``, section 25) plus the joint terms' direct dependence on the policy
    (section 18).

The three pathwise samplers share one step loop and differ only in their transition.  With ``b`` the value is
PILCO's exploration objective (section 24), mean_p ret_p + b sum_t sigma_t with sigma_t^2 = sum_k c_k^2 Var_p[r_kpt]
over the additive terms (unbiased variance), sigma_t = sqrt(sigma_t^2) if sigma_t^2 > 1e-12, else 0 (constant); at
b = 0 the bonus is not added, so the graph is that of the call without it.

The RBF policy's beta = (K + sn2 I)^-1 Yc goes through a Cholesky solve, so the gradient w.r.t. the centres, targets and
lengthscales includes the factorisation, as the device's does.  Also the closed form of the predict VJP
(pilco_gp_predict_vjp) in numpy.  Test infrastructure only."""
import numpy as np
import torch

from pilco_b200 import _lib
import particle_oracle as po

F64 = torch.float64
T = lambda a: torch.as_tensor(np.asarray(a, dtype=np.float64))
FLOOR = 1e-12           # the exploration bonus's floor on sigma_t^2
CHOL_TAU = 1e-12        # the refit's degenerate-column rule (resample_math.cuh)


def _se(Xs, C, ell, sf2):
    d = (Xs[:, None, :] - C[None, :, :]) / ell[None, None, :]
    return sf2 * torch.exp(-0.5 * (d * d).sum(-1))


def rbf_beta(Xc, Yc, ell, sf2, sn2):
    """beta [U,bf] = (K_j + sn2_j I)^-1 Yc[:, j] through a Cholesky solve (torch or numpy inputs, torch out)"""
    Xc, Yc, ell = (torch.as_tensor(a, dtype=F64) for a in (Xc, Yc, ell))
    bf = Xc.shape[0]
    out = []
    for j in range(Yc.shape[1]):
        K = _se(Xc, Xc, ell[j], float(sf2[j])) + float(sn2[j]) * torch.eye(bf, dtype=F64)
        out.append(torch.cholesky_solve(Yc[:, j:j + 1], torch.linalg.cholesky(K))[:, 0])
    return torch.stack(out, 0)


def rbf_pol_np(Xc, Yc, ell, maxa, sf2=None, sn2=None, squash=True):
    """the numpy oracle's RBF policy dict for the parameters (Xc [bf,Ds], Yc [bf,U], ell [U,Ds])"""
    U = Yc.shape[1]
    sf2 = np.ones(U) if sf2 is None else sf2
    sn2 = 1e-4 * np.ones(U) if sn2 is None else sn2
    return dict(kind=_lib.POLICY_RBF, squash=squash, maxa=maxa, C=Xc, ell=ell, sf2=sf2,
                beta=rbf_beta(Xc, Yc, ell, sf2, sn2).numpy())


def policy(pol):
    """(parameters with requires_grad, x -> squashed action) of pol = dict(kind, squash, maxa, W, b) or dict(kind,
    squash, maxa, Xc, Yc, ell, sf2, sn2); the parameters are {'W','b'} or {'X','Y','ell'}"""
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


def point_value(term, x, u):
    """particle_oracle.point_value in torch (box terms: value only, flat almost everywhere)"""
    W = T(term["W"])
    if term["kind"] == _lib.REWARD_BOX:
        return T(po.box_point(W.numpy(), x.detach().numpy()))
    z = torch.cat([x, u], 1) if po.is_joint(term) else x
    if term["kind"] in (_lib.REWARD_LINEAR, _lib.REWARD_LINEAR_SA):
        return z @ W.reshape(-1)
    d = z - T(term["t"]).reshape(1, -1)
    return torch.exp(-0.5 * torch.einsum("pi,ij,pj->p", d, W.reshape(d.shape[1], d.shape[1]), d))


def feature_map_torch(x, angle_dims=None):
    """particle_oracle.feature_map in torch (x [P,Ds]).  None or empty: x itself"""
    if not angle_dims:
        return x
    dims = [int(a) for a in angle_dims]
    keep = [j for j in range(x.shape[1]) if j not in dims]
    parts = [x[:, keep]]
    for a in dims:
        parts += [torch.sin(x[:, a:a + 1]), torch.cos(x[:, a:a + 1])]
    return torch.cat(parts, 1)


def gp_latent(dyn, xt):
    """particle_oracle.gp_latent in torch -> mean, latent variance [T,E]"""
    C, ell, sf2, iK, bd = (T(dyn[k]) for k in ("C", "ell", "sf2", "iK", "beta"))
    n = C.shape[0]
    mu, var = [], []
    for k in range(ell.shape[0]):
        K = _se(xt, C, ell[k], sf2[k])
        mu.append(K @ bd[k])
        var.append(sf2[k] - ((K @ iK[k][:n, :n]) * K).sum(1))
    return torch.stack(mu, 1), torch.stack(var, 1)


class TorchFunctionSample:
    """particle_oracle.FunctionSample in torch: step(Xt [P,D], eps_t [P,E]) -> (mean' [P,E], var' [P,E])"""

    def __init__(self, dyn, swap=False):
        self.dyn = dyn
        self.C, self.ell, self.sf2, self.iK = (T(dyn[k]) for k in ("C", "ell", "sf2", "iK"))
        self.n, self.E, self.swap = self.C.shape[0], self.ell.shape[0], swap
        self.X, self.L, self.piv, self.eps = [], [], [], []
        self.min_ratio = np.inf                 # the smallest pivot d2 / (TAU sf2) kept by the mask

    def _pairs(self, A, B):
        out = []
        for e in range(self.E):
            Ka, Kb = _se(A, self.C, self.ell[e], self.sf2[e]), _se(B, self.C, self.ell[e], self.sf2[e])
            iK = self.iK[e][:self.n, :self.n]
            q = (Ka * (Kb @ iK)).sum(1) if self.swap else ((Ka @ iK) * Kb).sum(1)
            d = (A - B) / self.ell[e][None, :]
            out.append(self.sf2[e] * torch.exp(-0.5 * (d * d).sum(-1)) - q)
        return torch.stack(out, 1)

    def step(self, Xt, eps_t):
        mu = gp_latent(self.dyn, Xt)[0]
        var = self._pairs(Xt, Xt)
        cols = []
        for s in range(len(self.X)):
            c = self._pairs(Xt, self.X[s])
            if s:
                c = c - (self.L[s] * torch.stack(cols, -1)).sum(-1)
            piv = self.piv[s]
            cols.append(torch.where(piv > 0.0, c / torch.where(piv > 0.0, piv, torch.ones_like(piv)), torch.zeros_like(c)))
        l = torch.stack(cols, -1) if cols else torch.zeros(Xt.shape[0], self.E, 0, dtype=F64)
        d2 = var - (l * l).sum(-1)
        mask = d2.detach() > po.TAU * self.sf2[None]
        if mask.any():
            self.min_ratio = min(self.min_ratio, float((d2.detach()[mask] / (po.TAU * self.sf2[None].expand_as(d2)[mask])).min()))
        vp = torch.clamp(d2, min=0.0)
        vp = torch.where(mask, vp, vp.detach())                 # the tau rule: a degenerate step's own noise is constant
        mean = mu + ((l * torch.stack(self.eps, -1)).sum(-1) if self.eps else 0.0)
        self.X.append(Xt); self.L.append(l); self.eps.append(eps_t)
        self.piv.append(torch.where(mask, torch.sqrt(torch.where(mask, d2, torch.ones_like(d2))), torch.zeros_like(d2)))
        return mean, vp


def _grads(value, prm):
    keys = list(prm)
    if not value.requires_grad:                 # e.g. H = 0: nothing depends on the policy
        return {k: np.zeros(prm[k].shape) for k in keys}
    g = torch.autograd.grad(value, [prm[k] for k in keys], allow_unused=True)
    return {k: (np.zeros(prm[k].shape) if gi is None else gi.numpy()) for k, gi in zip(keys, g)}


def chol(S):
    """the column-by-column factor of S's lower triangle (torch, differentiable); a column whose pivot d_j <=
    CHOL_TAU S_jj (or S_jj <= 0) is zero, as in resample_math.cuh, so autograd differentiates the factor as executed"""
    n = S.shape[0]
    zero = S.new_zeros(())
    L = [[zero] * n for _ in range(n)]
    for j in range(n):
        d = S[j, j]
        for k in range(j):
            d = d - L[j][k] * L[j][k]
        sjj, dv = float(S[j, j].detach()), float(d.detach())
        if not (sjj > 0.0 and dv > CHOL_TAU * sjj):
            continue
        piv = torch.sqrt(d)
        L[j][j] = piv
        for i in range(j + 1, n):
            s = S[i, j]
            for k in range(j):
                s = s - L[i][k] * L[j][k]
            L[i][j] = s / piv
    return torch.stack([torch.stack(row) for row in L])


def chol_np(S):
    return chol(T(S)).numpy()


def chol_bwd_np(S, Lb):
    """d <Lb, chol(S)> / d S on S's lower triangle (its upper triangle is 0), by autograd"""
    St = T(S).clone().requires_grad_()
    L = chol(St)
    if not L.requires_grad:
        return np.zeros(St.shape)
    g, = torch.autograd.grad((L * T(Lb)).sum(), St, allow_unused=True)
    return np.zeros(St.shape) if g is None else np.tril(g.numpy())


def _moments(x):
    """the sample mean and unbiased covariance of the particles x [P,Ds]"""
    m = x.mean(0)
    c = x - m[None]
    return m, c.T @ c / (x.shape[0] - 1)


def step_var(terms, value):
    """sigma_t^2 of one step: sum_k c_k^2 torch.var(r_k, unbiased=True) over the additive terms, in term order"""
    var = torch.zeros((), dtype=F64)
    for term in po.additive(terms):
        c = float(term.get("coef", 1.0))
        var = var + c * c * torch.var(value(term), unbiased=True)
    return var


def sigma(var):
    """section 21's floor: sqrt above 1e-12, else a constant 0"""
    return torch.sqrt(var) if float(var.detach()) > FLOOR else torch.zeros((), dtype=F64)


def _step(act, terms, x, nu_t, sv, angle_dims, with_var=False):
    """one step's work at the states x [P,Ds] (sv: the tensor sqrt(v), or None) -> (phi(x), u = pi(phi(z)), reward
    [P], risk [P], and sigma_t^2 when ``with_var``, else None)"""
    xf = feature_map_torch(x, angle_dims)
    zf = xf if sv is None else feature_map_torch(po.measurement(x, nu_t, sv), angle_dims)
    u = act(zf)
    value = po.step_point(x, xf, u, point_value)
    r, k = po.step_values(terms, value, torch.zeros(x.shape[0], dtype=F64))
    return xf, u, r, k, (step_var(terms, value) if with_var else None)


def _pathwise(pol, terms, x0, eps, mult_mu, transition, angle_dims=None, nu=None, v=None, b=None):
    """the step loop: the mean particle return (plus b sum_t sigma_t with ``b``) and its gradient w.r.t. the policy
    parameters; ``transition(x, [phi(x), u], eps_t)`` -> the next state.  -> (value, grads, dict(traj, act, rew, risk,
    ret), with ``b`` also step_var [H])"""
    P, H = eps.shape[:2]
    sv = po._scale(v)
    prm, act = policy(pol)
    x, e = T(x0), T(eps)
    n, svt = (None, None) if sv is None else (T(nu), T(sv))
    traj, acts, rews, risks, svar = [x], [], [], [], []
    for t in range(H):
        xf, u, r, k, var = _step(act, terms, x, None if n is None else n[:, t], svt, angle_dims, b is not None)
        acts.append(u); rews.append(r); risks.append(k); svar.append(var)
        x = transition(x, torch.cat([xf, u], 1), e[:, t])
        traj.append(x)
    stack = lambda w: torch.stack(w, 1) if H else torch.zeros((P, 0), dtype=F64)
    rew, risk = stack(rews), stack(risks)
    ret = po.particle_return(terms, rew, risk, mult_mu)
    value = ret.mean()
    if b and H:
        bonus = torch.zeros((), dtype=F64)
        for var in svar:
            bonus = bonus + sigma(var)
        value = value + b * bonus
    nd = lambda w: w.detach().numpy()
    hist = dict(traj=nd(torch.stack(traj, 1)), act=nd(torch.stack(acts, 1)) if H else np.zeros((P, 0, 0)),
                rew=nd(rew), risk=nd(risk), ret=nd(ret))
    if b is not None:
        hist["step_var"] = np.array([float(var.detach()) for var in svar])
    return float(value.detach()), _grads(value, prm), hist


def _stepwise(dyn):
    """the step-wise sampler's transition: x + mu + sqrt(max(var, 0)) eps_t"""
    def transition(x, xt, e):
        mu, var = gp_latent(dyn, xt)
        return x + mu + torch.sqrt(torch.clamp(var, min=0.0)) * e
    return transition


def value_and_grad(dyn, pol, terms, x0, eps, mult_mu=0.0, angle_dims=None, nu=None, v=None, b=None):
    """value = mean return of the step-wise sampler and its gradient w.r.t. the policy parameters at fixed x0, eps (and
    nu).  dyn = dict(C, ell, sf2, iK, beta) (numpy); pol as ``policy`` takes it.  -> (value, {'W','b'} or
    {'X','Y','ell'}), with ``b`` also step_var [H]"""
    value, grad, hist = _pathwise(pol, terms, x0, eps, mult_mu, _stepwise(dyn), angle_dims, nu, v, b)
    return (value, grad) if b is None else (value, grad, hist["step_var"])


def consistent_value_and_grad(dyn, pol, terms, x0, eps, mult_mu=0.0, swap=False, angle_dims=None, nu=None, v=None,
                              b=None):
    """``value_and_grad`` of the consistent sampler -> (value, grads, smallest kept pivot d2 / (TAU sf2)), with ``b``
    also step_var [H]"""
    fs = TorchFunctionSample(dyn, swap)

    def transition(x, xt, e):
        mean, var = fs.step(xt, e)
        return x + mean + torch.sqrt(var) * e
    value, grad, hist = _pathwise(pol, terms, x0, eps, mult_mu, transition, angle_dims, nu, v, b)
    return (value, grad, fs.min_ratio) + (() if b is None else (hist["step_var"],))


def resampled_rollout(dyn, pol, terms, x0, eps, xi, mult_mu=0.0):
    """the step-wise sampler with the refit at every step t >= 1: x'_t = the step-wise transition of x_{t-1},
    mu^_t, S^_t = the sample mean and unbiased covariance of x'_t, x_t = mu^_t + chol(S^_t) xi_{t-1}.  -> dict(traj
    [P,H+1,Ds], act, rew, risk, ret, step_mean [H+1,Ds], step_cov [H+1,Ds,Ds], xp [H,P,Ds], value, grad) of one restart;
    grad = d value / d the policy parameters, value = mean return, x0, eps and xi held fixed"""
    P, H, Ds = eps.shape
    step, z = _stepwise(dyn), T(xi)
    m, S = _moments(T(x0))
    means, covs, xps = [m], [S], []

    def transition(x, xt, e):
        xp = step(x, xt, e)
        m, S = _moments(xp)
        means.append(m); covs.append(S); xps.append(xp)
        return m[None] + z[:, len(xps) - 1] @ chol(S).T
    value, grad, out = _pathwise(pol, terms, x0, eps, mult_mu, transition)
    nd = lambda w: w.detach().numpy()
    out.update(step_mean=nd(torch.stack(means)), step_cov=nd(torch.stack(covs)),
               xp=nd(torch.stack(xps)) if H else np.zeros((0, P, Ds)), value=value, grad=grad)
    return out


def _log_density(dyn, xt, e):
    """the step-wise transition's score term at [phi(x_t), u_t]: a mu + b var, whose gradient at theta0 is that of
    log N(y; mu(theta), var(theta)) with y = mu(theta0) + s(theta0) eps held fixed (0 where var0 <= 0)"""
    mu, var = gp_latent(dyn, xt)
    v0 = var.detach()
    pos = v0 > 0.0
    safe = torch.where(pos, v0, torch.ones_like(v0))
    a = torch.where(pos, e / torch.sqrt(safe), torch.zeros_like(v0))
    b = torch.where(pos, (e * e - 1.0) / (2.0 * safe), torch.zeros_like(v0))
    return a * mu + b * var


def _whitened(fs, xt, e, f):
    """the consistent transition's score term: -eps_t(theta)^2 / 2 - log piv_t(theta) with eps_t(theta) = (f_t -
    mean'_t(theta)) / piv_t(theta), f_t = x_{t+1} - x_t held fixed; eps_t(theta) takes the caller's eps_t as its value
    and the residual's derivative, so the rounding of f_t does not enter.  A masked step drops its term and keeps the
    caller's eps_t, which is what the later steps' mean' reads"""
    mean, _ = fs.step(xt, e)
    piv = fs.piv[-1]
    on = piv > 0.0
    safe = torch.where(on, piv, torch.ones_like(piv))
    r = (f - mean) / safe
    et = torch.where(on, e + (r - r.detach()), e)
    fs.eps[-1] = et
    return torch.where(on, -0.5 * et * et - torch.log(safe), torch.zeros_like(et))


def score_grad(dyn, pol, terms, traj, eps, mult_mu=0.0, baseline=True, direct=True, transitions=True, angle_dims=None,
               nu=None, v=None, w=None, consistent=False, swap=False):
    """The score-function gradient of the mean return over the rollout (traj [P,H+1,Ds], eps [P,H,Ds], nu [P,H,Ds]; the
    device's, or particle_oracle's), pol as ``policy`` takes it, with x_t and nu held fixed and theta entering through
    u_t = pi(phi(z_t)) inside every x~_t = [phi(x_t), u_t].  With ``transitions`` the surrogate

        (1/P) sum_p sum_{t < H-1} w_pt s_pt(theta)

    is differentiated, s_pt the transition's log-density (step-wise sampler, ``_log_density``) or, with ``consistent``,
    the whitened log-density of the particle's function sample (``_whitened``, the factor rows and pivots of
    TorchFunctionSample with its tau mask).  w is ``weights`` (or the caller's ``w`` [P,H-1]).  With ``direct``, the
    joint terms' own dependence on the parameters through u_t at fixed states, (1/P) sum_p sum_{t<H} a_kt
    v_k([phi(x_pt), u_pt]), is added.  -> {'W','b'} or {'X','Y','ell'} numpy arrays; with ``consistent`` also the
    smallest kept pivot d2 / (TAU sf2) of the steps t < H-1"""
    traj, eps = np.asarray(traj, dtype=np.float64), np.asarray(eps, dtype=np.float64)
    P, H = eps.shape[:2]
    sv = po._scale(v)
    prm, act = policy(pol)
    if H == 0:
        g = _grads(torch.zeros(()), prm)
        return (g, np.inf) if consistent else g
    steps = [_step(act, terms, T(traj[:, s]), None if sv is None else T(nu[:, s]), None if sv is None else T(sv),
                   angle_dims) for s in range(H)]
    rew, risk = po.path_rewards(terms, traj, np.stack([st[1].detach().numpy() for st in steps], 1), angle_dims)
    G = po.weights(terms, rew, risk, mult_mu, baseline) if w is None else np.asarray(w, dtype=np.float64)
    mult = any(po.is_mult(t) for t in terms)
    fs = TorchFunctionSample(dyn, swap) if consistent else None
    sur = torch.zeros((), dtype=F64)
    for s, (x, u) in enumerate(st[:2] for st in steps):
        if transitions and s < H - 1:
            xt, e = torch.cat([x, u], 1), T(eps[:, s])
            term = _whitened(fs, xt, e, T(traj[:, s + 1] - traj[:, s])) if consistent else _log_density(dyn, xt, e)
            sur = sur + (T(G[:, s])[:, None] * term).sum()
        if direct:
            wm = mult_mu * np.prod(np.delete(1.0 - risk, s, axis=1), axis=1) if mult else np.zeros(P)
            for term in terms:
                if po.is_joint(term):
                    c = float(term.get("coef", 1.0)) * (T(wm) if po.is_mult(term) else 1.0)
                    sur = sur + (c * point_value(term, x, u)).sum()
    g = _grads(sur / P, prm)
    return (g, fs.min_ratio) if consistent else g


def fixed_inputs_objective(dyn, Xs, eps, mbar, vbar):
    """sum_t sum_e mbar_te mean'_te + vbar_te var'_te of ONE particle's draw at the fixed inputs Xs [T,D] (torch,
    differentiable in Xs), with the tau rule of consistent_value_and_grad"""
    fs = TorchFunctionSample(dyn)
    tot = 0.0
    for t in range(Xs.shape[0]):
        mean, vp = fs.step(Xs[t:t + 1], torch.as_tensor(eps[t:t + 1]))
        tot = tot + (torch.as_tensor(mbar[t]) * mean[0]).sum() + (torch.as_tensor(vbar[t]) * vp[0]).sum()
    return tot


def reverse_steps(dyn, Xs, eps, mbar, vbar):
    """d/dXs of fixed_inputs_objective by DESIGN.md section 15's steps 1-6, written out: Xs [T,D], eps, mbar, vbar [T,E]
    -> gX [T,D]"""
    C, ell, sf2, iK, beta = (dyn[k] for k in ("C", "ell", "sf2", "iK", "beta"))
    n, (T_, D), E = C.shape[0], Xs.shape, ell.shape[0]
    gX = np.zeros((T_, D))
    for e in range(E):
        K = po.se_k(Xs, C, ell[e], sf2[e])                         # K*_t rows [T,n]
        iKe = iK[e][:n, :n]
        kx = po.se_k(Xs, Xs, ell[e], sf2[e])                       # k_e(x~_t, x~_s)
        kp = kx - K @ iKe @ K.T                                    # the posterior covariance
        Lm, piv = np.zeros((T_, T_)), np.zeros(T_)
        for t in range(T_):                                        # the forward: rows l_t. and pivots
            for s in range(t):
                if piv[s] > 0.0:
                    Lm[t, s] = (kp[t, s] - Lm[s, :s] @ Lm[t, :s]) / piv[s]
            d2 = kp[t, t] - Lm[t, :t] @ Lm[t, :t]
            piv[t] = np.sqrt(d2) if d2 > po.TAU * sf2[e] else 0.0
        Lam, G = np.zeros((T_, T_)), np.zeros((T_, T_))
        for t in range(T_ - 1, -1, -1):
            db = vbar[t, e] + Lam[t, t] / (2.0 * piv[t]) if piv[t] > 0.0 else 0.0              # 1
            lb = Lam[t, :t] + mbar[t, e] * eps[:t, e] - 2.0 * db * Lm[t, :t]                   # 3
            for s in range(t - 1, -1, -1):                                                      # 4
                c = lb[s] / piv[s] if piv[s] > 0.0 else 0.0
                Lam[s, s] -= c * Lm[t, s]
                lb[:s] -= c * Lm[s, :s]
                Lam[s, :s] -= c * Lm[t, :s]
                G[t, s] = G[s, t] = c                                                           # 5
            others = np.arange(T_) != t                                                         # 6
            a = -2.0 * db * K[t] - G[t, others] @ K[others]
            cn = K[t] * (mbar[t, e] * beta[e] + a @ iKe)
            direct = ((G[t, others] * kx[t, others])[:, None] * (Xs[others] - Xs[t])).sum(0)
            gX[t] += ((cn[:, None] * (C - Xs[t])).sum(0) + direct) / ell[e] ** 2
    return gX


def predict_vjp(dyn, Xs, gmean, gvar):
    """closed form of pilco_gp_predict_vjp in numpy -> (gXs [T,D], scale [T,D]: the sum of |terms|, with |iK| k for w)"""
    C, ell, sf2, iK, beta = (dyn[k] for k in ("C", "ell", "sf2", "iK", "beta"))
    n = C.shape[0]
    g, scale = np.zeros(Xs.shape), np.zeros(Xs.shape)
    diff = C[None, :, :] - Xs[:, None, :]                         # [T,n,D]
    for e in range(ell.shape[0]):
        K = po.se_k(Xs, C, ell[e], sf2[e])
        w = K @ iK[e][:n, :n]
        c = K * (gmean[:, e:e + 1] * beta[e][None] - 2.0 * gvar[:, e:e + 1] * w)
        g += (c[:, :, None] * diff).sum(1) / ell[e] ** 2
        # the rounding of w = iK k is bounded by sum |iK| k, not by |w|: that enters the scale
        ca = K * (np.abs(gmean[:, e:e + 1] * beta[e][None]) + 2.0 * np.abs(gvar[:, e:e + 1]) * (K @ np.abs(iK[e][:n, :n])))
        scale += (ca[:, :, None] * np.abs(diff)).sum(1) / ell[e] ** 2
    return g, scale
