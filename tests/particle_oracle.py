"""Numpy statement of the particle rollouts for the tests: P particles from the caller's x0 [P,Ds], driven by the
caller's standard normals eps [P,H,Ds], through a factorised dynamics GP (centres C, ell, sf2, iK, beta) under a linear
or RBF policy, with the reward terms evaluated at each particle's pre-step state and action.

  * ``particle_rollout``: the step-wise sampler (pilco_particles_rollout, DESIGN.md section 11), a fresh draw from the
    latent marginal at every step;
  * ``consistent_rollout``: the consistent sampler (pilco_particles_rollout_consistent, DESIGN.md section 14), each
    particle following ONE function per dynamics output drawn from the latent posterior
    k_post(a, b) = k_e(a, b) - k(a, C) iK_e k(C, b), sampled sequentially along the particle's own inputs with the
    semidefinite Cholesky rule (a pivot d2 <= TAU sf2_e leaves its column out of later substitutions).

Both take the optional features of the device's particle paths:

  * ``angle_dims`` (DESIGN.md section 20): the feature map
        phi(x) = [x_j, j not an angle, increasing j] ++ [sin x_a, cos x_a for a in angle_dims order]
    where the policy, the transition and the joint terms read the state; the state, the state terms and the GP's
    outputs stay raw.  phi is written here, independently of the engine's;
  * ``nu``, ``v`` (DESIGN.md section 23): the policy reads the measurement z_t = x_t + sqrt(v) o nu_t (nu [P,H,Ds]
    standard normals, v [Ds] variances), u_t = pi(phi(z_t)), while the transition reads [phi(x_t), u_t].

Without them (None, empty, or v all zero) the policy reads x_t itself and every output is that of the plain rollout.
State terms (REWARD_EXP / LINEAR / BOX) see x_t, joint terms (REWARD_EXP_SA / LINEAR_SA, DESIGN.md section 18) see
[phi(x_t), u_t]; within a step the state terms are added first, then the joint terms, each in term order, as on the
device.  Also the sample moments of the step rewards (the exploration objective, DESIGN.md section 24) and the score
estimator's return-to-go weights (DESIGN.md section 16).  Test infrastructure only; vectorised over particles and
outputs."""
import numpy as np

from pilco_b200 import _lib

RBF_VAR = 1e-6          # output variance of the deterministic-GP (RBF) policy at a point, as compute_action sees it
TAU = 1e-10
JOINT = (_lib.REWARD_EXP_SA, _lib.REWARD_LINEAR_SA)


def is_joint(term):
    return term["kind"] in JOINT


def is_mult(term):
    return int(term.get("channel", _lib.CHANNEL_ADD)) == _lib.CHANNEL_MULT


def se_k(Xs, C, ell, sf2):
    """sf2 exp(-0.5 |(x - c)/ell|^2) in the direct difference form -> [T, n]"""
    d = (Xs[:, None, :] - C[None, :, :]) / ell[None, None, :]
    return sf2 * np.exp(-0.5 * (d * d).sum(-1))


def gp_latent(dyn, Xs):
    """posterior mean and latent variance [T,E] of the factorised model dyn = dict(C, ell, sf2, iK, beta)"""
    C, ell, sf2, iK, beta = (dyn[k] for k in ("C", "ell", "sf2", "iK", "beta"))
    n = C.shape[0]
    M, V = [], []
    for e in range(ell.shape[0]):
        K = se_k(Xs, C, ell[e], sf2[e])
        M.append(K @ beta[e])
        V.append(sf2[e] - ((K @ iK[e][:n, :n]) * K).sum(1))
    return np.stack(M, 1), np.stack(V, 1)


def policy_action(pol, x):
    """squashed action [P,U]; pol = dict(kind, squash, maxa, W, b) (linear) or dict(kind, squash, maxa, C, ell, sf2,
    beta) (RBF: the deterministic GP's mean, its output variance RBF_VAR enters the squash as in compute_action)"""
    if pol["kind"] == _lib.POLICY_LINEAR:
        u, var = x @ np.asarray(pol["W"]).T + np.asarray(pol["b"]).reshape(1, -1), 0.0
    else:
        u = np.stack([se_k(x, pol["C"], pol["ell"][j], pol["sf2"][j]) @ pol["beta"][j]
                      for j in range(pol["ell"].shape[0])], 1)
        var = RBF_VAR
    if pol.get("squash", True):
        u = np.asarray(pol["maxa"]).reshape(1, -1) * np.exp(-0.5 * var) * np.sin(u)
    return u


def feature_map(x, angle_dims=None):
    """phi(x) along the last axis.  None or empty: x itself (the same object)"""
    if not angle_dims:
        return x
    dims = [int(a) for a in angle_dims]
    keep = [j for j in range(x.shape[-1]) if j not in dims]
    parts = [x[..., keep]]
    for a in dims:
        parts += [np.sin(x[..., a:a + 1]), np.cos(x[..., a:a + 1])]
    return np.concatenate(parts, -1)


def _scale(v):
    """sqrt(v) [Ds], or None for no measurement noise (v None or all zero)"""
    if v is None:
        return None
    v = np.asarray(v, dtype=np.float64).reshape(-1)
    return np.sqrt(v) if np.any(v != 0.0) else None


def measurement(x, nu_t, sv):
    """z = x + sqrt(v) o nu (numpy, or torch with sv a tensor); x itself (the same object) when sv is None"""
    return x if sv is None else x + sv[None] * nu_t


def box_point(prm, x):
    nd, inside = int(prm[0]), prm[1] != 0.0
    ok = np.ones(x.shape[0], dtype=bool)
    for k in range(nd):
        v = x[:, int(prm[3 + 3 * k])]
        ok &= (prm[4 + 3 * k] < v) & (v < prm[5 + 3 * k])
    return (ok == inside).astype(np.float64)


def point_value(term, x, u=None):
    """one reward term (engine dict: kind, W, t) at the states x [P,Ds] and, for a joint term, actions u [P,U] -> [P]"""
    W = np.asarray(term["W"], dtype=np.float64)
    if term["kind"] == _lib.REWARD_BOX:
        return box_point(W, x)
    z = np.hstack([x, u]) if is_joint(term) else x
    if term["kind"] in (_lib.REWARD_LINEAR, _lib.REWARD_LINEAR_SA):
        return z @ W.reshape(-1)
    d = z - np.asarray(term["t"], dtype=np.float64).reshape(1, -1)
    return np.exp(-0.5 * np.einsum("pi,ij,pj->p", d, W.reshape(d.shape[1], d.shape[1]), d))


def in_step_order(terms):
    """the terms in the device's order within a step: state terms first, then joint terms, each in term order"""
    return [t for t in terms if not is_joint(t)] + [t for t in terms if is_joint(t)]


def additive(terms):
    """the ADD-channel terms that have a variance (not box), in term order"""
    return [t for t in terms if not is_mult(t) and t["kind"] != _lib.REWARD_BOX]


def step_values(terms, value, zero):
    """(reward, risk) of one step: the sum of coef * value(term) over each channel's terms from ``zero``, in
    ``in_step_order``.  Numpy or torch: ``value`` and ``zero`` decide."""
    rew = risk = zero
    for term in in_step_order(terms):
        v = float(term.get("coef", 1.0)) * value(term)
        if is_mult(term):
            risk = risk + v
        else:
            rew = rew + v
    return rew, risk


def step_point(x, xf, u, point_value=point_value):
    """term -> its value at one step: a state term at the raw x, a joint term at [xf, u] (xf = phi(x))"""
    return lambda term: point_value(term, xf if is_joint(term) else x, u)


def path_rewards(terms, traj, act, angle_dims=None):
    """step_reward, step_risk [P,H] of the terms at the states traj[:, t] and actions act[:, t] of every step t < H"""
    P, H = act.shape[:2]
    rew, risk = np.zeros((P, H)), np.zeros((P, H))
    for t in range(H):
        x = traj[:, t]
        rew[:, t], risk[:, t] = step_values(terms, step_point(x, feature_map(x, angle_dims), act[:, t]), np.zeros(P))
    return rew, risk


def sample_moments(terms, traj, act, angle_dims=None):
    """(mean [H], var [H]) of the step rewards over the particles of traj [P,H+1,Ds], act [P,H,U]: mean_t =
    sum_k c_k mean_p r_kpt and var_t = sum_k c_k^2 Var_p[r_kpt] (ddof 1) over the ``additive`` terms"""
    H = act.shape[1]
    mean, var = np.zeros(H), np.zeros(H)
    for t in range(H):
        x = traj[:, t]
        value = step_point(x, feature_map(x, angle_dims), act[:, t])
        for term in additive(terms):
            c = float(term.get("coef", 1.0))
            r = value(term)
            mean[t] += c * r.mean()
            var[t] += c * c * r.var(ddof=1)
    return mean, var


def particle_return(terms, rew, risk, mult_mu):
    """the return [P] of step rewards and risks [P,H] (numpy or torch): sum_t r_t, plus mult_mu (1 - prod_t (1 - k_t))
    when a term is on the MULT channel"""
    ret = rew.sum(1)
    if any(is_mult(t) for t in terms):
        ret = ret + mult_mu * (1.0 - (1.0 - risk).prod(1))
    return ret


def _rollout(pol, terms, x0, eps, mult_mu, transition, angle_dims=None, nu=None, v=None):
    """the step loop: u_t = pi(phi(z_t)), ``transition(x, [phi(x), u], eps_t)`` -> the next state"""
    P, H = eps.shape[:2]
    sv = _scale(v)
    x = np.asarray(x0, dtype=np.float64).copy()
    traj, act = [x], []
    for t in range(H):
        xf = feature_map(x, angle_dims)
        zf = xf if sv is None else feature_map(measurement(x, nu[:, t], sv), angle_dims)
        u = policy_action(pol, zf)
        x = transition(x, np.hstack([xf, u]), eps[:, t])
        traj.append(x); act.append(u)
    traj, act = np.stack(traj, 1), np.stack(act, 1) if H else np.zeros((P, 0, 0))
    rew, risk = path_rewards(terms, traj, act, angle_dims)
    return traj, act, rew, risk, particle_return(terms, rew, risk, mult_mu)


def particle_rollout(dyn, pol, terms, x0, eps, mult_mu=0.0, angle_dims=None, nu=None, v=None):
    """-> traj [P,H+1,Ds], act [P,H,U], step_reward [P,H], step_risk [P,H], ret [P] of the step-wise sampler"""
    def transition(x, xt, e):
        mu, var = gp_latent(dyn, xt)
        return x + mu + np.sqrt(np.maximum(var, 0.0)) * e
    return _rollout(pol, terms, x0, eps, mult_mu, transition, angle_dims, nu, v)


def consistent_rollout(dyn, pol, terms, x0, eps, mult_mu=0.0, swap=False, angle_dims=None, nu=None, v=None):
    """-> traj, act, step_reward, step_risk, ret of the consistent sampler (eps[:, t] is the step-t normal of every
    output; the draw conditions on the particle's earlier [phi(x), u]).  ``swap`` reorders the posterior's sums: the
    difference of the two is the sampler's own sensitivity to rounding"""
    fs = FunctionSample(dyn, eps.shape[0], swap)
    return _rollout(pol, terms, x0, eps, mult_mu, lambda x, xt, e: x + fs.step(xt, e), angle_dims, nu, v)


def _posterior(dyn, A, B):
    """latent posterior covariance k_post(A, B) per output -> [E, |A|, |B|]"""
    C, ell, sf2, iK = (dyn[k] for k in ("C", "ell", "sf2", "iK"))
    n = C.shape[0]
    out = []
    for e in range(ell.shape[0]):
        Ka, Kb = se_k(A, C, ell[e], sf2[e]), se_k(B, C, ell[e], sf2[e])
        out.append(se_k(A, B, ell[e], sf2[e]) - Ka @ iK[e][:n, :n] @ Kb.T)
    return np.stack(out)


class FunctionSample:
    """The running state of one draw per (particle, output): the visited inputs, their K* rows and the packed factor
    rows.  ``step(Xt, eps_t)`` -> f(Xt) [P,E] given the draws at the earlier inputs.  Written over numpy's generic
    arithmetic: with ``np.longdouble`` factors, inputs and normals it runs in extended precision."""

    def __init__(self, dyn, P, swap=False):
        self.dyn, self.P, self.swap = dyn, P, swap
        self.E = dyn["ell"].shape[0]
        self.X = []              # visited inputs, each [P,D]
        self.K, self.KiK = [], []    # their K* [E,P,n] and K* iK [E,P,n]
        self.L = []              # rows l [P,E,s] of the factor, below the diagonal
        self.piv = []            # pivots [P,E] (0: degenerate column)
        self.eps = []            # the normals [P,E] of the earlier steps
        self.mean, self.var = [], []     # each step's mean' = mu + sum_s l_s eps_s and d2 = var - sum_s l_s^2, [P,E]

    def _pairs(self, Xt, K, KiK, s):
        """k_post(Xt_p, X_s,p) [P,E] (s None: Xt itself).  ``swap``: the quadratic form as k_t (iK k_s) instead of
        (k_t iK) k_s, the same value with other roundings"""
        ell, sf2 = self.dyn["ell"], self.dyn["sf2"]
        Xs, Ks, KiKs = (Xt, K, KiK) if s is None else (self.X[s], self.K[s], self.KiK[s])
        out = []
        for e in range(self.E):
            d = (Xt - Xs) / ell[e][None, :]
            q = (K[e] * KiKs[e]).sum(1) if self.swap else (KiK[e] * Ks[e]).sum(1)
            out.append(sf2[e] * np.exp(-0.5 * (d * d).sum(-1)) - q)
        return np.stack(out, 1)

    def step(self, Xt, eps_t):
        dyn, P, E, t = self.dyn, self.P, self.E, len(self.X)
        C, ell, sf2, iK, beta = (dyn[k] for k in ("C", "ell", "sf2", "iK", "beta"))
        n = C.shape[0]
        K = np.stack([se_k(Xt, C, ell[e], sf2[e]) for e in range(E)])
        KiK = np.stack([K[e] @ iK[e][:n, :n] for e in range(E)])
        mu = np.stack([K[e] @ beta[e] for e in range(E)], 1)
        var = self._pairs(Xt, K, KiK, None)                 # [P,E]
        l = np.zeros((P, E, t), dtype=var.dtype)
        for s in range(t):                                  # forward substitution, one column at a time
            c = self._pairs(Xt, K, KiK, s)
            sub = (self.L[s] * l[:, :, :s]).sum(-1) if s else 0.0
            piv = self.piv[s]
            l[:, :, s] = np.where(piv > 0.0, (c - sub) / np.where(piv > 0.0, piv, 1.0), 0.0)
        d2 = var - (l * l).sum(-1)
        f = mu + np.sqrt(np.maximum(d2, 0.0)) * eps_t
        mean = mu
        if t:
            le = (l * np.stack(self.eps, -1)).sum(-1)
            f, mean = f + le, mu + le
        self.X.append(Xt.copy()); self.K.append(K); self.KiK.append(KiK)
        self.L.append(l); self.eps.append(eps_t.copy()); self.mean.append(mean); self.var.append(d2)
        self.piv.append(np.where(d2 > TAU * np.asarray(sf2).reshape(1, E), np.sqrt(np.maximum(d2, 0.0)), 0.0))
        return f


def joint_draw(dyn, Xs, eps):
    """f at the fixed inputs Xs [T,D] from the normals eps [T,E] as mu + chol(K_post) eps, per output (K_post positive
    definite) -> [T,E]"""
    K = _posterior(dyn, Xs, Xs)
    mu = gp_latent(dyn, Xs)[0]
    return mu + np.stack([np.linalg.cholesky(K[e]) @ eps[:, e] for e in range(K.shape[0])], 1)


def weights(terms, rew, risk, mult_mu=0.0, baseline=True):
    """w [P, H-1]: the return-to-go G_pt of every transition t < H-1 from the step rewards and risks [P,H], minus the
    leave-one-out mean of the other particles' G_qt when ``baseline`` (and P > 1)"""
    P, H = rew.shape
    mult = any(is_mult(t) for t in terms)
    G = np.zeros((P, max(H - 1, 0)))
    for t in range(H - 1):
        G[:, t] = rew[:, t + 1:].sum(1)
        if mult:
            G[:, t] += mult_mu * np.prod(1.0 - risk[:, :t + 1], 1) * (1.0 - np.prod(1.0 - risk[:, t + 1:], 1))
    if baseline and P > 1:
        G = G - (G.sum(0, keepdims=True) - G) / (P - 1)
    return G


def moment_check(samples, mean, cov, nse=5.0):
    """largest deviation, in standard errors estimated from the samples, of the sample mean and covariance of
    samples [P,Ds] from (mean [Ds], cov [Ds,Ds])"""
    P = samples.shape[0]
    xm = samples.mean(0)
    z = samples - xm
    worst = np.max(np.abs(xm - mean) / (samples.std(0) / np.sqrt(P)))
    for i in range(samples.shape[1]):
        for j in range(i + 1):
            zz = z[:, i] * z[:, j]
            worst = max(worst, abs(zz.mean() - cov[i, j]) / (zz.std() / np.sqrt(P)))
    return float(worst)
