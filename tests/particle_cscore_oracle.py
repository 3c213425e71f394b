"""Torch statement of the score-function gradient over consistent function samples (pilco_particles_consistent_score_grad_*,
DESIGN.md section 25) for the tests.  Given a consistent rollout (traj [P,H+1,E], the normals eps [P,H,E] that drove it,
and with measurement noise nu [P,H,E] and its variances v) it forms, per particle and output, the surrogate

    J(theta) = (1/P) sum_p sum_{t<H-1, piv_t>0} w_pt (-eps_t(theta)^2 / 2 - log piv_t(theta)),
    eps_t(theta) = (f_t - mean'_t(theta)) / piv_t(theta),  mean'_t = mu(x~_t) + sum_{s<t} l_ts eps_s(theta)

with the increments f_t = x_{t+1} - x_t and the states held fixed, theta entering through u_s = pi(phi(z_s)) inside every
x~_s = [phi(x_s), u_s], and returns autograd's gradient at the rollout's theta.  The factor rows and pivots are those of
particle_grad_oracle.TorchFunctionSample (the same tau mask); a masked step drops its term and keeps the caller's
eps_t.  eps_t(theta) takes the caller's eps_t as its value and (f_t - mean'_t) / piv_t's derivative, so the rounding
of f_t does not enter.  w_pt is particle_oracle.weights (or ``w``), and with ``direct`` the joint terms' own dependence on
the parameters through u_t at fixed states is added as particle_grad_oracle.score_grad adds it.  Test infrastructure
only."""
import numpy as np
import torch

import particle_angles_oracle as pao
import particle_grad_oracle as pgo
import particle_noise_oracle as pno
import particle_oracle as po

F64 = torch.float64


def score_grad(dyn, pol, terms, traj, eps, mult_mu=0.0, nu=None, v=None, angle_dims=None, baseline=True, direct=True,
               swap=False, w=None):
    """-> ({'W','b'} or {'X','Y','ell'} numpy arrays, the smallest kept pivot d2 / (TAU sf2) of the steps t < H-1)"""
    traj, eps = np.asarray(traj, dtype=np.float64), np.asarray(eps, dtype=np.float64)
    P, H, E = eps.shape
    sv = pno._scale(v)
    prm, act = pgo.policy(pol)
    if H == 0:
        return pgo._grads(torch.zeros(()), prm), np.inf
    xs = [pao.feature_map_torch(pgo.T(traj[:, s]), angle_dims) for s in range(H)]
    zs = xs if sv is None else [pao.feature_map_torch(pgo.T(pno.measurement(traj[:, s], nu[:, s], sv)), angle_dims)
                                for s in range(H)]
    us = [act(z) for z in zs]
    rew, risk = pao.path_rewards(terms, traj, np.stack([u.detach().numpy() for u in us], 1), angle_dims)
    W = po.weights(terms, rew, risk, mult_mu, baseline) if w is None else np.asarray(w, dtype=np.float64)
    fs = pgo.TorchFunctionSample(dyn, swap)
    sur = torch.zeros((), dtype=F64)
    for t in range(H - 1):
        e = pgo.T(eps[:, t])
        mean, _ = fs.step(torch.cat([xs[t], us[t]], 1), e)
        piv = fs.piv[-1]
        on = piv > 0.0
        safe = torch.where(on, piv, torch.ones_like(piv))
        r = (pgo.T(traj[:, t + 1] - traj[:, t]) - mean) / safe
        et = torch.where(on, e + (r - r.detach()), e)              # the caller's value, the residual's derivative
        fs.eps[-1] = et                                            # what the later steps' mean' reads
        term = torch.where(on, -0.5 * et * et - torch.log(safe), torch.zeros_like(et))
        sur = sur + (pgo.T(W[:, t])[:, None] * term).sum()
    if direct:
        mult = any(po.is_mult(t) for t in terms)
        for s, (x, u) in enumerate(zip(xs, us)):
            wm = mult_mu * np.prod(np.delete(1.0 - risk, s, axis=1), axis=1) if mult else np.zeros(P)
            for term in terms:
                if po.is_joint(term):
                    c = float(term.get("coef", 1.0)) * (pgo.T(wm) if po.is_mult(term) else 1.0)
                    sur = sur + (c * pgo.point_value(term, x, u)).sum()
    return pgo._grads(sur / P, prm), fs.min_ratio
