"""Torch statement of the moment-matching rollout under a time-varying linear policy (pilco_rollout_scheduled_*,
DESIGN.md section 27): step t applies u_t = sq(W_t x~ + b_t) through oracle/torch_port.py's linear_action and
squash_sin, and everything else is tests/obs_noise_oracle.py's cascade (angles, measurement noise, exploration, joint
terms, the SafePILCO channel).  A constant schedule is that oracle's stationary linear policy step for step.  Autograd
through it is the gradient oracle.  Test infrastructure only."""
import numpy as np
import torch

import obs_noise_oracle as no
from oracle import torch_port as tp

F64 = torch.float64
T = no.T


def step_action(Ws, bs, maxa):
    """the action function of the cascade: call k applies (Ws[k], bs[k]); Ws [H,U,Dh], bs [H,U] (tensors)"""
    step = [0]

    def act(m, s):
        t = step[0]
        step[0] += 1
        return tp.linear_action(Ws[t], bs[t].reshape(1, -1), m, s, maxa)
    return act


def dynamics(X, Y, ell, sf2, sn2, Z=None):
    """the dynamics moment match of an exact GP, or of FITC over the inducing points Z"""
    if Z is None:
        iK, beta = tp.calculate_factorizations(T(X), T(Y), T(ell), T(sf2), T(sn2))
        C = T(X)
    else:
        iK, beta = tp.fitc_factorizations(T(X), T(Z), T(Y), T(ell), T(sf2), T(sn2))
        C = T(Z)
    return lambda m, s: tp.predict_given_factorizations(C, T(ell), T(sf2), m, s, iK, beta)


def scheduled_rollout(dyn_fn, Ws, bs, maxa, terms, m0, S0, H, b=0.0, v=None, mult_mu=0.0, angle_dims=None):
    """the H-step cascade from N(m0, S0) under the schedule (Ws [>=H,U,Dh], bs [>=H,U]); maxa [U] or None (no squash);
    v: measurement-noise variances [Ds] or None.  -> obs_noise_oracle.noisy_rollout's dict"""
    ma = None if maxa is None else T(maxa)[None]
    m0 = m0 if torch.is_tensor(m0) else T(m0)
    S0 = S0 if torch.is_tensor(S0) else T(S0)
    v = torch.zeros(S0.shape[0], dtype=F64) if v is None else T(np.asarray(v, dtype=np.float64))
    return no.noisy_rollout(dyn_fn, step_action(Ws, bs, ma), terms, m0, S0, H, b, v, mult_mu, angle_dims)
