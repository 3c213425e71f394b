"""Tanh MLP policies (DESIGN.md section 29) in the shared particle oracles, tests/particle_oracle.py (numpy) and
tests/particle_grad_oracle.py (torch), without a copy of their step loops.

Both oracles evaluate the policy through one name each: the numpy loop calls ``po.policy_action(pol, z)``, the torch
loops (``value_and_grad``, ``consistent_value_and_grad``, ``resampled_rollout``) make one action closure per rollout
with ``pgo.policy(pol)``.  Inside ``with mlp_policies():`` those two names also serve an MLP policy dict
pol = dict(kind=POLICY_MLP, squash, maxa, Ds, U, hidden, theta [n_theta]):
    h_1 = tanh(A_1 [x; 1]), (two layers) h_2 = tanh(A_2 [h_1; 1]), z = A_out [h_L; 1], u = maxa sin(z) or z
with theta = A_1, (A_2,) A_out, each row-major [out, in + 1] with the bias last; the torch gradient is {'theta'}.
Every other policy dict goes to the oracles' own functions unchanged.  Test infrastructure only."""
import contextlib

import numpy as np
import torch

import particle_grad_oracle as pgo
import particle_oracle as po
from pilco_b200 import _lib


def mlp_layers(theta, Ds, U, hidden):
    """a tanh MLP's flat theta (numpy or torch) -> its blocks A_l [out, in + 1], in order, output layer last"""
    widths = [int(Ds)] + [int(w) for w in hidden] + [int(U)]
    out, o = [], 0
    for l in range(len(widths) - 1):
        n = widths[l + 1] * (widths[l] + 1)
        out.append(theta[o:o + n].reshape(widths[l + 1], widths[l] + 1))
        o += n
    assert o == theta.shape[-1], "theta has %d entries, the MLP %d" % (theta.shape[-1], o)
    return out


def _raw(layers, x, tanh):
    """z = A_out [h_L; 1] at the rows of x (numpy or torch)"""
    h = x
    for l, A in enumerate(layers):
        h = h @ A[:, :-1].T + A[:, -1][None]
        if l < len(layers) - 1:
            h = tanh(h)
    return h


def action(pol, x):
    """the squashed action [P,U] of the MLP pol at the rows of x (numpy), output variance 0 as the linear policy"""
    layers = mlp_layers(np.asarray(pol["theta"], dtype=np.float64), pol["Ds"], pol["U"], pol["hidden"])
    u = _raw(layers, x, np.tanh)
    if pol.get("squash", True):
        u = np.asarray(pol["maxa"]).reshape(1, -1) * np.exp(-0.5 * 0.0) * np.sin(u)
    return u


def policy(pol):
    """pgo.policy for the MLP pol: ({'theta' with requires_grad}, x -> squashed action)"""
    prm = {"theta": pgo.T(pol["theta"]).reshape(-1).clone().requires_grad_()}
    layers = mlp_layers(prm["theta"], pol["Ds"], pol["U"], pol["hidden"])
    maxa = pgo.T(pol["maxa"]).reshape(1, -1)
    raw = lambda x: _raw(layers, x, torch.tanh)
    act = (lambda x: maxa * np.exp(-0.5 * 0.0) * torch.sin(raw(x))) if pol.get("squash", True) else raw
    return prm, act


@contextlib.contextmanager
def mlp_policies():
    np_action, torch_policy = po.policy_action, pgo.policy
    is_mlp = lambda p: p["kind"] == _lib.POLICY_MLP

    po.policy_action = lambda p, x: action(p, x) if is_mlp(p) else np_action(p, x)
    pgo.policy = lambda p: policy(p) if is_mlp(p) else torch_policy(p)
    try:
        yield
    finally:
        po.policy_action, pgo.policy = np_action, torch_policy
