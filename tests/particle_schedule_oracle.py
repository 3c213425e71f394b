"""Time-varying linear policies (DESIGN.md section 28) in the shared particle oracles, tests/particle_oracle.py (numpy)
and tests/particle_grad_oracle.py (torch), without a copy of their step loops.

Both oracles evaluate the policy exactly once per step, in step order: the numpy loop calls ``po.policy_action(pol, z)``,
the torch loops (``value_and_grad``, ``consistent_value_and_grad``, ``resampled_rollout``, ``score_grad``) make one
action closure per rollout with ``pgo.policy(pol)`` and call it once per step.  Inside ``with schedule(pol):`` those two
names serve the scheduled linear policy pol = dict(kind, squash, maxa, W [H,U,Dh], b [H,U]), H the rollout's horizon:
a rollout's k-th evaluation reads W[k], b[k], and the torch gradients are per step, {'W' [H,U,Dh], 'b' [H,U]}.  Any
other policy dict goes to the oracles' own functions.  The action is the stationary oracles' expression at W[k], b[k],
so a constant schedule reproduces the stationary oracles bit for bit.  Test infrastructure only."""
import contextlib

import numpy as np
import torch

import particle_grad_oracle as pgo
import particle_oracle as po


@contextlib.contextmanager
def schedule(pol):
    W, b = np.asarray(pol["W"], dtype=np.float64), np.asarray(pol["b"], dtype=np.float64)
    H = W.shape[0]
    np_action, torch_policy = po.policy_action, pgo.policy
    calls = [0]                                         # numpy evaluations so far; a rollout takes H of them

    def policy_action(p, x):
        if p is not pol:
            return np_action(p, x)
        t = calls[0] % H
        calls[0] += 1
        return np_action(dict(p, W=W[t], b=b[t]), x)

    def policy(p):
        if p is not pol:
            return torch_policy(p)
        prm = {"W": pgo.T(W).clone().requires_grad_(), "b": pgo.T(b).clone().requires_grad_()}
        maxa = pgo.T(p["maxa"]).reshape(1, -1)
        step = [0]

        def act(x):                                     # pgo.policy's linear action at step t's W_t, b_t
            t = step[0] % H
            step[0] += 1
            raw = x @ prm["W"][t].T + prm["b"][t][None]
            return maxa * np.exp(-0.5 * 0.0) * torch.sin(raw) if p.get("squash", True) else raw
        return prm, act

    po.policy_action, pgo.policy = policy_action, policy
    try:
        yield
    finally:
        po.policy_action, pgo.policy = np_action, torch_policy
