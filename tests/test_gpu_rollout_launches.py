"""The kernels, memsets and copies one forward plus one reverse sweep of the moment-matching rollout enqueues, in launch
order, for a covering set of its options (policy kind, angles, measurement noise, exploration, joint and multiplicative
reward terms, taped and recomputing reverse sweep), against tests/golden/rollout_launches.json
(tests/golden/make_rollout_launches.py).  It pins that a rollout without a feature runs exactly the launches it ran
before that feature existed, and that each feature adds only its own."""
import json
import os

import numpy as np
import pytest
import torch

from pilco_b200 import engine, _lib, rewards
from particle_cases import BOX2
from util import make_gp_problem

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "rollout_launches.json")
H, R, Ds, U = 3, 2, 3, 1

# name: policy, angle dims, terms, exploration b, measurement noise, taped reverse sweep
CASES = {
    "linear": ("linear", (), "state", None, False, True),
    "linear_recompute": ("linear", (), "state", None, False, False),
    "rbf": ("rbf", (), "state", None, False, True),
    "rbf_recompute": ("rbf", (), "state", None, False, False),
    "rbf_joint": ("rbf", (), "joint", None, False, True),
    "linear_safe_recompute": ("linear", (), "safe", None, False, False),
    "rbf_angles": ("rbf", (1,), "state", None, False, True),
    "rbf_angles_recompute": ("rbf", (0, 2), "joint", None, False, False),
    "linear_angles_joint": ("linear", (1,), "joint", None, False, True),
    "rbf_explore": ("rbf", (), "joint", 0.4, False, True),
    "linear_explore_b0": ("linear", (), "state", 0.0, False, False),
    "rbf_angles_explore": ("rbf", (1,), "state", 0.3, False, False),
    "rbf_noise": ("rbf", (), "state", None, True, True),
    "linear_noise_recompute": ("linear", (), "joint", None, True, False),
    "rbf_angles_noise_explore": ("rbf", (1,), "joint", 0.5, True, True),
    "linear_angles_noise_recompute": ("linear", (0,), "safe", None, True, False),
}


def _terms(which, Dh, seed=0):
    rng = np.random.RandomState(seed)
    t = 0.4 * rng.randn(Ds)
    state = rewards.CombinedRewards(Ds, [rewards.ExponentialReward(Ds, W=np.diag(0.5 + rng.rand(Ds)), t=t),
                                         rewards.LinearReward(Ds, rng.randn(Ds))], coefs=[1.0, 0.3]).terms()
    if which == "state":
        return state
    if which == "safe":
        return state + [dict(kind=_lib.REWARD_BOX, coef=1.0, channel=_lib.CHANNEL_MULT, W=BOX2, t=None)]
    combined = rewards.CombinedRewards(Ds, [rewards.ExponentialReward(Ds, t=t), rewards.action_cost(Dh, U)],
                                       coefs=[1.0, 0.2]).terms()
    return combined + [dict(kind=_lib.REWARD_LINEAR_SA, coef=0.3, W=rng.randn(Dh + U), t=None)]


def make_plan(name, seed=5):
    """the seeded RolloutPlan of case `name`"""
    kind, dims, terms, b, noise, taped = CASES[name]
    Dh = Ds + len(dims)
    X, Y, ell, sf2, sn2 = make_gp_problem(40, Dh + U, Ds, seed=seed)
    rng = np.random.RandomState(seed + 1)
    maxa = 0.7 + rng.rand(U)
    if kind == "linear":
        spec = dict(kind=_lib.POLICY_LINEAR, Ds=Dh, U=U, squash=True, max_action=maxa, W=0.5 * rng.randn(R, U, Dh),
                    b=0.3 * rng.randn(R, U))
    else:
        bf = 8
        pgp = engine.gp_factorize(rng.randn(R, bf, Dh) * 0.5 + 0.5, 0.1 * rng.randn(R, bf, U),
                                  1.0 + 0.1 * rng.randn(R, U, Dh), np.ones((R, U)), 1e-4 * np.ones((R, U)),
                                  need_iK=False, mode=1)
        spec = dict(kind=_lib.POLICY_RBF, Ds=Dh, U=U, squash=True, max_action=maxa, gp=pgp)
    B = rng.randn(Ds, Ds)
    gp = engine.gp_factorize(X, 0.1 * Y, ell, sf2, sn2)
    return engine.RolloutPlan(gp, spec, _terms(terms, Dh), X[0, :Ds], 0.03 * B @ B.T + 0.02 * np.eye(Ds), H, R=R,
                              mult_mu=1.5, grad=taped, angles=list(dims) or None, exploration=b,
                              measurement_noise=(0.01 + 0.05 * rng.rand(Ds)) if noise else None)


def launches(plan):
    """device activity names of one forward() + backward(), in launch order (after a warm-up pair)"""
    plan.forward()
    plan.backward()
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        plan.forward()
        plan.backward()
        torch.cuda.synchronize()
    ev = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    ev.sort(key=lambda e: e.time_range.start)
    return [e.name for e in ev]


def record():
    return {name: launches(make_plan(name)) for name in CASES}


@pytest.mark.parametrize("name", sorted(CASES))
def test_launch_sequence(name):
    with open(GOLDEN) as f:
        want = json.load(f)[name]
    plan = make_plan(name)
    assert (plan.tape is not None) == CASES[name][5]
    got = launches(plan)
    assert got == want, "\n".join("%3d %s | %s" % (i, g, w) for i, (g, w) in enumerate(zip(got, want)) if g != w)
