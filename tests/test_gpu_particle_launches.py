"""The kernels, memsets and copies one warmed-up call of the particle rollouts enqueues, in launch order, for a covering
set of their options (sampler, forward-only / pathwise / score-function gradient, policy kind, angles, measurement
noise, exploration, state, joint and multiplicative box terms, restarts, horizon), against
tests/golden/particle_launches.json (tests/golden/make_particle_launches.py).  It pins that each call runs exactly the
launches it ran when the golden was recorded, whichever C entry point the engine reaches it through."""
import json
import os
import subprocess
import sys
import time

import numpy as np
import pytest
import torch

from pilco_b200 import engine, _lib, rewards
from particle_cases import BOX2
from util import make_gp_problem

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "particle_launches.json")
MAKER = os.path.join(HERE, "golden", "make_particle_launches.py")
Ds, U, P = 3, 1, 200

# name: sampler, call, policy, angle dims, measurement noise, exploration b, terms, R, H
CASES = {
    "step_fwd_linear": ("step", "fwd", "linear", (), False, None, "state", 1, 3),
    "step_fwd_rbf_angles_joint": ("step", "fwd", "rbf", (1,), False, None, "joint", 1, 3),
    "step_fwd_linear_noise_box": ("step", "fwd", "linear", (), True, None, "box", 1, 1),
    "cons_fwd_rbf_box": ("cons", "fwd", "rbf", (), False, None, "box", 1, 3),
    "cons_fwd_linear_angles_noise_joint": ("cons", "fwd", "linear", (0,), True, None, "joint", 1, 3),
    "step_path_linear": ("step", "path", "linear", (), False, None, "state", 1, 3),
    "step_path_rbf_joint_R2": ("step", "path", "rbf", (), False, None, "joint", 2, 3),
    "step_path_linear_angles_box_R2": ("step", "path", "linear", (1,), False, None, "box", 2, 3),
    "step_path_rbf_noise_H1": ("step", "path", "rbf", (), True, None, "state", 1, 1),
    "step_path_linear_angles_noise_joint_R2": ("step", "path", "linear", (0, 2), True, None, "joint", 2, 3),
    "step_path_rbf_explore_b0_R2": ("step", "path", "rbf", (), False, 0.0, "state", 2, 3),
    "step_path_linear_angles_noise_explore_joint": ("step", "path", "linear", (1,), True, 0.4, "joint", 1, 3),
    "step_score_linear_box_R2": ("step", "score", "linear", (), False, None, "box", 2, 3),
    "step_score_rbf_angles_joint": ("step", "score", "rbf", (1,), False, None, "joint", 1, 3),
    "step_score_linear_noise_R2_H1": ("step", "score", "linear", (), True, None, "state", 2, 1),
    "cons_path_linear": ("cons", "path", "linear", (), False, None, "state", 1, 3),
    "cons_path_rbf_angles_noise_joint_R2": ("cons", "path", "rbf", (1,), True, None, "joint", 2, 3),
    "cons_path_linear_explore_R2": ("cons", "path", "linear", (), False, 0.3, "state", 2, 3),
    "cons_path_rbf_noise_explore_b0_joint_H1": ("cons", "path", "rbf", (), True, 0.0, "joint", 1, 1),
    "cons_score_linear_box_R2": ("cons", "score", "linear", (), False, None, "box", 2, 3),
    "cons_score_rbf_angles_noise_joint": ("cons", "score", "rbf", (1,), True, None, "joint", 1, 3),
}


def _terms(which, Dh, seed=0):
    rng = np.random.RandomState(seed)
    t = 0.4 * rng.randn(Ds)
    state = rewards.CombinedRewards(Ds, [rewards.ExponentialReward(Ds, W=np.diag(0.5 + rng.rand(Ds)), t=t),
                                         rewards.LinearReward(Ds, rng.randn(Ds))], coefs=[1.0, 0.3]).terms()
    if which == "state":
        return state
    if which == "box":
        return state + [dict(kind=_lib.REWARD_BOX, coef=1.0, channel=_lib.CHANNEL_MULT, W=BOX2, t=None)]
    combined = rewards.CombinedRewards(Ds, [rewards.ExponentialReward(Ds, t=t), rewards.action_cost(Dh, U)],
                                       coefs=[1.0, 0.2]).terms()
    return combined + [dict(kind=_lib.REWARD_LINEAR_SA, coef=0.3, W=rng.randn(Dh + U), t=None)]


def make_plan(name, seed=5):
    """the seeded plan of case `name`, its inputs set"""
    sampler, call, kind, dims, noise, b, terms, R, H = CASES[name]
    Dh = Ds + len(dims)
    X, Y, ell, sf2, sn2 = make_gp_problem(40, Dh + U, Ds, seed=seed)
    rng = np.random.RandomState(seed + 1)
    maxa = 0.7 + rng.rand(U)
    lead = (R,) if R > 1 else ()
    if kind == "linear":
        spec = dict(kind=_lib.POLICY_LINEAR, Ds=Dh, U=U, squash=True, max_action=maxa, W=0.5 * rng.randn(*lead, U, Dh),
                    b=0.3 * rng.randn(*lead, U))
    else:
        bf = 8
        pgp = engine.gp_factorize(rng.randn(*lead, bf, Dh) * 0.5 + 0.5, 0.1 * rng.randn(*lead, bf, U),
                                  1.0 + 0.1 * rng.randn(*lead, U, Dh), np.ones(lead + (U,)), 1e-4 * np.ones(lead + (U,)),
                                  need_iK=False, mode=1)
        spec = dict(kind=_lib.POLICY_RBF, Ds=Dh, U=U, squash=True, max_action=maxa, gp=pgp)
    gp = engine.gp_factorize(X, 0.1 * Y, ell, sf2, sn2)
    kw = dict(mult_mu=1.5, R=R, angles=list(dims) or None, exploration=b,
              measurement_noise=(0.01 + 0.05 * rng.rand(Ds)) if noise else None)
    est = "score" if call == "score" else "pathwise"
    if sampler == "cons" and call != "fwd":
        plan = engine.ConsistentGradPlan(gp, spec, _terms(terms, Dh), P, H, estimator=est, **kw)
    else:
        plan = engine.ParticlePlan(gp, spec, _terms(terms, Dh), P, H, grad=call != "fwd", estimator=est,
                                   consistent=sampler == "cons", **kw)
    x0 = 0.5 + 0.2 * rng.randn(P, Ds)
    plan.set_inputs(x0, rng.randn(P, H, Ds), rng.randn(P, H, Ds) if noise else None)
    return plan


def run(plan):
    """one call of the plan's case"""
    if plan.grad is None:
        plan.launch()
    else:
        plan.launch_grad()


def launches(plan):
    """device activity names of one call, in launch order (after a warm-up call).  The capture opens with a fill kernel,
    a synchronise and a 10 ms pause, and the fill and anything before it are dropped: the profiler can miss an activity
    that starts right after the capture opens, and that would drop the call's first launch."""
    run(plan)
    marker = torch.empty(1, device="cuda")
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        marker.fill_(1.0)
        torch.cuda.synchronize()
        time.sleep(0.01)
        run(plan)
        torch.cuda.synchronize()
    ev = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    ev.sort(key=lambda e: e.time_range.start)
    names = [e.name for e in ev]
    fills = [i for i, n in enumerate(names) if "FillFunctor" in n]
    return names[fills[-1] + 1:] if fills else names


def record():
    return {name: launches(make_plan(name)) for name in CASES}


@pytest.fixture(scope="module")
def recorded(tmp_path_factory):
    """every case's launches, recorded by the golden's maker in a child process, so no profiler capture is taken in the
    test process: after captures here, later captures in the same process (the moment-matching launch test's, minutes
    later in the suite) came back without their first launches, or empty."""
    out = tmp_path_factory.mktemp("particle_launches") / "launches.json"
    flags = [f for f, on in (("-I", sys.flags.isolated), ("-E", sys.flags.ignore_environment),
                             ("-s", sys.flags.no_user_site)) if on]
    res = subprocess.run([sys.executable, *flags, MAKER, str(out)], capture_output=True, text=True, timeout=1200)
    assert res.returncode == 0, res.stdout[-4000:] + res.stderr[-4000:]
    with open(out) as f:
        return json.load(f)


@pytest.mark.parametrize("name", sorted(CASES))
def test_launch_sequence(name, recorded):
    with open(GOLDEN) as f:
        want = json.load(f)[name]
    got = recorded[name]
    assert got == want, "\n".join("%3d %s | %s" % (i, g, w) for i, (g, w) in enumerate(zip(got, want)) if g != w)
    assert len(got) == len(want)
