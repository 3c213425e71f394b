"""The kernels, memsets and copies one warmed-up call of the particle rollouts enqueues, in launch order, for a covering
set of their options (sampler, forward-only / pathwise / score-function gradient / batched forward, policy kind,
angles, measurement noise, exploration, state, joint and multiplicative box terms, restarts, horizon), and of one
CemPlan.launch() and one chunked ParticleBatchPlan.launch(), against
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

# name: sampler, call, policy, angle dims, measurement noise, exploration b, terms, R, H.  Samplers: step-wise, consistent,
# resampled, features; calls: forward, pathwise, score, ParticleBatchPlan ("batch", R policies; "_chunked": in chunks of
# 2) and CemPlan ("cem", R candidates, one iteration); policies: linear, RBF, scheduled linear, MLP.
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
    "res_fwd_linear": ("res", "fwd", "linear", (), False, None, "state", 1, 3),
    "res_path_rbf_joint_R2": ("res", "path", "rbf", (), False, None, "joint", 2, 3),
    "feat_fwd_linear_angles_noise_joint": ("feat", "fwd", "linear", (1,), True, None, "joint", 1, 3),
    "feat_path_rbf_explore_R2": ("feat", "path", "rbf", (), False, 0.3, "state", 2, 3),
    "step_batch_linear_angles_noise_box_R5_chunked": ("step", "batch", "linear", (1,), True, None, "box", 5, 3),
    "cons_batch_rbf_noise_joint_R3": ("cons", "batch", "rbf", (), True, None, "joint", 3, 3),
    "step_fwd_sched_angles_noise_box": ("step", "fwd", "sched", (1,), True, None, "box", 1, 3),
    "cons_fwd_sched": ("cons", "fwd", "sched", (), False, None, "state", 1, 3),
    "step_path_sched_explore_joint_R2": ("step", "path", "sched", (), False, 0.2, "joint", 2, 3),
    "cons_path_sched_angles_R2": ("cons", "path", "sched", (1,), False, None, "state", 2, 3),
    "step_score_sched_noise_box": ("step", "score", "sched", (), True, None, "box", 1, 3),
    "cons_score_sched_box_R2": ("cons", "score", "sched", (), False, None, "box", 2, 3),
    "res_fwd_sched": ("res", "fwd", "sched", (), False, None, "state", 1, 3),
    "res_path_sched_joint_R2": ("res", "path", "sched", (), False, None, "joint", 2, 3),
    "step_cem_sched_box_K4": ("step", "cem", "sched", (), False, None, "box", 4, 3),
    "cons_cem_sched_angles_noise_K4": ("cons", "cem", "sched", (1,), True, None, "state", 4, 3),
    "step_fwd_mlp": ("step", "fwd", "mlp", (), False, None, "state", 1, 3),
    "cons_fwd_mlp_joint": ("cons", "fwd", "mlp", (), False, None, "joint", 1, 3),
    "step_path_mlp_explore_R2": ("step", "path", "mlp", (), False, 0.3, "state", 2, 3),
    "cons_path_mlp_joint_R2": ("cons", "path", "mlp", (), False, None, "joint", 2, 3),
    "res_fwd_mlp": ("res", "fwd", "mlp", (), False, None, "state", 1, 3),
    "res_path_mlp_R2": ("res", "path", "mlp", (), False, None, "state", 2, 3),
    "feat_fwd_mlp": ("feat", "fwd", "mlp", (), False, None, "state", 1, 3),
    "feat_path_mlp_explore_b0_joint_R2": ("feat", "path", "mlp", (), False, 0.0, "joint", 2, 3),
    "step_batch_mlp_R3": ("step", "batch", "mlp", (), False, None, "state", 3, 3),
    "cons_batch_mlp_box_R3": ("cons", "batch", "mlp", (), False, None, "box", 3, 3),
}
F = 16                                                          # the feature sampler's features


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
    lead = (R,) if call == "batch" or (R > 1 and call != "cem") else ()       # CemPlan: R candidates of one W
    if kind in ("linear", "sched"):
        hw = (H,) if kind == "sched" else ()
        spec = dict(kind=_lib.POLICY_LINEAR, Ds=Dh, U=U, squash=True, max_action=maxa,
                    W=0.5 * rng.randn(*lead, *hw, U, Dh), b=0.3 * rng.randn(*lead, *hw, U), schedule=kind == "sched")
    elif kind == "mlp":
        spec = dict(kind=_lib.POLICY_MLP, Ds=Dh, U=U, squash=True, max_action=maxa, hidden=(8,),
                    theta=0.4 * rng.randn(*lead, engine.mlp_theta_size(Dh, U, (8,))))
    else:
        bf = 8
        pgp = engine.gp_factorize(rng.randn(*lead, bf, Dh) * 0.5 + 0.5, 0.1 * rng.randn(*lead, bf, U),
                                  1.0 + 0.1 * rng.randn(*lead, U, Dh), np.ones(lead + (U,)), 1e-4 * np.ones(lead + (U,)),
                                  need_iK=False, mode=1)
        spec = dict(kind=_lib.POLICY_RBF, Ds=Dh, U=U, squash=True, max_action=maxa, gp=pgp)
    gp = engine.gp_factorize(X, 0.1 * Y, ell, sf2, sn2)
    v = (0.01 + 0.05 * rng.rand(Ds)) if noise else None
    kw = dict(mult_mu=1.5, angles=list(dims) or None, measurement_noise=v)
    if call == "cem":
        plan = engine.CemPlan(gp, spec, _terms(terms, Dh), P, H, R, 2, 1, consistent=sampler == "cons", **kw)
    elif call == "batch":
        plan = engine.ParticleBatchPlan(gp, spec, _terms(terms, Dh), P, H, R, consistent=sampler == "cons", **kw)
        if name.endswith("_chunked"):
            plan = engine.ParticleBatchPlan(gp, spec, _terms(terms, Dh), P, H, R, consistent=sampler == "cons",
                                            max_ws_bytes=plan.bytes_needed(2), **kw)
            assert len(plan.chunks) == 3
    else:
        kw.update(R=R, exploration=b, schedule=kind == "sched", resample=sampler == "res",
                  num_features=F if sampler == "feat" else None)
        est = "score" if call == "score" else "pathwise"
        if sampler in ("cons", "feat") and call != "fwd":
            del kw["resample"]
            plan = engine.ConsistentGradPlan(gp, spec, _terms(terms, Dh), P, H, estimator=est, **kw)
        else:
            plan = engine.ParticlePlan(gp, spec, _terms(terms, Dh), P, H, grad=call != "fwd", estimator=est,
                                       consistent=sampler in ("cons", "feat"), **kw)
    x0 = 0.5 + 0.2 * rng.randn(P, Ds)
    eps, nu = rng.randn(P, H, Ds), rng.randn(P, H, Ds) if noise else None
    if call == "cem":
        plan.set_inputs(x0, eps, rng.randn(1, R, H, U), nu)
    elif call == "batch":
        plan.set_inputs(x0, eps, nu)
    elif sampler == "res":
        plan.set_inputs(x0, eps, nu, xi=rng.randn(P, H, Ds))
    elif sampler == "feat":
        draws = engine.feature_draws(gp, P, F, rng.randn(Ds, F, Dh + U), rng.randn(P, Ds, 2 * F), rng.randn(P, Ds, 40))
        plan.set_inputs(x0, None, nu, features=draws)
    else:
        plan.set_inputs(x0, eps, nu)
    return plan


def run(plan):
    """one call of the plan's case"""
    if getattr(plan, "grad", None) is None:
        plan.launch()
    else:
        plan.launch_grad()


def launches(plan):
    """device activity names of one call, in launch order (after a warm-up call).  The capture opens with a fill kernel,
    a synchronise and a 10 ms pause, and the fill and anything before it are dropped: the profiler can miss an activity
    that starts right after the capture opens, and that would drop the call's first launch.  The marker is the one
    float32 fill (CemPlan's call fills fp64 tensors); when the profiler misses it, nothing is dropped."""
    run(plan)
    marker = torch.empty(1, dtype=torch.float32, device="cuda")
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
    fills = [i for i, n in enumerate(names) if "FillFunctor<float>" in n]
    return names[fills[0] + 1:] if fills else names


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
