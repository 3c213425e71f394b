"""What one joint state-action reward term costs at the metric shape (dynamics n = 300, D = 12, E = 10; RBF policy,
bf = 50; H = 40; R = 32 restarts): the moment-matching forward and forward + reverse sweep (taped) with (a) the one
state exponential reward and (b) the same plus one PILCO_REWARD_EXP_SA action cost, alternated in one process, and
likewise one pathwise particle gradient call at P = 1024 (one policy).  ms from CUDA events after a warm-up, the median
and the min-max spread over several repeats, with the card's name and power limit read in the same run.  Needs a GPU:
engine.device() raises without one.
    python scripts/action_reward_timing.py  -> one JSON line"""
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "scripts"))
from pilco_b200 import _lib, engine, rewards       # noqa: E402
from predict_timing import card, timeit            # noqa: E402
from util import make_rollout_problem              # noqa: E402

N, DS, U, BF, H, R, P = 300, 10, 2, 50, 40, 32, 1024
REPEATS, REPS = 7, 10


def alternate(arms):
    """{name: fn} -> {name: {median_ms, min_ms, max_ms}}: REPEATS rounds, each timing every arm once (REPS calls)"""
    ms = {k: [] for k in arms}
    for _ in range(REPEATS):
        for k, fn in arms.items():
            ms[k].append(timeit(fn, REPS))
    return {k: {"median_ms": float(np.median(v)), "min_ms": min(v), "max_ms": max(v)} for k, v in ms.items()}


def main():
    engine.device()
    out = {"card": card(), "shape": dict(n=N, D=DS + U, E=DS, bf=BF, H=H, R=R, P=P), "repeats": REPEATS}
    pb = make_rollout_problem(N, DS, U, BF, R, seed=0)
    gp = engine.gp_factorize(pb["X"], pb["Y"], pb["ell"], pb["sf2"], pb["sn2"])
    state = [dict(kind=_lib.REWARD_EXP, coef=1.0, W=pb["W"], t=pb["t"])]
    terms = {"state": state, "state_plus_exp_sa": state + rewards.action_cost(DS, U, 2.0 * np.eye(U)).terms(0.1)}

    def policy(r):
        lead = (slice(None),) if r is None else (r,)
        ones = np.ones((R, U)) if r is None else np.ones(U)
        pgp = engine.gp_factorize(pb["Xc"][lead], pb["Yc"][lead], pb["lc"][lead], ones, 1e-4 * ones, need_iK=False, mode=1)
        return dict(kind=_lib.POLICY_RBF, Ds=DS, U=U, squash=True, max_action=pb["maxa"], gp=pgp)

    fwd, both, part = {}, {}, {}
    for name, tt in terms.items():
        pf = engine.RolloutPlan(gp, policy(None), tt, pb["m0"], pb["S0"], H, R=R)
        pg = engine.RolloutPlan(gp, policy(None), tt, pb["m0"], pb["S0"], H, R=R, grad=True)
        fwd[name] = pf.forward
        both[name] = lambda pg=pg: (pg.forward(), pg.backward())
        pp = engine.ParticlePlan(gp, policy(0), tt, P, H, grad=True)
        rng = np.random.RandomState(1)
        pp.set_inputs(pb["m0"][None] + np.sqrt(0.1) * rng.randn(P, DS), rng.randn(P, H, DS))
        part[name] = pp.launch_grad
    out["rollout_forward"] = alternate(fwd)
    out["rollout_forward_backward"] = alternate(both)
    out["particle_gradient_P1024"] = alternate(part)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
