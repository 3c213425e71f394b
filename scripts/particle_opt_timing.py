"""Timing of policy optimisation on the sampled return at the metric shape (dynamics n = 300, D = 12, E = 10; RBF
policy, bf = 50; one exponential reward; H = 40): one batched pilco_particles_rollout_batch_grad call of R = 32 policies
against the same 32 policies as 32 sequential pilco_particles_rollout_grad calls, at P = 256 and 1024 particles (ms
from CUDA events after a warm-up), then the wall time of one PILCO.optimize_policy_sampled(maxiter=50, restarts=32,
num_samples=1024) with its number of evaluations, and the card's name and power limit read in the same run.
    python scripts/particle_opt_timing.py  -> one JSON line"""
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "scripts"))
from pilco_b200 import _lib, engine, policy_opt   # noqa: E402
from predict_timing import card, timeit            # noqa: E402
from util import make_rollout_problem              # noqa: E402

PS = (256, 1024)
R, H, BF = 32, 40, 50


def batch_vs_sequential(pb, gp, terms):
    out = {}
    Ds, U = 10, 2
    pgp = engine.gp_factorize(pb["Xc"], pb["Yc"], pb["lc"], np.ones((R, U)), 1e-4 * np.ones((R, U)),
                              need_iK=False, mode=1)
    spec = dict(kind=_lib.POLICY_RBF, Ds=Ds, U=U, squash=True, max_action=pb["maxa"], gp=pgp)
    ldw = engine.pad_n(BF)
    singles = []
    for r in range(R):                          # restart r's policy arrays as an unbatched policy
        one = engine.DeviceGP(pgp.X[r], pgp.ell[r], pgp.sf2[r], pgp.beta[r], mode=1)
        one.fact_ws = pgp.fact_ws[r * U * ldw * ldw:(r + 1) * U * ldw * ldw]
        singles.append(dict(spec, gp=one))
    for P in PS:
        rng = np.random.RandomState(P)
        x0, eps = pb["m0"][None] + np.sqrt(0.1) * rng.randn(P, Ds), rng.randn(P, H, Ds)
        batch = engine.ParticlePlan(gp, spec, terms, P, H, grad=True, R=R)
        batch.set_inputs(x0, eps)
        plans = []
        for s in singles:
            p = engine.ParticlePlan(gp, s, terms, P, H, grad=True)
            p.set_inputs(x0, eps)
            plans.append(p)
        t_batch = timeit(batch.launch_grad, 5)
        t_seq = timeit(lambda: [p.launch_grad() for p in plans], 3)
        same = all(torch.equal(batch.ret[r], plans[r].ret) for r in range(R))
        out["P%d" % P] = {"batched_ms": t_batch, "sequential_ms": t_seq, "sequential_over_batched": t_seq / t_batch,
                          "batched_ns_per_particle_step": t_batch * 1e6 / (R * P * H), "returns_bitwise_equal": same}
        del batch, plans
        torch.cuda.empty_cache()
    return out


def optimisation(pb):
    from pilco.models import PILCO
    from pilco.controllers import RbfController
    from pilco.rewards import ExponentialReward
    np.random.seed(0)
    pilco = PILCO((pb["X"], pb["Y"]), controller=RbfController(10, 2, BF, max_action=1.0), horizon=H,
                  reward=ExponentialReward(10, pb["W"], pb["t"]), m_init=pb["m0"][None], S_init=pb["S0"])
    start = pilco.sample_trajectories(pilco.m_init, pilco.S_init, H, num_samples=1024, seed=1).returns.mean()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    value = pilco.optimize_policy_sampled(maxiter=50, restarts=R, num_samples=1024, seed=1)
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    held_out = pilco.sample_trajectories(pilco.m_init, pilco.S_init, H, num_samples=1024, seed=2).returns.mean()
    st = policy_opt.LAST_STATS
    return {"wall_s": wall, "evals": int(st["evals"]), "groups": int(st["groups"]), "restarts": R,
            "start_value": float(start), "best_value_in_sample": float(value), "value_other_seed": float(held_out)}


def main():
    engine.device()
    out = {"card": card(), "R": R, "H": H}
    pb = make_rollout_problem(300, 10, 2, BF, R, seed=0)
    gp = engine.gp_factorize(pb["X"], pb["Y"], pb["ell"], pb["sf2"], pb["sn2"])
    terms = [dict(kind=_lib.REWARD_EXP, coef=1.0, W=pb["W"], t=pb["t"])]
    out.update(batch_vs_sequential(pb, gp, terms))
    out["optimize_policy_sampled"] = optimisation(pb)
    out["card_after"] = card()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
