"""Timing of the consistent sampler's gradient (pilco_particles_rollout_consistent_grad) at the metric shape (dynamics
n = 300, D = 12, E = 10; RBF policy, bf = 50; one exponential reward; H = 40), in one process, ms from CUDA events after
a warm-up: the consistent forward alone against forward + gradient at P = 1024 and 4096; one batched call of R = 16
policies against the same 16 policies as 16 unbatched calls at P = 256; then the wall time of one
PILCO.optimize_policy_sampled(consistent=True, maxiter=50, restarts=32, num_samples=256) with its number of
evaluations; and the card's name and power limit read in the same run.
    python scripts/particle_consistent_grad_timing.py  -> one JSON line"""
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

H, BF, R, PB = 40, 50, 16, 256


def forward_vs_gradient(pb, gp, terms):
    out = {}
    pgp = engine.gp_factorize(pb["Xc"][0], pb["Yc"][0], pb["lc"][0], np.ones(2), 1e-4 * np.ones(2), need_iK=False,
                              mode=1)
    spec = dict(kind=_lib.POLICY_RBF, Ds=10, U=2, squash=True, max_action=pb["maxa"], gp=pgp)
    for P in (1024, 4096):
        rng = np.random.RandomState(P)
        x0, eps = pb["m0"][None] + np.sqrt(0.1) * rng.randn(P, 10), rng.randn(P, H, 10)
        fwd = engine.ParticlePlan(gp, spec, terms, P, H, consistent=True)
        fwd.set_inputs(x0, eps)
        t_fwd = timeit(fwd.launch, 5)
        ret = fwd.ret.clone()
        del fwd
        torch.cuda.empty_cache()
        grad = engine.ConsistentGradPlan(gp, spec, terms, P, H)
        grad.set_inputs(x0, eps)
        t_grad = timeit(grad.launch_grad, 5)
        out["P%d" % P] = {"forward_ms": t_fwd, "forward_and_gradient_ms": t_grad, "ratio": t_grad / t_fwd,
                          "workspace_GB": grad.gws.numel() * 8 / 1e9, "returns_bitwise_equal": torch.equal(ret, grad.ret)}
        del grad
        torch.cuda.empty_cache()
    return out


def batch_vs_sequential(pb, gp, terms):
    U = 2
    pgp = engine.gp_factorize(pb["Xc"][:R], pb["Yc"][:R], pb["lc"][:R], np.ones((R, U)), 1e-4 * np.ones((R, U)),
                              need_iK=False, mode=1)
    spec = dict(kind=_lib.POLICY_RBF, Ds=10, U=U, squash=True, max_action=pb["maxa"], gp=pgp)
    ldw = engine.pad_n(BF)
    singles = []
    for r in range(R):                          # restart r's policy arrays as an unbatched policy
        one = engine.DeviceGP(pgp.X[r], pgp.ell[r], pgp.sf2[r], pgp.beta[r], mode=1)
        one.fact_ws = pgp.fact_ws[r * U * ldw * ldw:(r + 1) * U * ldw * ldw]
        singles.append(dict(spec, gp=one))
    rng = np.random.RandomState(PB)
    x0, eps = pb["m0"][None] + np.sqrt(0.1) * rng.randn(PB, 10), rng.randn(PB, H, 10)
    batch = engine.ConsistentGradPlan(gp, spec, terms, PB, H, R=R)
    batch.set_inputs(x0, eps)
    plans = []
    for s in singles:
        p = engine.ConsistentGradPlan(gp, s, terms, PB, H)
        p.set_inputs(x0, eps)
        plans.append(p)
    t_batch = timeit(batch.launch_grad, 5)
    t_seq = timeit(lambda: [p.launch_grad() for p in plans], 3)
    same = all(torch.equal(batch.ret[r], plans[r].ret) for r in range(R))
    out = {"P": PB, "R": R, "batched_ms": t_batch, "sequential_ms": t_seq, "sequential_over_batched": t_seq / t_batch,
           "returns_bitwise_equal": same}
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
    kw = dict(num_samples=PB, consistent=True)
    start = pilco.sample_trajectories(pilco.m_init, pilco.S_init, H, seed=1, **kw).returns.mean()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    value = pilco.optimize_policy_sampled(maxiter=50, restarts=32, seed=1, **kw)
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    held_out = pilco.sample_trajectories(pilco.m_init, pilco.S_init, H, seed=2, **kw).returns.mean()
    st = policy_opt.LAST_STATS
    return {"wall_s": wall, "evals": int(st["evals"]), "groups": int(st["groups"]), "restarts": 32,
            "start_value": float(start), "best_value_in_sample": float(value), "value_other_seed": float(held_out)}


def main():
    engine.device()
    out = {"card": card(), "H": H}
    pb = make_rollout_problem(300, 10, 2, BF, R, seed=0)
    gp = engine.gp_factorize(pb["X"], pb["Y"], pb["ell"], pb["sf2"], pb["sn2"])
    terms = [dict(kind=_lib.REWARD_EXP, coef=1.0, W=pb["W"], t=pb["t"])]
    out["forward_vs_gradient"] = forward_vs_gradient(pb, gp, terms)
    out["batched_vs_sequential"] = batch_vs_sequential(pb, gp, terms)
    out["optimize_policy_sampled"] = optimisation(pb)
    out["card_after"] = card()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
