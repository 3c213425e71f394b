"""Timing and variance of pilco_particles_rollout_score_grad at the metric shape (dynamics n = 300, D = 12, E = 10; RBF
policy, bf = 50; one exponential reward), H = 40, P = 1024 and 16384: ms of the forward alone (pilco_particles_rollout),
of forward + pathwise gradient and of forward + score gradient, from CUDA events after a warm-up, the three alternated
in one process (median of the rounds).  Then, over 16 seeds at P = 1024, each estimator's summed per-component
variance of grad at H = 10 and H = 40 (the PIPPS comparison), and the card's name and power limit read in the same run.
    python scripts/particle_score_timing.py  -> one JSON line"""
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "scripts"))
from pilco_b200 import _lib, engine             # noqa: E402
from predict_timing import card, timeit          # noqa: E402
from util import make_rollout_problem            # noqa: E402

PS = (1024, 16384)
H = 40
ROUNDS = 5
SEEDS = 16


def _problem():
    pb = make_rollout_problem(300, 10, 2, 50, 1, seed=0)
    gp = engine.gp_factorize(pb["X"], pb["Y"], pb["ell"], pb["sf2"], pb["sn2"])
    pgp = engine.gp_factorize(pb["Xc"][0], pb["Yc"][0], pb["lc"][0], np.ones(2), 1e-4 * np.ones(2), need_iK=False, mode=1)
    spec = dict(kind=_lib.POLICY_RBF, Ds=10, U=2, squash=True, max_action=pb["maxa"], gp=pgp)
    terms = [dict(kind=_lib.REWARD_EXP, coef=1.0, W=pb["W"], t=pb["t"])]
    return pb, gp, spec, terms


def _inputs(pb, P, H, seed):
    rng = np.random.RandomState(seed)
    return pb["m0"][None] + np.sqrt(0.1) * rng.randn(P, 10), rng.randn(P, H, 10)


def main():
    engine.device()
    out = {"card": card(), "H": H, "rounds": ROUNDS}
    pb, gp, spec, terms = _problem()
    for P in PS:
        x0, eps = _inputs(pb, P, H, P)
        fwd = engine.ParticlePlan(gp, spec, terms, P, H)
        path = engine.ParticlePlan(gp, spec, terms, P, H, grad=True)
        score = engine.ParticlePlan(gp, spec, terms, P, H, grad=True, estimator="score")
        for p in (fwd, path, score):
            p.set_inputs(x0, eps)
        reps = max(2, min(20, int(2e5 // P)))
        runs = {"forward_ms": fwd.launch, "forward_pathwise_ms": path.launch_grad, "forward_score_ms": score.launch_grad}
        for fn in runs.values():                                # warm-up of every shape
            fn()
        torch.cuda.synchronize()
        times = {k: [] for k in runs}
        for _ in range(ROUNDS):                                 # alternated
            for k, fn in runs.items():
                times[k].append(timeit(fn, reps))
        res = {k: float(np.median(v)) for k, v in times.items()}
        res["score_over_pathwise"] = res["forward_score_ms"] / res["forward_pathwise_ms"]
        res["spread"] = {k: [float(min(v)), float(max(v))] for k, v in times.items()}
        out["P%d" % P] = res
        del fwd, path, score
    P = 1024
    for h in (10, 40):
        plans = {e: engine.ParticlePlan(gp, spec, terms, P, h, grad=True, estimator=e) for e in ("pathwise", "score")}
        draws = {e: [] for e in plans}
        for s in range(SEEDS):
            x0, eps = _inputs(pb, P, h, 1000 + s)
            for e, plan in plans.items():
                plan.set_inputs(x0, eps)
                g = plan.launch_grad()
                draws[e].append(np.concatenate([g[k].cpu().numpy().ravel() for k in ("X", "Y", "ell")]))
        res = {}
        for e, d in draws.items():
            a = np.stack(d)
            res[e] = {"summed_variance": float(a.var(0, ddof=1).sum()), "mean_norm": float(np.linalg.norm(a.mean(0)))}
        res["score_over_pathwise_variance"] = res["score"]["summed_variance"] / res["pathwise"]["summed_variance"]
        out["variance_P%d_H%d" % (P, h)] = res
    out["card_after"] = card()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
