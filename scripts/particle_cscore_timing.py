"""Timing and variance of pilco_particles_consistent_score_grad_rollout at the metric-like shape (dynamics n = 300,
D = 12, E = 10; RBF policy, bf = 50; one exponential reward), H = 40, P = 1024 and 4096: ms of the consistent forward
alone (pilco_particles_rollout_consistent), of forward + consistent pathwise gradient and of forward + consistent score
gradient, from CUDA events after a warm-up, the three alternated in one process (median of the rounds).  Then, over 16
seeds at P = 1024, each estimator's summed per-component variance of the gradient at H = 10 and H = 40, and the card's
name and power limit read in the same run.
    python scripts/particle_cscore_timing.py  -> one JSON line"""
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "scripts"))
from pilco_b200 import engine                                  # noqa: E402
from particle_score_timing import _inputs, _problem            # noqa: E402
from predict_timing import card, timeit                        # noqa: E402

PS = (1024, 4096)
H = 40
ROUNDS = 5
SEEDS = 16


def main():
    engine.device()
    out = {"card": card(), "H": H, "rounds": ROUNDS}
    pb, gp, spec, terms = _problem()
    for P in PS:
        x0, eps = _inputs(pb, P, H, P)
        fwd = engine.ParticlePlan(gp, spec, terms, P, H, consistent=True)
        path = engine.ConsistentGradPlan(gp, spec, terms, P, H)
        score = engine.ConsistentGradPlan(gp, spec, terms, P, H, estimator="score")
        for p in (fwd, path, score):
            p.set_inputs(x0, eps)
        reps = max(2, min(10, int(2e4 // P)))
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
        torch.cuda.empty_cache()
    P = 1024
    for h in (10, 40):
        plans = {e: engine.ConsistentGradPlan(gp, spec, terms, P, h, estimator=e) for e in ("pathwise", "score")}
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
        del plans
        torch.cuda.empty_cache()
    out["card_after"] = card()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
