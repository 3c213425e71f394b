"""Cost of planning with the cross-entropy method on the device (engine.CemPlan: pilco_particles_scheduled_*batch_rollout
and pilco_cem_update, DESIGN.md section 31) beside one evaluation of the gradient planner.

n = 300 dynamics points, E = 10 state dimensions, U = 2 (D = 12), an open-loop schedule (W = 0), 5 CEM iterations with
elites = K / 10; K in {256, 1024} candidates, P in {16, 32} particles, H in {25, 40}, the step-wise and the consistent
sampler.  For each configuration: the whole plan (``launch()``: a draw, then 5 x (batched forward, update)), eagerly
and as one replayed CUDA graph, one
batched forward of the K candidates and one update alone, each the median of ``--reps`` CUDA-event timings after one
warm-up call; and, on the same particles, one evaluation of the L-BFGS-B planner's objective (forward + pathwise
gradient of one schedule, ParticlePlan / ConsistentGradPlan with R = 1).  A configuration whose warm-up took longer
than ``--max-s`` seconds is reported as not measured.  Prints the card's name and power limit, then one JSON line per
configuration.
Usage: python scripts/particle_cem_timing.py [--reps 5] [--max-s 20] [--K 256 1024] [--P 16 32] [--H 25 40]"""
import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from pilco_b200 import engine, _lib                              # noqa: E402
from pilco_b200._lib import check, lib                          # noqa: E402
from obs_noise_timing import card                               # noqa: E402

n, E, U, ITERS = 300, 10, 2, 5


def problem(H, seed=0):
    D = E + U
    rng = np.random.RandomState(seed)
    X = rng.rand(n, D)
    Y = 0.05 * (np.sin(X) @ rng.rand(D, E))
    dyn = engine.gp_factorize(X, Y, 1.0 + rng.rand(E, D), 0.05 * (1.0 + rng.rand(E)), 1e-3 * np.ones(E))
    spec = dict(kind=_lib.POLICY_LINEAR, Ds=E, U=U, squash=True, max_action=np.ones(U), W=np.zeros((H, U, E)),
                b=0.1 * rng.randn(H, U), schedule=True)
    terms = [dict(kind=_lib.REWARD_EXP, coef=1.0, W=np.eye(E), t=np.zeros(E))]
    return dyn, spec, terms, X[0, :E]


def timed(fn, reps, max_s):
    """median ms of reps calls after one warm-up, or None when the warm-up took longer than max_s"""
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    if time.perf_counter() - t0 > max_s:
        return None
    out = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        out.append(a.elapsed_time(b))
    return round(float(np.median(out)), 3)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--max-s", type=float, default=20.0)
    ap.add_argument("--K", type=int, nargs="+", default=[256, 1024])
    ap.add_argument("--P", type=int, nargs="+", default=[16, 32])
    ap.add_argument("--H", type=int, nargs="+", default=[25, 40])
    args = ap.parse_args()
    print(json.dumps({"card": card(), "n": n, "E": E, "U": U, "iters": ITERS, "policy": "open-loop schedule"}))
    nm = lambda ms: ms if ms is not None else "not measured (over %g s)" % args.max_s
    for H in args.H:
        dyn, spec, terms, m0 = problem(H)
        for P in args.P:
            rng = np.random.RandomState(P + H)
            x0, eps = m0[None] + 0.1 * rng.randn(P, E), rng.randn(P, H, E)
            for consistent in (False, True):
                sampler = "consistent" if consistent else "stepwise"
                if consistent:
                    grad = engine.ConsistentGradPlan(dyn, spec, terms, P, H, schedule=True)
                else:
                    grad = engine.ParticlePlan(dyn, spec, terms, P, H, grad=True, schedule=True)
                grad.set_inputs(x0, eps)
                lbfgsb_ms = nm(timed(grad.launch_grad, args.reps, args.max_s))
                grad = None
                for K in args.K:
                    row = {"sampler": sampler, "K": K, "P": P, "H": H, "lbfgsb_eval_ms": lbfgsb_ms}
                    plan = engine.CemPlan(dyn, spec, terms, P, H, K, K // 10, ITERS, consistent=consistent)
                    plan.set_inputs(x0, eps, np.random.RandomState(K).randn(ITERS, K, H, U))
                    row["chunk"] = plan.chunk
                    row["plan_ms"] = nm(timed(plan.launch, args.reps, args.max_s))
                    if row["plan_ms"] != nm(None):
                        plan.capture()
                        row["plan_graph_ms"] = nm(timed(plan.replay, args.reps, args.max_s))
                    row["forward_ms"] = nm(timed(plan.rollout, args.reps, args.max_s))
                    update = lambda: check(lib.pilco_cem_update(C.byref(plan.updates[0]), plan.uws.data_ptr(),
                                                                plan.uws_bytes, engine.stream_ptr()), "cem_update")
                    row["update_ms"] = nm(timed(update, args.reps, args.max_s))
                    print(json.dumps(row), flush=True)
                    plan = None
                    torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
