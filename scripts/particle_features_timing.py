"""Cost of the random-feature function sampler (pilco_particles_features_*, DESIGN.md section 30) beside the exact
consistent sampler (section 14) and the step-wise sampler (section 11).

E = 10 state dimensions, U = 2 (D = 12), a linear policy, n in {300, 2000} dynamics points, H in {40, 200}, P in
{1024, 16384}; the feature sampler at F in {256, 1024}.  For each configuration and sampler: the forward rollout (R =
1) and the forward + pathwise gradient at R = 8 restarts, each the median of ``--reps`` CUDA-event timings after one
warm-up call, the samplers alternated within the configuration; the draw call is timed on its own, its normals
already on the device (the window holds the draw's allocations, kernels and products, not a host copy).  Workspace bytes
are reported; a configuration whose workspace exceeds ``--max-gb`` is reported as not fitting, and one whose warm-up
took longer than ``--max-s`` seconds is reported as not measured.  Prints the card's name and power limit, then one
JSON line per configuration.
``--n``, ``--H``, ``--P`` restrict the grid.
Usage: python scripts/particle_features_timing.py [--reps 3] [--max-gb 40] [--max-s 4] [--n 300 2000] [--H 40 200]
       [--P 1024 16384]"""
import argparse
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
from obs_noise_timing import card                               # noqa: E402

E, U, R = 10, 2, 8


def problem(n, seed=0):
    D = E + U
    rng = np.random.RandomState(seed)
    X = rng.rand(n, D)
    Y = 0.05 * (np.sin(X) @ rng.rand(D, E))
    dyn = engine.gp_factorize(X, Y, 1.0 + rng.rand(E, D), 0.05 * (1.0 + rng.rand(E)), 1e-3 * np.ones(E))
    W, b = 0.1 * rng.randn(R, U, E), 0.1 * rng.randn(R, U)
    lin = dict(kind=_lib.POLICY_LINEAR, Ds=E, U=U, squash=True, max_action=np.ones(U), W=W, b=b)
    terms = [dict(kind=_lib.REWARD_EXP, coef=1.0, W=np.eye(E), t=np.zeros(E))]
    return dyn, dict(lin, W=W[0], b=b[0]), lin, terms, X[0, :E]


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
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--max-gb", type=float, default=40.0)
    ap.add_argument("--max-s", type=float, default=4.0)
    ap.add_argument("--n", type=int, nargs="+", default=[300, 2000])
    ap.add_argument("--H", type=int, nargs="+", default=[40, 200])
    ap.add_argument("--P", type=int, nargs="+", default=[1024, 16384])
    args = ap.parse_args()
    cap = int(args.max_gb * 2 ** 30)
    print(json.dumps({"card": card(), "E": E, "D": E + U, "R_grad": R, "policy": "linear"}))
    for n in args.n:
        dyn, one, batch, terms, m0 = problem(n)
        for H in args.H:
            for P in args.P:
                rng = np.random.RandomState(P + H)
                x0, eps = m0[None] + 0.1 * rng.randn(P, E), rng.randn(P, H, E)
                row = {"n": n, "H": H, "P": P}
                arms = [("stepwise", None, False), ("consistent", None, True)] + \
                    [("features%d" % F, F, True) for F in (256, 1024)]
                for name, F, cons in arms:
                    draws = None
                    if F is not None:
                        rngf = np.random.RandomState(F)
                        z, w, ey = (engine.dev(rngf.randn(*shape)) for shape in ((E, F, E + U), (P, E, 2 * F),
                                                                                 (P, E, n)))
                        row[name + "_draw_ms"] = timed(lambda: engine.feature_draws(dyn, P, F, z, w, ey), args.reps,
                                                       args.max_s)
                        draws = engine.feature_draws(dyn, P, F, z, w, ey)
                    for what, grad in (("fwd", False), ("grad", True)):
                        key = "%s_%s" % (name, what)
                        try:
                            if grad and cons:
                                plan = engine.ConsistentGradPlan(dyn, batch, terms, P, H, R=R, max_ws_bytes=cap,
                                                                 num_features=F)
                            else:
                                if cons and F is None and engine.consistent_workspace_bytes(dyn, E, U, P, H) > cap:
                                    raise ValueError("workspace over the cap")
                                plan = engine.ParticlePlan(dyn, batch if grad else one, terms, P, H, grad=grad,
                                                           R=R if grad else 1, consistent=cons, num_features=F)
                            row[key + "_ws_bytes"] = int(plan.gws.numel() * 8 if grad else plan.ws.numel() * 8)
                            plan.set_inputs(x0, None if F else eps, features=draws)
                            ms = timed(plan.launch_grad if grad else plan.launch, args.reps, args.max_s)
                            row[key + "_ms"] = ms if ms is not None else "not measured (over %g s)" % args.max_s
                        except (ValueError, torch.cuda.OutOfMemoryError) as exc:
                            row[key + "_ms"] = "does not fit (%s)" % str(exc)[:60]
                        plan = None
                        torch.cuda.empty_cache()
                    draws = None
                print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
