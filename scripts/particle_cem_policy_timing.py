"""Cost of one iteration of the cross-entropy method over a stationary policy's parameters on the device
(policy_opt.CemPolicySearch: engine.ParticleBatchPlan and pilco_cem_update, DESIGN.md section 33) beside one
evaluation of the default L-BFGS-B optimizer's objective.

n = 300 dynamics points, E = 10 state dimensions, U = 2 (D = 12), H = 40, the step-wise sampler; a linear policy, an
RBF policy of 50 centres and a tanh MLP of 2 x 64 units; K in {64, 400} candidates (elites K / 10), P in {100, 1000}
particles.  For each configuration, each the median of ``--reps`` CUDA-event timings after one warm-up call: the
batched forward of the K candidates (``ParticleBatchPlan.launch``), the unpacking of the K flat rows into the policy
buffers (with the batched refactorisation for RBF), the update (pilco_cem_update), one whole iteration (the three, as
the search enqueues them); and on the same particles one evaluation of the L-BFGS-B objective (``ParticleEvaluator``
at R = 1: unpacking, forward, reverse sweep and gradient packing, as a replayed graph with its host round trip).  A
configuration whose warm-up took longer than ``--max-s`` seconds is reported as not measured.  Prints the card's
name, power limit and max SM clock, then one JSON line per configuration.
Usage: python scripts/particle_cem_policy_timing.py [--reps 5] [--max-s 30] [--K 64 400] [--P 100 1000]"""
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
from pilco_b200 import controllers, engine, policy_opt, rewards      # noqa: E402
from pilco_b200._lib import check, lib                              # noqa: E402
from pilco_b200.models.pilco import PILCO                           # noqa: E402
from obs_noise_timing import card                                   # noqa: E402

n, E, U, H = 300, 10, 2, 40


def problem(kind, seed=0):
    np.random.seed(seed)
    rng = np.random.RandomState(seed)
    X = rng.rand(n, E + U)
    Y = 0.05 * (np.sin(X) @ rng.rand(E + U, E))
    c = {"linear": lambda: controllers.LinearController(E, U),
         "rbf": lambda: controllers.RbfController(E, U, 50),
         "mlp": lambda: controllers.MlpController(E, U, (64, 64))}[kind]()
    p = PILCO((X, Y), controller=c, horizon=H, reward=rewards.ExponentialReward(E, t=np.zeros(E)),
              m_init=X[0:1, :E], S_init=0.01 * np.eye(E))
    for m in p.mgpr.models:
        m.likelihood.variance.assign(1e-3)
    return p


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
    ap.add_argument("--max-s", type=float, default=30.0)
    ap.add_argument("--K", type=int, nargs="+", default=[64, 400])
    ap.add_argument("--P", type=int, nargs="+", default=[100, 1000])
    ap.add_argument("--policy", nargs="+", default=["linear", "rbf", "mlp"])
    args = ap.parse_args()
    print(json.dumps({"card": card(), "n": n, "E": E, "U": U, "H": H, "sampler": "stepwise"}), flush=True)
    nm = lambda ms: ms if ms is not None else "not measured (over %g s)" % args.max_s
    for kind in args.policy:
        p = problem(kind)
        n_theta = p.controller.get_flat().size
        for P in args.P:
            x0, eps = p._particle_inputs(p.m_init, p.S_init, H, P, 1, "timing")
            ev = policy_opt.ParticleEvaluator(p, 1, x0, eps)
            flats = p.controller.get_flat()[None]
            ev.prepare(flats)
            ev.cache = None
            lbfgsb_ms = nm(timed(lambda: ev(flats), args.reps, args.max_s))
            ev = None
            for K in args.K:
                row = {"policy": kind, "n_theta": n_theta, "K": K, "P": P, "lbfgsb_eval_ms": lbfgsb_ms}
                s = policy_opt.CemPolicySearch(p, K, K // 10, 1, P, seed=K, std0=0.1)
                s.set_inputs(x0, eps)
                s.launch()
                row["chunk"] = s.plan.chunk
                row["forward_ms"] = nm(timed(s.plan.launch, args.reps, args.max_s))
                row["unpack_ms"] = nm(timed(lambda: s._unpack(s.cand, s.plan, s.gp), args.reps, args.max_s))
                update = lambda: check(lib.pilco_cem_update(C.byref(s.updates[0]), s.uws.data_ptr(), s.uws_bytes,
                                                            engine.stream_ptr()), "cem_update")
                row["update_ms"] = nm(timed(update, args.reps, args.max_s))
                row["iteration_ms"] = nm(timed(lambda: (s.evaluate(), update()), args.reps, args.max_s))
                print(json.dumps(row), flush=True)
                s = None
                torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
