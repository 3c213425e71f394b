"""Cost of one Adam iteration on fresh particles (policy_opt.StochasticEvaluator, DESIGN.md section 32) beside one
L-BFGS-B evaluation on fixed particles (policy_opt.ParticleEvaluator) at the same shapes, and the gap between the
in-sample and the out-of-sample value after each optimiser.

E = 10 state dimensions, U = 2 (D = 12), n = 300 dynamics points, H = 40, P = 1024 particles, R = 8 restarts; linear,
RBF (50 centres) and tanh MLP (2 x 64) policies; the step-wise sampler and the random-feature sampler at F = 256.  Per
configuration: the replayed graph of one iteration (draws, gradient, Adam step) and the draws alone, each the median of
``--reps`` CUDA-event timings on the group's stream, and one L-BFGS-B evaluation (its replayed graph with the host
copies and the synchronisation), the median of ``--reps`` host-clock timings.  Then, per policy with the step-wise
sampler and one restart: ``optimize_policy_sampled`` with each optimiser at the same ``--gap-iters`` iterations and P
particles, its returned value (L-BFGS-B: in-sample; Adam: held-out) and the last Adam step's in-sample value, beside
the out-of-sample mean return of 2^14 particles of another seed.  Prints the card's name and power limit, then one JSON
line per row.
Usage: python scripts/particle_sgd_timing.py [--reps 10] [--gap-iters 50] [--P 1024] [--H 40]"""
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
from pilco_b200 import controllers, engine, policy_opt, rewards      # noqa: E402
from pilco_b200.models.pilco import PILCO, _sqrt_factor             # noqa: E402
from obs_noise_timing import card                                   # noqa: E402

E, U, N, R = 10, 2, 300, 8


def make(policy, H, seed=0):
    np.random.seed(seed)
    rng = np.random.RandomState(seed)
    X = rng.rand(N, E + U)
    Y = 0.05 * (np.sin(X) @ rng.rand(E + U, E))
    c = {"linear": lambda: controllers.LinearController(E, U, max_action=1.0),
         "rbf50": lambda: controllers.RbfController(E, U, 50, max_action=1.0),
         "mlp2x64": lambda: controllers.MlpController(E, U, hidden=(64, 64), max_action=1.0)}[policy]()
    pilco = PILCO((X, Y), controller=c, horizon=H, reward=rewards.ExponentialReward(E, t=0.3 * np.ones(E)),
                  m_init=X[0:1, :E], S_init=0.01 * np.eye(E))
    for m in pilco.mgpr.models:
        m.likelihood.variance.assign(1e-3)
    return pilco


def event_ms(fn, stream, reps):
    with torch.cuda.stream(stream):
        fn()
        torch.cuda.synchronize()
        out = []
        for _ in range(reps):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            fn()
            b.record()
            torch.cuda.synchronize()
            out.append(a.elapsed_time(b))
    return round(float(np.median(out)), 3)


def timing_row(policy, F, P, H, reps):
    pilco = make(policy, H)
    flats = policy_opt.initial_flats(pilco.controller, R)
    m0 = np.asarray(pilco.m_init, dtype=np.float64).reshape(-1)
    kw = dict(consistent=F is not None, num_features=F)
    ev = policy_opt.StochasticEvaluator(pilco, R, flats, P, 7, m0, _sqrt_factor(pilco.S_init), lr=1e-3, **kw)
    ev.capture()
    row = {"policy": policy, "sampler": "features%d" % F if F else "stepwise", "P": P, "H": H, "R": R,
           "n_theta": int(flats.shape[1])}
    row["adam_iteration_ms"] = event_ms(ev.replay, ev.stream, reps)
    row["draws_ms"] = event_ms(lambda: ev._draw(ev.adam.iter, 0), ev.stream, reps)
    row["draws_share"] = round(row["draws_ms"] / row["adam_iteration_ms"], 3)
    p = ev.plan
    x0 = p.x0.clone()
    eps = None if F else p.eps_buf.clone()
    pe = policy_opt.ParticleEvaluator(pilco, R, x0, eps, features=ev.draws, **{"consistent": F is not None})
    pe.prepare(flats)
    pe.cache = None
    out = []
    for _ in range(reps):
        t0 = time.perf_counter()
        pe(flats)
        out.append(1e3 * (time.perf_counter() - t0))
    row["lbfgsb_evaluation_ms"] = round(float(np.median(out)), 3)
    return row


def gap_row(policy, P, H, iters):
    row = {"policy": policy, "sampler": "stepwise", "P": P, "H": H, "iters": iters, "restarts": 1}
    for opt in ("lbfgsb", "adam"):
        pilco = make(policy, H)
        kw = dict(optimizer="adam", learning_rate=1e-2) if opt == "adam" else {}
        v = pilco.optimize_policy_sampled(maxiter=iters, restarts=1, num_samples=P, seed=1, **kw)
        out = pilco.sample_policy_gradient(pilco.m_init, pilco.S_init, H, num_samples=1 << 14, seed=999)
        se = float(np.std(np.asarray(out.returns), ddof=1) / np.sqrt(1 << 14))
        row[opt] = {"returned_value": round(float(v), 5), "out_of_sample": round(float(out.value), 5),
                    "out_of_sample_se": round(se, 5)}
        if opt == "adam":
            row[opt]["last_in_sample"] = round(float(np.asarray(pilco.adam_trace.value)[-1, 0]), 5)
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--gap-iters", type=int, default=50)
    ap.add_argument("--P", type=int, default=1024)
    ap.add_argument("--H", type=int, default=40)
    args = ap.parse_args()
    print(json.dumps({"card": card(), "E": E, "D": E + U, "n": N, "R": R}), flush=True)
    for policy in ("linear", "rbf50", "mlp2x64"):
        for F in (None, 256):
            print(json.dumps(timing_row(policy, F, args.P, args.H, args.reps)), flush=True)
            torch.cuda.empty_cache()
    for policy in ("linear", "rbf50", "mlp2x64"):
        print(json.dumps(gap_row(policy, args.P, args.H, args.gap_iters)), flush=True)


if __name__ == "__main__":
    main()
