"""Timing of pilco_particles_rollout_consistent against pilco_particles_rollout at the metric shape (dynamics n = 300,
D = 12, E = 10; RBF policy, bf = 50; exponential reward), H = 40, P = 1024, 4096, 16384 particles, in one process: ms
per rollout from CUDA events after a warm-up, the ratio, the workspace, the bytes of K* history the conditioning
kernels read (P E np 8 H(H-1)/2) and the rate they imply, and the card's name and power limit read in the same run.
    python scripts/particle_consistent_timing.py  -> one JSON line"""
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

PS = (1024, 4096, 16384)
H = 40


def main():
    engine.device()
    out = {"card": card(), "H": H}
    pb = make_rollout_problem(300, 10, 2, 50, 1, seed=0)
    gp = engine.gp_factorize(pb["X"], pb["Y"], pb["ell"], pb["sf2"], pb["sn2"])
    pgp = engine.gp_factorize(pb["Xc"][0], pb["Yc"][0], pb["lc"][0], np.ones(2), 1e-4 * np.ones(2), need_iK=False, mode=1)
    spec = dict(kind=_lib.POLICY_RBF, Ds=10, U=2, squash=True, max_action=pb["maxa"], gp=pgp)
    terms = [dict(kind=_lib.REWARD_EXP, coef=1.0, W=pb["W"], t=pb["t"])]
    np_ = engine.pad_n(gp.n)
    for P in PS:
        rng = np.random.RandomState(P)
        x0, eps = pb["m0"][None] + np.sqrt(0.1) * rng.randn(P, 10), rng.randn(P, H, 10)
        marg = engine.ParticlePlan(gp, spec, terms, P, H)
        marg.set_inputs(x0, eps)
        reps = max(2, min(10, int(4e4 // P)))
        t_marg = timeit(marg.launch, reps)
        del marg
        cons = engine.ParticlePlan(gp, spec, terms, P, H, consistent=True)
        cons.set_inputs(x0, eps)
        t_cons = timeit(cons.launch, reps)
        hist = P * 10 * np_ * 8 * H * (H - 1) // 2
        out["P%d" % P] = {"marginal_ms": t_marg, "consistent_ms": t_cons, "ratio": t_cons / t_marg,
                          "workspace_GB": cons.ws.numel() * 8 / 1e9, "history_read_GB": hist / 1e9,
                          "history_read_TB_per_s_over_extra_time": hist / ((t_cons - t_marg) * 1e-3) / 1e12}
        del cons
        torch.cuda.empty_cache()
    out["card_after"] = card()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
