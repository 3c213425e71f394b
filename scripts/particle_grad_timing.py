"""Timing of pilco_particles_rollout_grad at the metric shape (dynamics n = 300, D = 12, E = 10; RBF policy, bf = 50;
exponential reward), H = 40, P = 1024, 16384, 131072 particles: ms of the forward alone (pilco_particles_rollout) and
of forward + pathwise gradient from CUDA events after a warm-up, pilco_gp_predict_vjp and pilco_gp_predict at T = P
timed alone in the same process, and the card's name and power limit read in the same run.
    python scripts/particle_grad_timing.py  -> one JSON line"""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "scripts"))
from pilco_b200 import _lib, engine             # noqa: E402
from predict_timing import card, timeit          # noqa: E402
from util import make_rollout_problem            # noqa: E402

PS = (1024, 16384, 131072)
H = 40


def main():
    engine.device()
    out = {"card": card(), "H": H}
    pb = make_rollout_problem(300, 10, 2, 50, 1, seed=0)
    gp = engine.gp_factorize(pb["X"], pb["Y"], pb["ell"], pb["sf2"], pb["sn2"])
    pgp = engine.gp_factorize(pb["Xc"][0], pb["Yc"][0], pb["lc"][0], np.ones(2), 1e-4 * np.ones(2), need_iK=False, mode=1)
    spec = dict(kind=_lib.POLICY_RBF, Ds=10, U=2, squash=True, max_action=pb["maxa"], gp=pgp)
    terms = [dict(kind=_lib.REWARD_EXP, coef=1.0, W=pb["W"], t=pb["t"])]
    for P in PS:
        rng = np.random.RandomState(P)
        plan = engine.ParticlePlan(gp, spec, terms, P, H, grad=True)
        plan.set_inputs(pb["m0"][None] + np.sqrt(0.1) * rng.randn(P, 10), rng.randn(P, H, 10))
        reps = max(2, min(20, int(2e5 // P)))
        t_fwd = timeit(plan.launch, reps)
        t_grad = timeit(plan.launch_grad, reps)
        Xs = engine.dev(np.hstack([plan.traj[:, H // 2].cpu().numpy(), plan.act_buf[:, H // 2].cpu().numpy()]))
        gm, gv = engine.dev(rng.randn(P, 10)), engine.dev(rng.randn(P, 10))
        t_pred = timeit(lambda: engine.gp_predict(gp, Xs), max(3, reps))
        t_vjp = timeit(lambda: engine.gp_predict_vjp(gp, Xs, gm, gv), max(3, reps))
        out["P%d" % P] = {"forward_ms": t_fwd, "forward_grad_ms": t_grad, "grad_over_forward": t_grad / t_fwd,
                          "predict_ms": t_pred, "vjp_ms": t_vjp, "vjp_over_predict": t_vjp / t_pred}
    out["card_after"] = card()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
