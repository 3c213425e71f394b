"""Incremental set_data against a refactorisation: the time of ``engine.gp_append`` (k rows appended to a factorised
n0-row model) and of ``engine.gp_factorize`` of the same n0 + k rows, both with the data already on the device (what
``MGPR.device_gp`` runs), at (n0, k) = (300, 40), (1000, 100), (2000, 100); dynamics-GP shape D = 6, E = 5, rows from
PILCO-like episodes at sn2 = 1e-4.  Prints one line per size and the card it ran on.
    python scripts/append_timing.py"""
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from pilco_b200 import engine                    # noqa: E402
from fact_cases import episodes                  # noqa: E402


def timeit(fn, reps=20):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                      text=True).stdout.strip()
print("card: %s" % card)
D, E = 6, 5
for n0, k in ((300, 40), (1000, 100), (2000, 100)):
    rng = np.random.RandomState(n0)
    X = episodes(n0 + k, D, rng)
    Y = 0.1 * np.sin(3.0 * X).dot(rng.rand(D, E))
    ell, sf2, sn2 = 1.0 + 0.1 * rng.rand(E, D), np.ones(E), 1e-4 * np.ones(E)
    Xd, Yd = engine.dev(X), engine.dev(Y)
    gp0 = engine.gp_factorize(Xd[:n0], Yd[:n0], ell, sf2, sn2)
    t_app = timeit(lambda: engine.gp_append(gp0, Xd, Yd))
    t_fac = timeit(lambda: engine.gp_factorize(Xd, Yd, ell, sf2, sn2))
    a, f = engine.gp_append(gp0, Xd, Yd), engine.gp_factorize(Xd, Yd, ell, sf2, sn2)
    torch.cuda.synchronize()
    diff = float((a.beta - f.beta).abs().max() / f.beta.abs().max())
    print("n0=%d k=%d: gp_append %.3f ms, gp_factorize %.3f ms, ratio %.2f (beta max rel diff %.1e)"
          % (n0, k, t_app, t_fac, t_fac / t_app, diff))
