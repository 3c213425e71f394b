"""Timing of pilco_gp_predict (diagonal path, fused DMMA kernel) at T = 32 .. 131072 test points for the exact GP at
(n, D, E) = (300, 12, 10) and (2000, 12, 10) and for FITC over M = 200 inducing points (N = 2000): call time from CUDA
events after a warm-up, the DMMA rate 2 T np^2 ne / t (np = n padded to 64: the MMA work the kernel issues) and its
fraction of DMMA.16x8x8 measured in the same process (pilco_microbench_fp64 which = 5), a same-device torch fp64
baseline (materialised K*, (K* @ iK) * K* row sums) with its largest difference from the kernel, and the card's name and
power limit read in the same run.   python scripts/predict_timing.py  -> one JSON line"""
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from pilco_b200 import _lib, engine             # noqa: E402
from util import make_gp_problem                 # noqa: E402

TS = (32, 1024, 16384, 131072)


def timeit(fn, reps):
    fn(); torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def torch_baseline(gp, Xs):
    n = gp.n
    means, vars_ = [], []
    for e in range(gp.E):
        il = 1.0 / gp.ell[e]
        K = gp.sf2[e] * torch.exp(-0.5 * torch.cdist(Xs * il, gp.X * il) ** 2)
        means.append(K @ gp.beta[e])
        vars_.append(gp.sf2[e] - ((K @ gp.iK[e, :n, :n]) * K).sum(1))
    return torch.stack(means, 1), torch.stack(vars_, 1)


def card():
    q = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=name,power.limit,clocks.max.sm",
                        "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
    return q or torch.cuda.get_device_name()


def main():
    engine.device()
    d = torch.cuda.current_device()
    out = {"card": card()}
    sink = torch.zeros(8, dtype=torch.float64, device="cuda")
    ms = C.c_float()
    blocks, iters = torch.cuda.get_device_properties(d).multi_processor_count * 4, 5000
    _lib.check(_lib.lib.pilco_microbench_fp64(5, iters, blocks, engine.ptr(sink), C.byref(ms), engine.stream_ptr()))
    peak = blocks * 8 * iters * 8.0 * 2048 / (ms.value * 1e-3) / 1e12        # 2048 flop per warp-level DMMA.16x8x8
    out["dmma_16x8x8_tflops"] = peak
    E, D = 10, 12
    models = {}
    for n in (300, 2000):
        X, Y, ell, sf2, sn2 = make_gp_problem(n, D, E, seed=n)
        models["exact_n%d" % n] = engine.gp_factorize(X, Y, ell, sf2, sn2)
    X, Y, ell, sf2, sn2 = make_gp_problem(2000, D, E, seed=7)
    models["fitc_N2000_M200"] = engine.fitc_factorize(X, np.random.RandomState(1).rand(200, D), Y, ell, sf2, sn2)
    for name, gp in models.items():
        np_ = engine.pad_n(gp.n)
        for T in TS:
            Xs = engine.dev(np.random.RandomState(T).rand(T, D))
            reps = max(3, min(200, int(2e9 // (T * np_ * np_ * E) + 1)))
            t_k = timeit(lambda: engine.gp_predict(gp, Xs), reps)
            t_b = timeit(lambda: torch_baseline(gp, Xs), max(2, reps // 4))
            mk, vk = engine.gp_predict(gp, Xs)
            mb, vb = torch_baseline(gp, Xs)
            rate = 2.0 * T * np_ * np_ * E / (t_k * 1e-3) / 1e12
            out["%s_T%d" % (name, T)] = {
                "ms": t_k, "dmma_tflops": rate, "frac_of_dmma_16x8x8": rate / peak, "torch_fp64_ms": t_b,
                "max_mean_diff_rel": float((mk - mb).abs().max() / mb.abs().max()),
                "max_var_diff_over_sf2": float(((vk - vb).abs() / gp.sf2).max())}
    out["card_after"] = card()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
