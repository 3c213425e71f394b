"""Timing of pilco_gp_predict_samples (posterior function samples, full covariance) at T = 1024, 4096, 16384 points and
S = 1, 256 samples, one output, for the exact GP at (n, D) = (300, 12) and (2000, 12) and for FITC over M = 200
inducing points (N = 2000): the call time from CUDA events (median over alternated rounds against the baseline), the
same-device torch baseline (pilco_gp_predict's covariance, then torch.linalg.cholesky and a matmul) with its largest
difference from the call (relative to the samples and to their L eps part), the full_cov=False call, and the split of one call's kernel time into covariance, Cholesky
and sample GEMM (torch.profiler, kernels attributed by launch order), with the card's name and power limit read in
the same run.   python scripts/predict_samples_timing.py [--quick]  -> one JSON line"""
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from pilco_b200 import engine                    # noqa: E402
from util import make_gp_problem                 # noqa: E402

QUICK = "--quick" in sys.argv
TS = (1024,) if QUICK else (1024, 4096, 16384)
SS = (1, 256)
ROUNDS = 3 if QUICK else 5


def card():
    q = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=name,power.limit,clocks.max.sm",
                        "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
    return q or torch.cuda.get_device_name()


def event_ms(fn, reps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def baseline(gp, Xs, eps):
    mean, cov = engine.gp_predict(gp, Xs, ne=1, full_cov=True)
    L = torch.linalg.cholesky(cov[0] + 1e-6 * torch.eye(cov.shape[1], dtype=cov.dtype, device=cov.device))
    return mean[:, 0][None] + eps[:, :, 0] @ L.T


def split(fn):
    """kernel milliseconds of one call: (covariance, Cholesky, sample GEMM), by launch order: the Cholesky starts at the
    jitter kernel, the sample GEMM at the first transpose.  NaN when the profiler returned no kernel list (3 tries)."""
    from torch.profiler import ProfilerActivity, profile
    for _ in range(3):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        ks = sorted((e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA),
                    key=lambda e: e.time_range.start)
        names = [e.name for e in ks]
        a = next((i for i, nm in enumerate(names) if "add_diag_const_kernel" in nm), None)
        b = next((i for i, nm in enumerate(names) if "gp_sample_transpose_kernel" in nm), None)
        if a is not None and b is not None:
            us = [e.time_range.elapsed_us() for e in ks]
            return sum(us[:a]) / 1e3, sum(us[a:b]) / 1e3, sum(us[b:]) / 1e3
    return float("nan"), float("nan"), float("nan")


def main():
    engine.device()
    out = {"card": card(), "rounds": ROUNDS}
    D = 12
    models = {}
    for n in (300, 2000):
        X, Y, ell, sf2, sn2 = make_gp_problem(n, D, 1, seed=n)
        models["exact_n%d" % n] = engine.gp_factorize(X, Y, ell, sf2, sn2)
    X, Y, ell, sf2, sn2 = make_gp_problem(2000, D, 1, seed=7)
    models["fitc_N2000_M200"] = engine.fitc_factorize(X, np.random.RandomState(1).rand(200, D), Y, ell, sf2, sn2)
    for name, gp in models.items():
        for T in TS:
            Xs = engine.dev(np.random.RandomState(T).rand(T, D))
            for S in SS:
                eps = torch.randn((S, T, 1), dtype=torch.float64, device="cuda",
                                  generator=torch.Generator(device="cuda").manual_seed(S))
                ours = lambda: engine.gp_predict_samples(gp, Xs, eps)
                diag = lambda: engine.gp_predict_samples(gp, Xs, eps, full_cov=False)
                base = lambda: baseline(gp, Xs, eps)
                reps = 1 if T >= 16384 else (3 if T >= 4096 else 10)
                for f in (ours, diag, base):                 # warm-up of every shape
                    f()
                torch.cuda.synchronize()
                t_o, t_d, t_b = [], [], []
                for _ in range(ROUNDS):
                    t_o.append(event_ms(ours, reps))
                    t_b.append(event_ms(base, reps))
                    t_d.append(event_ms(diag, reps))
                so, info = ours()
                sb = base()
                mean, _ = engine.gp_predict(gp, Xs, ne=1)
                dev_b = sb - mean[:, 0][None]                  # L eps of the baseline: the part the two compute differently
                splits = np.array([split(ours) for _ in range(3)])
                cov_ms, chol_ms, gemm_ms = np.median(splits, 0)
                out["%s_T%d_S%d" % (name, T, S)] = {
                    "ms": float(np.median(t_o)), "ms_all": [round(t, 3) for t in t_o],
                    "torch_baseline_ms": float(np.median(t_b)), "diag_ms": float(np.median(t_d)),
                    "kernel_ms_covariance": float(cov_ms), "kernel_ms_cholesky": float(chol_ms),
                    "kernel_ms_sample_gemm": float(gemm_ms), "info": int(info.abs().max().item()),
                    "max_diff_vs_baseline_rel": float((so[:, :, 0] - sb).abs().max() / sb.abs().max()),
                    "max_diff_vs_baseline_rel_to_L_eps": float((so[:, :, 0] - sb).abs().max() / dev_b.abs().max())}
                del eps, so, sb, dev_b
                torch.cuda.empty_cache()
    out["card_after"] = card()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
