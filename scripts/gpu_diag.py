"""First-light diagnostics on the GPU: fp64 pipe microbenchmarks + raw timing of the moment-match
kernels at the metric configuration.  Writes gpurun_out/diag.json."""
import ctypes as C
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from pilco_b200 import engine, _lib          # noqa: E402
from pilco_b200._lib import lib              # noqa: E402
from util import make_gp_problem, make_input  # noqa: E402

out = {}
d = engine.device()
print(torch.cuda.get_device_name(0))
sink = torch.zeros(8, dtype=torch.float64, device=d)
ms = C.c_float()
names = {0: "dfma", 1: "dmma", 2: "dfma+dmma", 3: "exp_tab", 4: "exp_libdevice"}
iters, blocks = 20000, torch.cuda.get_device_properties(0).multi_processor_count * 4
for which in range(5):
    _lib.check(lib.pilco_microbench_fp64(which, iters, blocks, engine.ptr(sink), C.byref(ms), engine.stream_ptr()))
    thread_ops = blocks * 256 * iters * 8.0
    t = ms.value * 1e-3
    rec = {"ms": ms.value}
    if which == 0:
        rec["TFLOPS"] = 2 * thread_ops / t / 1e12
    elif which == 1:
        rec["TFLOPS"] = 2 * (blocks * 8 * iters * 16.0) * 256 / t / 1e12     # 16 DMMA/warp/iter x 256 FMA
    elif which == 2:
        rec["dfma_TFLOPS"] = 2 * thread_ops / t / 1e12
        rec["dmma_TFLOPS"] = 2 * (blocks * 8 * iters * 16.0) * 256 / t / 1e12
    else:
        rec["Gexp_per_s"] = thread_ops / t / 1e9
    out[names[which]] = rec
    print(names[which], rec)


def time_fn(fn, n=20, warm=3):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


for (n, D, E, R) in [(300, 12, 10, 1), (300, 12, 10, 32), (300, 5, 4, 32), (500, 10, 8, 32)]:
    X, Y, ell, sf2, sn2 = make_gp_problem(n, D, E, seed=1)
    t0 = time.time()
    gp = engine.gp_factorize(X, Y, ell, sf2, sn2)
    torch.cuda.synchronize()
    tf = time.time() - t0
    m = np.concatenate([make_input(D, seed=r)[0] for r in range(R)])
    s = np.stack([0.1 * make_input(D, seed=r)[1] for r in range(R)])
    md, sd = engine.dev(m), engine.dev(s)
    M = torch.empty((R, E), dtype=torch.float64, device=d)
    S = torch.empty((R, E, E), dtype=torch.float64, device=d)
    V = torch.empty((R, D, E), dtype=torch.float64, device=d)
    info = torch.zeros(R, dtype=torch.int32, device=d)
    wsb = lib.pilco_mm_workspace_bytes(n, D, E, R)
    ws = torch.empty(wsb // 8, dtype=torch.float64, device=d)
    g = gp.struct()

    def call():
        _lib.check(lib.pilco_mm_forward(C.byref(g), R, engine.ptr(md), engine.ptr(sd), engine.ptr(M), engine.ptr(S),
                                        engine.ptr(V), engine.ptr(info), engine.ptr(ws), wsb, engine.stream_ptr()))
    t = time_fn(call)
    P = E * (E + 1) // 2
    elems = P * n * n * R
    rec = {"ms_per_call": t, "mm_per_s": R / (t * 1e-3), "Gelem_per_s": elems / (t * 1e-3) / 1e9,
           "factorize_s_first": tf}
    out["mm_n%d_D%d_E%d_R%d" % (n, D, E, R)] = rec
    print((n, D, E, R), rec)

os.makedirs(os.path.join(ROOT, "gpurun_out"), exist_ok=True)
with open(os.path.join(ROOT, "gpurun_out", "diag.json"), "w") as f:
    json.dump(out, f, indent=1)
