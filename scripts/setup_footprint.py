"""SM footprint of the dynamics setup kernels in the flagship forward rollout (bench.py's metric shape by default):
`python scripts/setup_footprint.py [--config metric] [--R 32] [--nsplit 8] [--H 40] [--out DIR]`.

A setup CTA that holds an SM slot is a slot no tile CTA of another sub-batch can use, so beside each kernel's device time
this reports its CTAs and its slot time, CTA-us = grid size x kernel duration, summed over the launches of one graph
replay, as a share of the dynamics tile kernel's.  Three parts, all from one process on one card:
  graph  -- scripts/profile_breakdown.py's graph view (one replay of the R-restart rollout in nsplit sub-batches), with
            the grid of every launch read from the profiler trace;
  eager  -- profile_breakdown's eager view (one sub-batch's forward run eagerly);
  setup  -- the R-restart setup call on its own through pilco_mm_forward_profile (ms_out[0]), mean of 5 after 3 warm-up
            calls, with an L2 flush before each.
The card's name, power limit and SM clock go in the header.  With --out DIR the text is also written to
DIR/setup_footprint.txt."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile
from collections import defaultdict

import numpy as np
import torch
from torch.profiler import ProfilerActivity, profile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
import bench                                     # noqa: E402  (the benchmark's seeded workload and policies)
import profile_breakdown as pb                   # noqa: E402
from pilco_b200 import engine, _lib              # noqa: E402
from pilco_b200._lib import lib                  # noqa: E402
from pilco_b200.engine import ptr, stream_ptr    # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()),
                            "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = ""
    return q or torch.cuda.get_device_name()


def kernel_slots(prof):
    """(name, grid) -> [launches, summed us, summed CTA-us] from the profiler's trace (kernel events carry their grid)."""
    with tempfile.TemporaryDirectory() as td:
        path = os.path.join(td, "trace.json")
        prof.export_chrome_trace(path)
        with open(path) as f:
            events = json.load(f)["traceEvents"]
    out = defaultdict(lambda: [0, 0.0, 0.0])
    for ev in events:
        if ev.get("cat") != "kernel":
            continue
        name = ev["name"].split("(")[0]
        if name.startswith("void "):
            name = name[5:]
        grid = tuple(ev.get("args", {}).get("grid", (0, 0, 0)))
        ctas = int(np.prod(grid)) if grid else 0
        row = out[(name, grid)]
        row[0] += 1
        row[1] += ev["dur"]
        row[2] += ctas * ev["dur"]
    return out


def slot_table(title, slots):
    tile = max((k for k in slots if k[0].startswith("mm_tile")), key=lambda k: slots[k][2], default=None)
    ref = slots[tile][2] if tile else 0.0
    lines = [title + "  (slot time = grid CTAs x duration; share: of the dynamics tile's, %s grid %s)" % tile if tile else title,
             "%-40s %14s %8s %10s %14s %8s" % ("kernel", "grid", "launches", "us each", "CTA-us", "share")]
    for k in sorted(slots, key=lambda k: slots[k][2], reverse=True):
        n, us, cus = slots[k]
        lines.append("%-40s %14s %8d %10.1f %14.0f %7.1f%%" % (k[0][:40], "x".join(map(str, k[1])), n, us / n, cus,
                                                             100.0 * cus / ref if ref else 0.0))
    return "\n".join(lines)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="metric", choices=sorted(bench.CONFIGS))
    ap.add_argument("--R", type=int, default=0, help="restarts (default: the config's)")
    ap.add_argument("--nsplit", type=int, default=8)
    ap.add_argument("--H", type=int, default=0, help="rollout steps (default: the config's)")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    cfg = bench.CONFIGS[a.config]
    R, H = a.R or cfg["R"], a.H or cfg["H"]
    Ds, U = cfg["Ds"], cfg["U"]
    D = Ds + U
    nsplit = max(1, min(a.nsplit, R))
    wl = bench.make_workload(cfg)
    gp = engine.gp_factorize(wl["X"], wl["Y"], wl["ell"], wl["sf2"], wl["sn2"])
    pol = bench.make_policies(cfg, np.arange(R))
    ones, noise = np.ones((R, U)), 1e-4 * np.ones((R, U))
    rew = [dict(kind=_lib.REWARD_EXP, coef=1.0, W=wl["W"], t=wl["t"])]

    def make_plan(lo, hi):
        pg = engine.gp_factorize(pol["Xc"][lo:hi], pol["Yc"][lo:hi], pol["lc"][lo:hi], ones[lo:hi], noise[lo:hi], need_iK=False, mode=1)
        spec = dict(kind=_lib.POLICY_RBF, Ds=Ds, U=U, squash=True, max_action=np.ones(U), gp=pg)
        return engine.RolloutPlan(gp, spec, rew, wl["m0"], wl["S0"], H, R=hi - lo)

    out = []
    split = engine.SplitRollout(make_plan, R, nsplit=nsplit)
    for _ in range(3):
        split.replay()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        split.replay()
        torch.cuda.synchronize()
    out.append(pb.fmt("graph: R=%d, H=%d, %d sub-batches, one replay" % (R, H, nsplit), *pb.kernel_table(prof), H))
    out.append(slot_table("graph slot time, one replay", kernel_slots(prof)))

    plan = make_plan(0, R // nsplit)
    for _ in range(2):
        plan.forward()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        plan.forward()
        torch.cuda.synchronize()
    out.append(pb.fmt("eager: one sub-batch, R=%d, H=%d" % (R // nsplit, H), *pb.kernel_table(prof), H))

    # the R-restart setup call on its own (setup = stage 1, output and pair kernels in stream order)
    d = engine.device()
    E, n_c = Ds, gp.n
    g = gp.struct()
    ms3 = (C.c_float * 3)()
    Mo = torch.empty((R, E), dtype=torch.float64, device=d); So = torch.empty((R, E, E), dtype=torch.float64, device=d)
    Vo = torch.empty((R, D, E), dtype=torch.float64, device=d); info = torch.zeros(R, dtype=torch.int32, device=d)
    wsb = lib.pilco_mm_workspace_bytes(n_c, D, E, R)
    ws = torch.empty(wsb // 8, dtype=torch.float64, device=d)
    mj = engine.dev(np.tile(np.concatenate([wl["m0"], np.zeros(U)]), (R, 1)))
    sj = engine.dev(np.tile(0.1 * np.eye(D), (R, 1, 1)))
    flush = torch.empty(256 * 1024 * 1024 // 8, dtype=torch.float64, device=d)       # > L2 (50 MB on H100)
    setup = []
    for i in range(8):
        flush.fill_(1.0)
        _lib.check(lib.pilco_mm_forward_profile(C.byref(g), R, ptr(mj), ptr(sj), ptr(Mo), ptr(So), ptr(Vo), ptr(info),
                                                ptr(ws), wsb, ms3, stream_ptr()))
        if i >= 3:
            setup.append(1e3 * ms3[0])
    out.append("setup call alone: R=%d, pilco_mm_forward_profile ms_out[0]: %.1f us (mean of 5; min %.1f, max %.1f)"
               % (R, np.mean(setup), np.min(setup), np.max(setup)))

    text = "%s (%s)\n\n%s\n" % (card(), bench.metric_name(cfg), "\n\n".join(out))
    print(text)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "setup_footprint.txt"), "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
