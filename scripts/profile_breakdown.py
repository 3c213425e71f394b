"""Per-kernel breakdown of the flagship forward rollout (bench.py's metric shape by default) with torch.profiler:
`python scripts/profile_breakdown.py [--config metric] [--R 32] [--nsplit 8] [--H 40] [--out DIR]`.

Two views of the same workload, each warmed up and then profiled over one pass:
  graph  -- what bench.py times: the H-step rollout of R restarts as ONE captured CUDA graph of `nsplit` sub-batches
            on parallel streams, one replay;
  eager  -- one sub-batch's plan (R / nsplit restarts), its forward run eagerly for the same H steps.
For each it prints the kernels' summed device time, launch count and share of the summed kernel time.  Sub-batches
overlap on the device, so the shares are shares of kernel time, not of wall time.  With --out DIR the tables are also
written to DIR/profile_breakdown.txt."""
import argparse
import os
import sys
from collections import defaultdict

import numpy as np
import torch
from torch.profiler import ProfilerActivity, profile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench                                     # noqa: E402  (the benchmark's seeded workload and policies)
from pilco_b200 import engine, _lib              # noqa: E402


def kernel_table(prof):
    tot, cnt = defaultdict(float), defaultdict(int)
    for ev in prof.events():
        if ev.device_type == torch.autograd.DeviceType.CUDA and ev.device_time_total > 0:
            name = ev.name.split("(")[0]
            if name.startswith("void "):
                name = name[5:]
            tot[name] += ev.device_time_total
            cnt[name] += 1
    return tot, cnt


def fmt(title, tot, cnt, steps):
    s = sum(tot.values())
    lines = ["%s: %d kernels, %.1f us summed kernel time (%.2f us per rollout step)" % (title, sum(cnt.values()), s, s / steps),
             "%-58s %8s %12s %7s" % ("kernel", "launches", "total us", "share")]
    for k in sorted(tot, key=tot.get, reverse=True):
        lines.append("%-58s %8d %12.1f %6.1f%%" % (k[:58], cnt[k], tot[k], 100.0 * tot[k] / s if s else 0.0))
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
    out.append(fmt("graph: R=%d, H=%d, %d sub-batches, one replay" % (R, H, nsplit), *kernel_table(prof), H))

    plan = make_plan(0, R // nsplit)
    for _ in range(2):
        plan.forward()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        plan.forward()
        torch.cuda.synchronize()
    out.append(fmt("eager: one sub-batch, R=%d, H=%d" % (R // nsplit, H), *kernel_table(prof), H))

    text = "%s (%s)\n\n%s\n" % (torch.cuda.get_device_name(), bench.metric_name(cfg), "\n\n".join(out))
    print(text)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "profile_breakdown.txt"), "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
