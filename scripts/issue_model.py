"""Static issue-path model of the tile kernels' hot loops, read from the SASS of the built library (no GPU needed).

For every innermost loop that holds DMMA instructions it counts the instruction classes and prices them per warp on one
SM sub-partition with the rates measured on an H100 SXM (80GB HBM3, 700 W, 1980 MHz): DMMA.8x8x4 from bench.py's
pilco_microbench_fp64 (31.7 TFLOP/s over 132 SMs x 4 sub-partitions), the fp64 instructions from scripts/ubench/fp64_mix.cu:

    DMMA.8x8x4 (512 flop)                       17 cycles of the fp64 pipe per warp (about half the H100's fp64 tensor
                                                rate: the native DMMA.16x8x16 reaches 54.8 TFLOP/s in the same process)
    DMMA.16x8x4 / 16x8x8 / 16x8x16              the same pipe time per flop as their measured rates say (DMMA_CYCLES)
    DADD / DMUL / DFMA, <= 2 distinct registers  2 cycles
    DFMA with three distinct register sources    3 cycles   (operand bandwidth)
    everything else                             not priced (co-issues; what it really costs is the gap between this model
                                                and the measurement -- shuffles and the table gather, DESIGN.md section 6)

    python scripts/issue_model.py [kernel-regex ...]      default: the forward and the taped tile kernel at the metric shape

Output: one line per loop -- SASS address range, DMMA (by shape) / fp64 (3-register ones apart) / LDS / SHFL / other counts, model
cycles per iteration.  tests/test_sass_properties.py::test_issue_model_of_the_hot_loops and tests/test_sass_m16.py pin the
structure it finds.
"""
import os
import re
import shutil
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "pilco_b200", "libpilco_b200.so")
CUOBJDUMP = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
DEFAULT = [r"mm_tile_m16_kernelILi3E", r"mm_tape_tile_m16_kernelILi3E", r"mm_tile_kernelILi3ELi3ELb1E", r"mm_tape_tile_kernelILi3ELi256E"]

# fp64-pipe cycles per warp instruction and SM sub-partition, by DMMA shape: 17 for DMMA.8x8x4 (31.7 TFLOP/s), the 16x8
# shapes scaled by flop / rate against it (pilco_microbench_fp64 which = 7, 5, 6 on an H100 SXM: 16x8x8 51.3 and 16x8x16
# 54.8 TFLOP/s at 700 W; 16x8x4 49.1 TFLOP/s at 400 W, where 8x8x4 also measured 31.7)
DMMA_CYCLES = {"8x8x4": 17, "16x8x4": 22, "16x8x8": 42, "16x8x16": 79}

INS = re.compile(r"^\s+/\*([0-9a-f]{4,})\*/\s+(.*?);")


def functions(pattern, lib=LIB):
    out = subprocess.run([CUOBJDUMP, "-sass", lib], capture_output=True, text=True, timeout=600).stdout
    funcs, name = {}, None
    for line in out.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            name = m.group(1) if re.search(pattern, m.group(1)) else None
            if name:
                funcs[name] = []
        elif name:
            mi = INS.match(line)
            if mi:
                funcs[name].append((int(mi.group(1), 16), mi.group(2).strip()))
    return funcs


def distinct_registers(text):
    """64-bit register sources of an fp64 instruction (the destination is the first operand)"""
    ops = text.split(None, 1)[1] if " " in text else ""
    srcs = [o.strip() for o in ops.split(",")[1:]]
    regs = set()
    for o in srcs:
        m = re.match(r"^[-|]*R(\d+)", o)
        if m:
            regs.add(int(m.group(1)))
    return len(regs)


def loops(code):
    """innermost loops = backward branches whose range holds no other backward-branch target range"""
    addr = [a for a, _ in code]
    spans = []
    for a, t in code:
        m = re.search(r"\bBRA(?:\.\S+)?\s+(?:\S+,\s+)?(0x[0-9a-f]+)", t)
        if m and not t.startswith("BRA.DIV"):
            tgt = int(m.group(1), 16)
            if tgt <= a and tgt in addr:
                spans.append((tgt, a))
    inner = [s for s in spans if not any(o != s and s[0] <= o[0] and o[1] <= s[1] for o in spans)]
    return sorted(set(inner))


def model(code, lo, hi):
    c = dict(dmma=0, fp64=0, fp64_3=0, lds=0, shfl=0, other=0, dmma_cycles=0, shapes={})
    for a, t in code:
        if a < lo or a > hi:
            continue
        body = re.sub(r"^@!?U?P\d+\s+", "", t)
        op = body.split()[0]
        if op.startswith("DMMA"):
            c["dmma"] += 1
            shape = op.split(".")[1] if "." in op else "8x8x4"
            c["shapes"][shape] = c["shapes"].get(shape, 0) + 1
            c["dmma_cycles"] += DMMA_CYCLES[shape]
        elif op.split(".")[0] in ("DADD", "DMUL", "DFMA"):
            if op.startswith("DFMA") and distinct_registers(body) >= 3:
                c["fp64_3"] += 1
            else:
                c["fp64"] += 1
        elif op.startswith("LDS"):
            c["lds"] += 1
        elif op.startswith("SHFL"):
            c["shfl"] += 1
        elif op != "NOP":
            c["other"] += 1
    c["cycles"] = c["dmma_cycles"] + 2 * c["fp64"] + 3 * c["fp64_3"]
    return c


def analyse(pattern, lib=LIB):
    res = {}
    for name, code in functions(pattern, lib).items():
        rows = []
        for lo, hi in loops(code):
            c = model(code, lo, hi)
            if c["dmma"]:
                rows.append(((lo, hi), c))
        res[name] = rows
    return res


if __name__ == "__main__":
    pats = sys.argv[1:] or DEFAULT
    for pat in pats:
        for name, rows in analyse(pat).items():
            print(name)
            for (lo, hi), c in rows:
                print("  loop %05x-%05x  DMMA %3d (%s)  fp64 %3d (+%2d three-register)  LDS %3d  SHFL %2d  other %3d  -> model %4d cycles/iteration"
                      % (lo, hi, c["dmma"], " ".join("%sx%d" % kv for kv in sorted(c["shapes"].items())), c["fp64"], c["fp64_3"],
                         c["lds"], c["shfl"], c["other"], c["cycles"]))
