"""Build-time evidence that the hot kernels are what DESIGN.md says they are, read from the SASS of the built
library with cuobjdump (no GPU needed): the forward and backward tile kernels use the fp64 tensor-core path
(DMMA.8x8x4), stage their operands with TMA bulk copies completing on an mbarrier (UBLKCP / SYNCS) and keep
everything in registers (no local-memory loads/stores); every device cubin targets sm_90a (H100)."""
import os
import re
import subprocess

import pytest

from util import CUOBJDUMP, ROOT, sass

LIB = os.path.join(ROOT, "pilco_b200", "libpilco_b200.so")

pytestmark = pytest.mark.skipif(not os.path.exists(CUOBJDUMP), reason="cuobjdump not available")


def test_device_code_targets_sm_90a():
    out = subprocess.run([CUOBJDUMP, "-lelf", LIB], capture_output=True, text=True, timeout=120).stdout
    cubins = re.findall(r"ELF file\s+\d+: (\S+)", out)
    assert len(cubins) >= 9 and all(c.endswith(".sm_90a.cubin") for c in cubins), cubins


def test_tile_kernels_use_dmma_tma_and_no_local_memory():
    fwd = sass(r"mm_tile_kernelILi\dELi3ELb1E")                              # the launched instantiation: 3 CTAs/SM, two row octets per warp
    bwd = sass(r"mm_btile_kernel")
    assert len(fwd) == 4 and len(bwd) == 8                                     # KS = 1..4 (x DIAG for the backward)
    for name, text in list(fwd.items()) + list(bwd.items()):
        assert "DMMA.8x8x4" in text, name
        assert "UBLKCP" in text and "SYNCS.ARRIVE.TRANS64" in text and "TRYWAIT" in text, name
    for name, text in fwd.items():
        assert not re.search(r"\b(STL|LDL)\b", text), "local memory traffic in %s" % name
    metric = [t for n, t in fwd.items() if "ILi3ELi3E" in n][0]                # D = 12 instantiation (metric shape)
    # off-diagonal body: two octets x (12 + 9 + 6 + 3) DMMA of the unrolled 4/3/2/1-tile groups + the one-octet form; diagonal bodies: 12 + 3 each
    assert metric.count("DMMA.8x8x4") >= 60 + 30 + 30
    assert "MUFU.EX2" not in metric                                            # table exp, not the SFU path


def test_taped_path_kernels_use_dmma_and_stay_in_registers():
    """Round 2: the taped forward tile kernel (what optimize_policy runs) and the tape-driven reverse-sweep kernel.
    Tile: DMMA for both products (exponent + H.[Z,1]), TMA-staged columns, no local memory in the launched register variant,
    table exp.  Finish: the weighted moment sums are DMMA (no DFMA inner product loops), metric-shape instantiation
    spill-free apart from a few bytes."""
    tile = sass(r"mm_tape_tile_kernelILi\d")
    assert len(tile) == 12                                                     # KS = 1..4 x 3 register variants
    for name, text in tile.items():
        assert "DMMA.8x8x4" in text and "UBLKCP" in text and "TRYWAIT" in text, name
        if "ELi256E" in name:                                                  # the launched variant (the 96- / 80-register tuning variants may spill a few scalars)
            assert not re.search(r"\b(STL|LDL)\b", text), "local memory traffic in %s" % name
        assert "MUFU.EX2" not in text, name
    metric = [t for n, t in tile.items() if "ILi3ELi256E" in n][0]             # D = 12, default register variant
    # per octet and 8-column tile: 3 (exponent) + 4 (H.[Z,1]) DMMA; two octets per pass, x 2 pair kinds x {1, 2 live octets}
    assert metric.count("DMMA.8x8x4") >= 2 * (7 + 14)
    fin = sass(r"rb_dyn_finish_kernelILi12E|mm_tape_bfinish_kernelILi12E")
    assert len(fin) == 2
    for name, text in fin.items():
        assert text.count("DMMA.8x8x4") >= 10, name                            # 3 + 3 symmetric tiles + 4 (Z'HZ) per k-step
        assert len(re.findall(r"\bSTL\b", text)) <= 24, name                   # (a handful of spilled scalars, no arrays)


def test_reverse_sweep_policy_kernels_present():
    """The recomputing VJP kernels that remain on the path (RBF policy, need_param) exist in every instantiation,
    finish + reduce are one kernel (no mm_breduce_kernel launch any more)."""
    names = sass(r"mm_bfinish_kernel|mm_breduce_kernel|mm_setup_fused_kernel")
    assert sum("mm_bfinish_kernel" in n for n in names) == 4
    assert not any("mm_breduce_kernel" in n for n in names)
    assert sum("mm_setup_fused_kernel" in n for n in names) == 8               # DP = 4..16 x {forward, ordered-pair backward}


def test_session3_shuffle_and_chain_properties():
    """Round 2, session 3: (1) the taped tile kernel's column sums use a reduce-scatter butterfly (3 64-bit shuffles per
    tile, none for the symmetric diagonal pairs): the whole metric-shape kernel -- four sweep loops plus the per-pass warp
    reductions -- holds fewer than 100 SHFL (it was 128 with the 6-shuffle butterfly in every loop); (2) the expected rewards
    are their own kernels, off the per-step chain: ro_state carries no LU / reward code any more (two shuffles: the
    partial-sum pairs of mm_finish)."""
    tile = sass(r"mm_tape_tile_kernelILi3ELi256E")
    assert len(tile) == 1
    assert sum(t.count("SHFL") for t in tile.values()) < 100
    ro = sass(r"ro_state_kernel|ro_reward_kernel|ro_reward_sum_kernel")
    assert len(ro) == 3
    state = [t for n, t in ro.items() if "ro_state" in n][0]
    assert state.count("SHFL") <= 4
    rew = [t for n, t in ro.items() if "ro_reward_kernel" in n][0]
    assert "MUFU" in rew                                                          # the reward's divisions / sqrt live here now


def test_issue_model_of_the_hot_loops():
    """scripts/issue_model.py on the built library: the structure of the innermost DMMA loops DESIGN.md section 6 reasons about.
    Forward tile kernel (metric shape): the two-octet loop issues 24 DMMA per 8 tiles with 36 LDS (one octet: 12 per 4 tiles,
    28 LDS) and not one shuffle; priced with the rates measured on an H100 (DMMA.8x8x4 17 cycles, fp64 2, three-register
    DFMA 3) that is 85 cycles per 8x8 tile.  Taped tile kernel: 14 DMMA per tile and octet pair; 6 shuffles in the loops of the non-symmetric
    pairs, none in those of the symmetric diagonal pairs."""
    import sys
    sys.path.insert(0, os.path.join(ROOT, "scripts"))
    import issue_model
    fwd = list(issue_model.analyse(r"mm_tile_kernelILi3ELi3ELb1E").values())
    assert len(fwd) == 1
    two = [c for _, c in fwd[0] if c["dmma"] == 24]
    one = [c for _, c in fwd[0] if c["dmma"] == 12]
    assert len(two) == 1 and len(one) == 1
    assert two[0]["shfl"] == 0 and one[0]["shfl"] == 0
    assert two[0]["lds"] <= 36 and one[0]["lds"] <= 28
    assert two[0]["cycles"] == 2 * one[0]["cycles"] and 83 <= two[0]["cycles"] / 8.0 <= 87      # 12*17 + 8*(7*2+3) = 340 per 4 tiles
    tape = list(issue_model.analyse(r"mm_tape_tile_kernelILi3ELi256E").values())
    assert len(tape) == 1
    pair_loops = [c for _, c in tape[0] if c["dmma"] == 14]
    single_loops = [c for _, c in tape[0] if c["dmma"] == 7]
    assert len(pair_loops) == 2 and len(single_loops) == 2                         # {symmetric diagonal, other} pairs x {2, 1} live octets
    assert sorted(c["shfl"] for c in pair_loops) == [0, 6]
    assert sorted(c["shfl"] for c in single_loops) == [0, 6]
