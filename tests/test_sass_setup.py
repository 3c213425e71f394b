"""Build-time evidence, read from the SASS of the built library (no GPU needed), that the forward two-stage setup is what
DESIGN.md section 3 describes: stage 2 runs as a pair kernel, which stages zeta and the pair block with TMA bulk copies
on an mbarrier, and an output kernel; neither touches local memory, and the fused stage-2 kernel of both task kinds is
gone (the ordered-pair backward mode keeps its own stage-2 kernel).  These checks pin structure only: that the split
kernels compute what the fused single-restart path computes, bit for bit, is checked on the GPU by test_gpu_configs'
batch-position test (R=32 two-stage against R=1 fused; its swimmer case, np=512 at ldz=12, runs the pair kernel with two
row chunks per pair)."""
import os
import re

import pytest

from util import CUOBJDUMP, sass

pytestmark = pytest.mark.skipif(not os.path.exists(CUOBJDUMP), reason="cuobjdump not available")


def test_forward_stage2_kernels_stay_in_registers_and_pair_kernel_uses_tma():
    pair = sass(r"mm_setup2_pair_kernel")
    out = sass(r"mm_setup2_out_kernel")
    assert len(pair) == 4 and len(out) == 4                                    # DP = 4, 8, 12, 16
    for name, text in list(pair.items()) + list(out.items()):
        assert not re.search(r"\b(STL|LDL)\b", text), "local memory traffic in %s" % name
    for name, text in pair.items():
        assert "UBLKCP" in text and "SYNCS.ARRIVE.TRANS64" in text and "TRYWAIT" in text, name
        assert "DMMA.8x8x4" in text, name
    metric = [t for n, t in pair.items() if "ILi12E" in n][0]
    # two octets per sweep step: 2 x 6 DMMA for the B pieces, 2 x 6 for the row operands (D = 12: KS = 3, two n-tiles)
    assert metric.count("DMMA.8x8x4") >= 24


def test_combined_forward_stage2_kernel_is_gone():
    names = sass(r"mm_setup2")
    assert not any(re.search(r"mm_setup2_kernel", n) for n in names)
    assert sum("mm_setup2_bwd_kernel" in n for n in names) == 4
