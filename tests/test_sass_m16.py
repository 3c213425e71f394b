"""Build-time evidence for the tile kernels on Hopper's native 16x8 fp64 MMA shapes (mm_tile_m16_kernel,
mm_tape_tile_m16_kernel), read from the SASS of the built library with cuobjdump (no GPU needed): the off-diagonal
loops issue DMMA.16x8x* only, the columns are TMA-staged, nothing lives in local memory, the exp is the table exp,
and the hot loops keep the structure DESIGN.md section 6 prices (scripts/issue_model.py)."""
import os
import re
import sys

import pytest

from util import CUOBJDUMP, ROOT, sass

pytestmark = pytest.mark.skipif(not os.path.exists(CUOBJDUMP), reason="cuobjdump not available")

# K decomposition of the exponent per KS (k-steps of 4): one MMA per K chunk
EXPONENT_SHAPES = {1: ["16x8x4"], 2: ["16x8x8"], 3: ["16x8x8", "16x8x4"], 4: ["16x8x16"]}


def _issue_model():
    sys.path.insert(0, os.path.join(ROOT, "scripts"))
    import issue_model
    return issue_model


def _ks(name):
    return int(re.search(r"m16_kernelILi(\d)E", name).group(1))


def test_m16_kernels_use_16x8_dmma_tma_and_no_local_memory():
    fwd = sass(r"mm_tile_m16_kernelILi\dE")
    tape = sass(r"mm_tape_tile_m16_kernelILi\dE")
    assert len(fwd) == 4 and len(tape) == 4                                    # KS = 1..4
    for name, text in list(fwd.items()) + list(tape.items()):
        for shape in EXPONENT_SHAPES[_ks(name)]:
            assert "DMMA." + shape in text, (name, shape)
        assert "UBLKCP" in text and "TRYWAIT" in text, name
        assert not re.search(r"\b(STL|LDL)\b", text), "local memory traffic in %s" % name
        assert "MUFU.EX2" not in text, name
    for name, text in tape.items():
        assert "DMMA.16x8x8" in text, name                                     # H.[Z,1]: one 16x8x8 per n-tile
        assert "DMMA.8x8x4" not in text, name                                  # no one-octet fall-back anywhere


def test_m16_forward_loops():
    """Every KS: the off-diagonal loop (the one with 16x8 MMAs) issues no DMMA.8x8x4 and no shuffle; the 8x8x4 loops
    left are the diagonal pairs' one-octet bodies.  Metric shape (KS = 3): one 16x8x8 + one 16x8x4 per 16x8 tile (groups
    of 3 column tiles), i.e. 8 DMMA per 8 8x8 tiles where the 8x8x4 kernel issues 24, with no more LDS per tile than its
    36 per 8 tiles, and a lower model price per tile."""
    im = _issue_model()
    for name, rows in im.analyse(r"mm_tile_m16_kernelILi\dE").items():
        ks = _ks(name)
        m16 = [c for _, c in rows if any(s.startswith("16x8") for s in c["shapes"])]
        assert m16, name
        for c in m16:
            assert "8x8x4" not in c["shapes"], (name, c["shapes"])
            assert c["shfl"] == 0, name
        if ks == 3:
            assert len(m16) == 1
            c = m16[0]
            n16 = c["shapes"].get("16x8x8", 0)                                 # 16x8 tiles per iteration = 2 n16 8x8 tiles
            assert n16 >= 2 and c["shapes"] == {"16x8x8": n16, "16x8x4": n16}, c["shapes"]
            assert c["lds"] * 8 <= 36 * 2 * n16
            old = list(im.analyse(r"mm_tile_kernelILi3ELi3ELb1E").values())[0]
            two = [o for _, o in old if o["dmma"] == 24][0]
            assert c["cycles"] / (2.0 * n16) < two["cycles"] / 8.0             # the model's price per 8x8 tile drops


def test_m16_taped_loops():
    """Taped kernel, metric shape: per 8-column tile and octet pair one 16x8x8 + one 16x8x4 (exponent) and two 16x8x8
    (H.[Z,1], NT = 2) -- 4 DMMA where the 8x8x4 kernel issues 14; the column-sum butterfly keeps its 6 shuffles, none for
    the symmetric diagonal pairs.  No one-octet loop is left (the last pass pairs the remaining octets instead)."""
    im = _issue_model()
    rows = list(im.analyse(r"mm_tape_tile_m16_kernelILi3E").values())
    assert len(rows) == 1
    loops = [c for _, c in rows[0]]
    assert len(loops) == 2                                                     # {symmetric diagonal, other} pairs
    for c in loops:
        assert c["shapes"] == {"16x8x8": 3, "16x8x4": 1}, c["shapes"]
    assert sorted(c["shfl"] for c in loops) == [0, 6]
