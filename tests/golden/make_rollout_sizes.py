"""Record tests/golden/rollout_sizes.npz: the sizes the moment-matching rollout's size queries report over the grid of
tests/test_rollout_sizes_host.py (no GPU needed).  PILCO_B200_LIB selects the library to record.

    python tests/golden/make_rollout_sizes.py
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, os.path.dirname(HERE))

import test_rollout_sizes_host as ts  # noqa: E402
from pilco_b200 import _lib  # noqa: E402

if __name__ == "__main__":
    np.savez_compressed(os.path.join(HERE, "rollout_sizes.npz"), sizes=ts.sizes(_lib.lib))
