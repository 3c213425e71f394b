"""Record tests/golden/particle_abi.npz: the status of every particle rollout call and the bytes of every particle size
query over the grid of tests/test_particle_abi_host.py (no GPU needed).  PILCO_B200_LIB selects the library to record.

    python tests/golden/make_particle_abi.py
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, os.path.dirname(HERE))

import test_particle_abi_host as ta  # noqa: E402

if __name__ == "__main__":
    np.savez_compressed(os.path.join(HERE, "particle_abi.npz"), **ta.record())
