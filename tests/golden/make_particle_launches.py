"""Record tests/golden/particle_launches.json: the launch sequence of one call per case of
tests/test_gpu_particle_launches.py (needs a CUDA device).

    python tests/golden/make_particle_launches.py [OUT.json]
"""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.join(os.path.dirname(HERE), "shims"))

import test_gpu_particle_launches as tl  # noqa: E402

if __name__ == "__main__":
    out = sys.argv[1] if len(sys.argv) > 1 else os.path.join(HERE, "particle_launches.json")
    with open(out, "w") as f:
        json.dump(tl.record(), f, indent=1, sort_keys=True)
        f.write("\n")
