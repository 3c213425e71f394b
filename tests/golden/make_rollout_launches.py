"""Record tests/golden/rollout_launches.json: the launch sequence of one forward plus one reverse sweep per case of
tests/test_gpu_rollout_launches.py (needs a CUDA device).

    python tests/golden/make_rollout_launches.py [OUT.json]
"""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.join(os.path.dirname(HERE), "shims"))

import test_gpu_rollout_launches as tl  # noqa: E402

if __name__ == "__main__":
    out = sys.argv[1] if len(sys.argv) > 1 else os.path.join(HERE, "rollout_launches.json")
    with open(out, "w") as f:
        json.dump(tl.record(), f, indent=1, sort_keys=True)
        f.write("\n")
