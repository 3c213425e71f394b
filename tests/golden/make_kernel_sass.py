"""Record tests/golden/kernel_sass.json: the SHA-256 of every kernel's SASS in a built library, keyed by mangled name.
tests/test_particles_cem_policy_host.py checks that the stationary policies' batched forward rollouts (DESIGN.md
section 33), which are host orchestration only, left every kernel's SASS as it was.

    python tests/golden/make_kernel_sass.py [LIBRARY.so] [OUT.json]
"""
import hashlib
import json
import os
import re
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
CUOBJDUMP = "/usr/local/cuda/bin/cuobjdump"


def kernel_hashes(lib):
    """{mangled name: [sha256 of its SASS text, one per module that has it, in the library's order]}, split as
    tests/util.py's sass() splits cuobjdump's output"""
    out = subprocess.run([CUOBJDUMP, "-sass", lib], capture_output=True, text=True, timeout=600).stdout
    funcs, name, lines = {}, None, []
    for line in out.splitlines() + ["Fatbin"]:
        m = re.match(r"\s*Function : (\S+)", line)
        if m or line.startswith("Fatbin"):
            if name:
                funcs.setdefault(name, []).append(hashlib.sha256("\n".join(lines).encode()).hexdigest())
            name, lines = (m.group(1) if m else None), []
        elif name:
            lines.append(line)
    return funcs


if __name__ == "__main__":
    lib = sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "pilco_b200", "libpilco_b200.so")
    out = sys.argv[2] if len(sys.argv) > 2 else os.path.join(HERE, "kernel_sass.json")
    with open(out, "w") as f:
        json.dump(kernel_hashes(lib), f, indent=0, sort_keys=True)
        f.write("\n")
