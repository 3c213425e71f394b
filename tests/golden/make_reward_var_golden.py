"""Generate tests/golden/reward_var.npz by EXECUTING the reference's reward.m (the checksummed copy under
tests/reference_tests/Matlab Code) with oracle/mrun.py for all six outputs, on the inputs of the reward_2 / reward_5
recipes (tests/golden/make_golden.py): the reward variance sR and its derivatives dsRdm, dsRdS, which the exploration
objective's gradient uses (DESIGN.md section 21).

    python tests/golden/make_reward_var_golden.py
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
from oracle import mrun            # noqa: E402


def main():
    out = {}
    for kdim in (2, 5):
        g = np.load(os.path.join(HERE, "reward_%d.npz" % kdim))
        m, s, W, t = g["m"], g["s"], g["W"], g["t"]
        muR, dm, dS, sR, dsm, dsS = mrun.run("reward", m.T, s, t.T, W, nout=6)
        for k, v in dict(m=m, s=s, W=W, t=t, muR=muR, dmuRdm=dm, dmuRdS=dS, sR=sR, dsRdm=dsm, dsRdS=dsS).items():
            out["%s_%d" % (k, kdim)] = np.asarray(v, dtype=np.float64)
    np.savez_compressed(os.path.join(HERE, "reward_var.npz"), **out)
    print("wrote reward_var", {k: v.shape for k, v in out.items()})


if __name__ == "__main__":
    main()
