"""The workspace and tape sizes the ten size queries of the moment-matching rollout report (pilco_rollout_*,
pilco_rollout_angles_*, pilco_rollout_explore_*, pilco_rollout_noisy_*), over a grid of descriptions: linear and RBF
policies, rollouts shaped for 0, 1 or 2 angle dimensions queried with and without angles (also mismatched ones),
exploration off / inactive / b = 0 with step_var / b != 0, measurement noise off and on, state, joint and MULT-channel
reward terms, H = 0 and H > 0, with and without a tape, and a dynamics GP too large for the taped pass.  Against
tests/golden/rollout_sizes.npz (tests/golden/make_rollout_sizes.py): a buffer sized by one build fits every other."""
import ctypes
import itertools
import os

import numpy as np

from abi_fakes import FAKE, _gp, _rollout

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "rollout_sizes.npz")
QUERIES = ("workspace_bytes", "tape_bytes", "bwd_workspace_bytes", "angles_workspace_bytes", "angles_tape_bytes",
           "angles_bwd_workspace_bytes", "explore_workspace_bytes", "explore_bwd_workspace_bytes",
           "noisy_workspace_bytes", "noisy_bwd_workspace_bytes")
TERMS = ("state", "joint", "mult")
# (angle dimensions the rollout is shaped for, those of the query; None: no pilco_angles)
ANGLES = ((0, None), (0, 0), (0, 1), (1, None), (1, 1), (1, 2), (2, 0), (2, 2))
EXPLORE = ("off", "b0", "b0_step_var", "b")


def grid():
    return list(itertools.product((0, 1), TERMS, (0, 4), ((40, False), (40, True), (3000, True)), ANGLES, EXPLORE,
                                  (False, True)))


def _description(rbf, terms, H, n_tape, shape_A):
    from pilco_b200 import _lib
    Ds, U, R = 3, 2, 3
    Dh = Ds + shape_A
    ro = _rollout(kind=_lib.POLICY_RBF if rbf else _lib.POLICY_LINEAR)
    ro.R, ro.H = R, H
    ro.dyn = _gp(n=n_tape[0], D=Dh + U, E=Ds)
    ro.pol.Ds, ro.pol.U = Dh, U
    if rbf:
        ro.pol.rbf = _gp(n=12, D=Dh, E=U, mode=1, iK=None, ldk=0)
    if terms != "state":
        k = ro.n_rewards
        ro.n_rewards = k + 1
        ro.rewards[k].kind = _lib.REWARD_EXP_SA if terms == "joint" else _lib.REWARD_BOX
        ro.rewards[k].channel = _lib.CHANNEL_MULT if terms == "mult" else _lib.CHANNEL_ADD
        ro.rewards[k].coef, ro.rewards[k].W, ro.rewards[k].t = 0.5, FAKE, FAKE
    if n_tape[1]:
        ro.tape, ro.tape_bytes = FAKE, 1 << 40
    return ro


def sizes(lib):
    """[len(grid()), len(QUERIES)] of what `lib` reports"""
    from pilco_b200 import _lib
    C = ctypes
    out = np.zeros((len(grid()), len(QUERIES)), dtype=np.int64)
    for i, (rbf, terms, H, n_tape, (shape_A, A), ex, noisy) in enumerate(grid()):
        ro = C.byref(_description(rbf, terms, H, n_tape, shape_A))
        ang = None
        if A is not None:
            a = _lib.Angles()
            a.A = A
            for j in range(A):
                a.dims[j] = j
            ang = C.byref(a)
        e = None if ex == "off" else C.byref(_lib.Exploration(0.5 if ex == "b" else 0.0,
                                                             FAKE if ex == "b0_step_var" else None))
        nz = C.byref(_lib.ObsNoise()) if noisy else None
        f = lambda q: getattr(lib, "pilco_rollout_" + q)
        out[i] = [f("workspace_bytes")(ro), f("tape_bytes")(ro), f("bwd_workspace_bytes")(ro),
                  f("angles_workspace_bytes")(ro, ang), f("angles_tape_bytes")(ro, ang),
                  f("angles_bwd_workspace_bytes")(ro, ang), f("explore_workspace_bytes")(ro, ang, e),
                  f("explore_bwd_workspace_bytes")(ro, ang, e), f("noisy_workspace_bytes")(ro, ang, e, nz),
                  f("noisy_bwd_workspace_bytes")(ro, ang, e, nz)]
    return out


def test_sizes_match_the_golden():
    from pilco_b200 import _lib
    want = np.load(GOLDEN)["sizes"]
    got = sizes(_lib.lib)
    assert got.shape == want.shape
    bad = np.argwhere(got != want)
    g = grid()
    assert bad.size == 0, [(g[i], QUERIES[j], int(got[i, j]), int(want[i, j])) for i, j in bad[:10]]
    # the grid reaches every layout: no tape for the large GP, and each feature moves some size
    assert (want[:, 1] == 0).any() and (want[:, 1] > 0).any()
    for j, base in ((3, 0), (5, 2), (6, 3), (8, 6), (9, 7)):
        assert (want[:, j] != want[:, base]).any(), QUERIES[j]
