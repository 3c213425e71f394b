"""Error behaviour of the C ABI (include/pilco_b200.h: "0 ok, <0 invalid argument"), checked WITHOUT a GPU: every
entry point validates its arguments on the host before it enqueues anything, so invalid calls must come back with
the documented status and never touch the device.  Pointers below are fake non-null addresses; a call that passed
validation would launch kernels, so only rejecting calls are made here."""
import ctypes as C

import pytest

from pilco_b200 import _lib
from pilco_b200._lib import lib
from abi_fakes import OK, ERR_NULL, ERR_DIM, ERR_WS, ERR_ALIGN, ERR_LAUNCH, ERR_UNSUP, FAKE, _gp, _rollout


def test_status_strings():
    for code in (OK, ERR_NULL, ERR_DIM, ERR_WS, ERR_ALIGN, ERR_LAUNCH, ERR_UNSUP):
        assert len(lib.pilco_status_string(code)) > 1
    assert b"unknown" in lib.pilco_status_string(-99)


def test_mm_forward_argument_validation():
    args = lambda g, R=1, ws=FAKE, wsb=1 << 30: (C.byref(g), R, FAKE, FAKE, FAKE, FAKE, FAKE, None, ws, wsb, None)
    assert lib.pilco_mm_forward(None, 1, FAKE, FAKE, FAKE, FAKE, FAKE, None, FAKE, 1 << 30, None) == ERR_NULL
    assert lib.pilco_mm_forward(*args(_gp(D=17))) == ERR_DIM                 # D > PILCO_MAX_D
    assert lib.pilco_mm_forward(*args(_gp(E=0))) == ERR_DIM
    assert lib.pilco_mm_forward(*args(_gp(mode=2))) == ERR_DIM
    assert lib.pilco_mm_forward(*args(_gp(ldk=32))) == ERR_DIM               # ldk < pilco_pad_n(n)
    assert lib.pilco_mm_forward(*args(_gp(iK=FAKE + 8))) == ERR_ALIGN
    assert lib.pilco_mm_forward(*args(_gp(), R=0)) == ERR_DIM
    assert lib.pilco_mm_forward(*args(_gp(), wsb=16)) == ERR_WS
    assert lib.pilco_mm_forward(*args(_gp(), ws=FAKE + 8)) == ERR_ALIGN
    g = _gp()
    assert lib.pilco_mm_forward(C.byref(g), 1, None, FAKE, FAKE, FAKE, FAKE, None, FAKE, 1 << 30, None) == ERR_NULL
    need = lib.pilco_mm_workspace_bytes(50, 4, 3, 1)
    assert need > 0 and lib.pilco_mm_forward(*args(_gp(), wsb=need - 8)) == ERR_WS


def test_closed_form_argument_validation():
    assert lib.pilco_squash_sin(0, 1, FAKE, FAKE, FAKE, FAKE, FAKE, FAKE, None) == ERR_DIM
    assert lib.pilco_squash_sin(2, 1, None, FAKE, FAKE, FAKE, FAKE, FAKE, None) == ERR_NULL
    assert lib.pilco_linear_action(17, 1, 1, FAKE, 0, FAKE, 0, FAKE, FAKE, FAKE, FAKE, FAKE, None) == ERR_DIM
    assert lib.pilco_exp_reward(3, 1, FAKE, None, FAKE, FAKE, FAKE, None, None, None) == ERR_NULL
    assert lib.pilco_box_risk(3, 1, None, FAKE, FAKE, FAKE, None, None, None) == ERR_NULL
    assert lib.pilco_box_risk(0, 1, FAKE, FAKE, FAKE, FAKE, None, None, None) == ERR_DIM
    assert lib.pilco_box_risk(3, 0, FAKE, FAKE, FAKE, FAKE, None, None, None) == ERR_DIM


def test_rollout_argument_validation():
    fwd = lambda ro: lib.pilco_rollout_forward(C.byref(ro), None)
    assert lib.pilco_rollout_forward(None, None) == ERR_NULL
    assert fwd(_rollout()) == ERR_WS                                       # valid description, no workspace
    assert lib.pilco_rollout_workspace_bytes(C.byref(_rollout())) > 0
    assert fwd(_rollout(kind=7)) == ERR_UNSUP
    assert fwd(_rollout(n_rewards=0)) == ERR_DIM and fwd(_rollout(n_rewards=9)) == ERR_DIM
    assert fwd(_rollout(reward_kind=9)) == ERR_UNSUP
    assert fwd(_rollout(channel=5)) == ERR_UNSUP
    assert fwd(_rollout(reward_kind=_lib.REWARD_BOX, channel=_lib.CHANNEL_MULT)) == ERR_WS     # accepted kinds reach the size check
    ro = _rollout(); ro.pol.U = 2                                          # Ds + U != dyn.D
    assert fwd(ro) == ERR_DIM
    ro = _rollout(); ro.rewards[0].t = None                                # exp reward needs its target
    assert fwd(ro) == ERR_NULL
    ro = _rollout(); ro.traj_S = None
    assert fwd(ro) == ERR_NULL
    ro = _rollout(); ro.ws_bytes = 1 << 30; ro.ws = FAKE + 8
    assert fwd(ro) == ERR_ALIGN
    ro = _rollout(kind=_lib.POLICY_RBF)                                    # RBF policy: its GP must be mode 1 with D=Ds, E=U
    ro.pol.rbf = _gp(n=10, D=3, E=1, mode=0)
    assert fwd(ro) == ERR_DIM
    g = _lib.RolloutGrad()
    assert lib.pilco_rollout_backward(C.byref(_rollout()), None, None) == ERR_NULL
    assert lib.pilco_rollout_backward(C.byref(_rollout()), C.byref(g), None) == ERR_NULL       # no backward workspace


def test_factorize_argument_validation():
    f = lambda n, D, E, B, X=FAKE, wsb=1 << 30: lib.pilco_gp_factorize(n, D, E, B, X, 0, FAKE, 0, FAKE, 0, FAKE, 0, FAKE, 0,
                                                                      FAKE, 64, FAKE, None, FAKE, wsb, None)
    assert f(50, 4, 3, 1, X=None) == ERR_NULL
    assert f(0, 4, 3, 1) == ERR_DIM and f(50, 17, 3, 1) == ERR_DIM and f(50, 4, 3, 0) == ERR_DIM
    assert f(50, 4, 3, 1, wsb=8) == ERR_WS
