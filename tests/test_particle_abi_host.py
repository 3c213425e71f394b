"""The status of every particle rollout call and the bytes of every particle size query over a grid of fake
descriptions, against tests/golden/particle_abi.npz (tests/golden/make_particle_abi.py).  The grid applies one defect,
and every pair of defects that can coexist, to valid descriptions of both policy kinds, unbatched and batched, H in
{0, 1, 5}, state, joint and multiplicative terms, with and without angles, measurement noise and exploration, so each
call's order of precedence is pinned and not only its single codes.  No call passes its workspace check: the
workspace is 0 bytes, or 8 bytes short of the size the query reports (after that size is checked against the golden)."""
import itertools
import os

import numpy as np

from pilco_b200 import _lib
from pilco_b200._lib import lib
from abi_fakes import (ERR_ALIGN, ERR_DIM, ERR_NULL, ERR_UNSUP, ERR_WS, FAKE, PT_MAX_P, _angles, _batched, _grad,
                       _noise, _particles)
from util import _ref

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "particle_abi.npz")
MISMATCH = 99           # status of a call not made because its query disagreed with the golden

# (rollout call, its size query, the arguments after pr: a = angles, n = noise, x = exploration, R, g = gradient)
CALLS = [
    ("pilco_particles_rollout", "pilco_particles_workspace_bytes", ""),
    ("pilco_particles_rollout_consistent", "pilco_particles_consistent_workspace_bytes", ""),
    ("pilco_particles_rollout_grad", "pilco_particles_grad_workspace_bytes", "g"),
    ("pilco_particles_rollout_batch_grad", "pilco_particles_batch_grad_workspace_bytes", "Rg"),
    ("pilco_particles_rollout_consistent_grad", "pilco_particles_consistent_grad_workspace_bytes", "Rg"),
    ("pilco_particles_rollout_score_grad", "pilco_particles_score_grad_workspace_bytes", "Rg"),
    ("pilco_particles_angles_rollout", "pilco_particles_angles_workspace_bytes", "a"),
    ("pilco_particles_angles_consistent_rollout", "pilco_particles_angles_consistent_workspace_bytes", "a"),
    ("pilco_particles_angles_batch_grad_rollout", "pilco_particles_angles_batch_grad_workspace_bytes", "aRg"),
    ("pilco_particles_angles_consistent_grad_rollout", "pilco_particles_angles_consistent_grad_workspace_bytes", "aRg"),
    ("pilco_particles_angles_score_grad_rollout", "pilco_particles_angles_score_grad_workspace_bytes", "aRg"),
    ("pilco_particles_noisy_rollout", "pilco_particles_noisy_workspace_bytes", "an"),
    ("pilco_particles_noisy_consistent_rollout", "pilco_particles_noisy_consistent_workspace_bytes", "an"),
    ("pilco_particles_noisy_batch_grad_rollout", "pilco_particles_noisy_batch_grad_workspace_bytes", "anRg"),
    ("pilco_particles_noisy_consistent_grad_rollout", "pilco_particles_noisy_consistent_grad_workspace_bytes", "anRg"),
    ("pilco_particles_noisy_score_grad_rollout", "pilco_particles_noisy_score_grad_workspace_bytes", "anRg"),
    ("pilco_particles_explore_batch_grad_rollout", "pilco_particles_explore_batch_grad_workspace_bytes", "anxRg"),
    ("pilco_particles_explore_consistent_grad_rollout", "pilco_particles_explore_consistent_grad_workspace_bytes",
     "anxRg"),
    ("pilco_particles_consistent_score_grad_rollout", "pilco_particles_consistent_score_grad_workspace_bytes", "anRg"),
]
# every status each call can return without a device (a launch error needs one)
CODES = {ERR_NULL, ERR_DIM, ERR_UNSUP, ERR_ALIGN, ERR_WS}


class Case:
    def __init__(self, pr, ang=None, nz=None, ex=None, R=1, g=None, short=False):
        self.pr, self.ang, self.nz, self.ex, self.R, self.g, self.short = pr, ang, nz, ex, R, g, short


def _term(pr, k, kind, channel=0, t=FAKE):
    pr.rewards[k].kind, pr.rewards[k].channel, pr.rewards[k].coef = kind, channel, 1.0
    pr.rewards[k].W, pr.rewards[k].t = FAKE, t


def base(kind, batched, H, terms, angles, noise, explore, P=1000):
    """a description every call accepts up to its workspace: E = 3 state dimensions, U = 1, two reward terms"""
    pr = (_batched if batched else _particles)(kind, P=P, H=H)
    if angles:                                          # one angle: the policy takes phi(x), 4 inputs
        pr.pol.Ds, pr.dyn.D = 4, 5
        if kind == _lib.POLICY_RBF:
            pr.pol.rbf.D = 4
    pr.n_rewards = 2
    if terms == "state":
        _term(pr, 1, _lib.REWARD_LINEAR, t=None)
    elif terms == "joint":
        _term(pr, 1, _lib.REWARD_EXP_SA)
    else:
        _term(pr, 1, _lib.REWARD_BOX, _lib.CHANNEL_MULT, t=None)
    return Case(pr, _angles(0) if angles else None, _noise() if noise else None,
                _lib.Exploration(0.5, FAKE) if explore else None, 3 if batched else 1, _grad())


def _strides(c, sign):
    if c.pr.pol.kind == _lib.POLICY_LINEAR:
        c.pr.pol.W_bs, c.pr.pol.b_bs = sign * 3, sign * 1
    else:
        c.pr.pol.rbf.X_bs, c.pr.pol.rbf.ell_bs = sign * 60, sign * 3


def _set(obj, **kw):
    if obj is not None:
        for k, v in kw.items():
            setattr(obj, k, v)


def _nu_null(c):
    c.nz = c.nz if c.nz is not None else _noise()
    c.nz.nu = None


def _a_neg(c):
    c.ang = _angles()
    c.ang.A = -1


def _ws(c, ws):
    _set(c.pr, ws=ws)
    _set(c.g, ws=ws)


def _box_add(c):
    _term(c.pr, 1, _lib.REWARD_BOX, _lib.CHANNEL_ADD, t=None)


# (name, field, mutation), applied in this order; two defects coexist when their fields differ
DEFECTS = [
    ("x0_null", "x0", lambda c: _set(c.pr, x0=None)),
    ("value_null", "g.value", lambda c: _set(c.g, value=None)),
    ("rbf_out_null", "g.gXc", lambda c: _set(c.g, gXc=None)),
    ("dyn_mode", "dyn.mode", lambda c: _set(c.pr.dyn, mode=1)),
    ("ldk_odd", "dyn.ldk", lambda c: _set(c.pr.dyn, ldk=65)),
    ("iK_misaligned", "dyn.iK", lambda c: _set(c.pr.dyn, iK=FAKE + 8)),
    ("width", "dyn.D", lambda c: _set(c.pr.dyn, D=c.pr.dyn.D + 1)),
    ("strides", "bs", lambda c: _strides(c, 1)),
    ("neg_stride", "bs", lambda c: _strides(c, -1)),
    ("R0", "R", lambda c: setattr(c, "R", 0)),
    ("R65536", "R", lambda c: setattr(c, "R", 65536)),
    ("R_over", "R", lambda c: setattr(c, "R", PT_MAX_P // c.pr.P + 1)),
    ("rewards0", "n_rewards", lambda c: _set(c.pr, n_rewards=0)),
    ("rewards9", "n_rewards", lambda c: _set(c.pr, n_rewards=9)),
    ("kind_unknown", "r0.kind", lambda c: _set(c.pr.rewards[0], kind=99)),
    ("channel_bad", "r0.channel", lambda c: _set(c.pr.rewards[0], channel=7)),
    ("t_null", "r0.t", lambda c: _set(c.pr.rewards[0], t=None)),
    ("box_add", "r1", _box_add),
    ("A0", "ang", lambda c: setattr(c, "ang", _angles())),
    ("ang_repeat", "ang", lambda c: setattr(c, "ang", _angles(1, 1))),
    ("ang_range", "ang", lambda c: setattr(c, "ang", _angles(3))),
    ("A_gt_E", "ang", lambda c: setattr(c, "ang", _angles(0, 1, 2, 0))),
    ("A_neg", "ang", _a_neg),
    ("rbf_D", "rbf.D", lambda c: _set(c.pr.pol.rbf, D=c.pr.pol.rbf.D + 1)),
    ("var_nan", "nz.var", lambda c: setattr(c, "nz", _noise((0.01, float("nan"), 0.03)))),
    ("var_neg", "nz.var", lambda c: setattr(c, "nz", _noise((0.01, 0.02, -0.5)))),
    ("var_inf", "nz.var", lambda c: setattr(c, "nz", _noise((float("inf"), 0.02, 0.03)))),
    ("nu_null", "nz.nu", _nu_null),
    ("ex_none", "ex", lambda c: setattr(c, "ex", None)),
    ("ex_b0", "ex", lambda c: setattr(c, "ex", _lib.Exploration(0.0, None))),
    ("ex_b0_step_var", "ex", lambda c: setattr(c, "ex", _lib.Exploration(0.0, FAKE))),
    ("ex_nan", "ex", lambda c: setattr(c, "ex", _lib.Exploration(float("nan"), FAKE))),
    ("ex_inf", "ex", lambda c: setattr(c, "ex", _lib.Exploration(float("inf"), None))),
    ("P1", "P", lambda c: _set(c.pr, P=1)),
    ("ws_null", "ws", lambda c: _ws(c, None)),
    ("ws_misaligned", "ws", lambda c: _ws(c, FAKE + 8)),
    ("ws_short", "ws", lambda c: setattr(c, "short", True)),
    ("g_null", "g", lambda c: setattr(c, "g", None)),
    ("pr_null", "pr", lambda c: setattr(c, "pr", None)),
]

BASES = list(itertools.product((_lib.POLICY_LINEAR, _lib.POLICY_RBF), (False, True), (0, 1, 5),
                               ("state", "joint", "mult"), (False, True), (False, True), (False, True)))


def cases():
    """(names, Case): every base without a defect and with each single defect, every coexisting pair of defects on
    the bases in turn, and the sizes past size_t and past 2^31 - 1 CTAs per step"""
    out = []
    for b in BASES:
        out.append(("", base(*b)))
        for i in range(len(DEFECTS)):
            c = base(*b)
            DEFECTS[i][2](c)
            out.append((DEFECTS[i][0], c))
    pairs = [(i, j) for i, j in itertools.combinations(range(len(DEFECTS)), 2) if DEFECTS[i][1] != DEFECTS[j][1]]
    for k, (i, j) in enumerate(pairs):
        c = base(*BASES[(7 * k) % len(BASES)])
        DEFECTS[i][2](c)
        DEFECTS[j][2](c)
        out.append((DEFECTS[i][0] + "+" + DEFECTS[j][0], c))
    for H in ((1 << 31) - 1, 131072):                   # size_t overflow; P H / 128 CTAs > 2^31 - 1 without it
        for kind, angles, noise, explore in itertools.product((_lib.POLICY_LINEAR, _lib.POLICY_RBF), (False, True),
                                                              (False, True), (False, True)):
            out.append(("H%d" % H, base(kind, False, H, "joint", angles, noise, explore, P=PT_MAX_P)))
    return out


def _args(c, sig):
    m = {"a": lambda: _ref(c.ang), "n": lambda: _ref(c.nz), "x": lambda: _ref(c.ex), "R": lambda: c.R,
         "g": lambda: _ref(c.g)}
    return [_ref(c.pr)] + [m[s]() for s in sig]


def run(cs, want=None):
    """status [case, call] and bytes [case, call]; with want (the golden's bytes) a call whose query disagrees is not
    made (status MISMATCH), so a short workspace is always short of the call's own layout"""
    status = np.zeros((len(cs), len(CALLS)), np.int8)
    size = np.zeros((len(cs), len(CALLS)), np.uint64)
    for i, c in enumerate(cs):
        for j, (call, query, sig) in enumerate(CALLS):
            need = getattr(lib, query)(*_args(c, sig.replace("g", "")))
            size[i, j] = need
            if want is not None and need != int(want[i, j]):
                status[i, j] = MISMATCH
                continue
            short = need - 8 if c.short and need >= 8 else 0
            _set(c.pr, ws_bytes=short)
            _set(c.g, ws_bytes=short)
            status[i, j] = getattr(lib, call)(*_args(c, sig), None)
            _set(c.pr, ws_bytes=0)
            _set(c.g, ws_bytes=0)
    return status, size


def record():
    named = cases()
    status, size = run([c for _, c in named])
    return dict(names=np.array([n for n, _ in named]), calls=np.array([c[0] for c in CALLS]), status=status, size=size)


def test_status_and_sizes_are_the_golden():
    gold = np.load(GOLDEN)
    named = cases()
    assert list(gold["names"]) == [n for n, _ in named]
    assert list(gold["calls"]) == [c[0] for c in CALLS]
    status, size = run([c for _, c in named], gold["size"])
    bad = np.argwhere((size != gold["size"]) | (status != gold["status"]))
    assert len(bad) == 0, "\n".join("%s %s: status %d (golden %d), bytes %d (golden %d)" % (
        named[i][0], CALLS[j][0], status[i, j], gold["status"][i, j], size[i, j], gold["size"][i, j])
        for i, j in bad[:20])


def test_golden_has_every_status_of_every_call():
    gold = np.load(GOLDEN)
    for j, (call, _, _) in enumerate(CALLS):
        assert set(gold["status"][:, j].tolist()) == CODES, call
    assert (gold["size"] > 0).any(axis=0).all() and (gold["size"] == 0).any(axis=0).all()


def test_every_engine_row_binds_its_argtypes():
    """every row of the engine's PARTICLE_ENTRY_POINTS: the size query is its rollout's pair, and the arguments
    engine.particle_args binds follow each one's argtypes, one per argtype (the rollout's final stream left out): each
    struct by reference to the slot of its type (NULL without one), R for the c_int and value for a c_dp"""
    import ctypes as C
    from pilco_b200 import engine
    structs = {t: t._type_ for t in engine._SLOTS if isinstance(getattr(t, "_type_", None), type)}
    slots = {engine._SLOTS[t]: s() for t, s in structs.items()}
    slots.update(R=7, value=FAKE)
    assert len(engine.PARTICLE_ENTRY_POINTS) == 32
    for key, (run, query) in engine.PARTICLE_ENTRY_POINTS.items():
        assert run.endswith("_rollout") and query == run[:-len("rollout")] + "workspace_bytes", key
        for name in (run, query):
            res, types = _lib.SIGNATURES[name]
            if res is C.c_int:
                assert types[-1] is _lib.c_dp, name
                types = types[:-1]
            else:
                assert res is C.c_size_t and _lib.c_dp not in types, name
            args = engine.particle_args(name, **slots)
            assert len(args) == len(types) and types[0] is C.POINTER(_lib.Particles), name
            for a, t in zip(args, types):
                want = {C.c_int: 7, _lib.c_dp: FAKE}.get(t)
                assert (a == want) if want is not None else (a._obj is slots[engine._SLOTS[t]]), (name, t)
            bare = engine.particle_args(name, R=7, value=FAKE)
            assert all(a is None for a, t in zip(bare, types) if t in structs), name
