"""CPU tests of the time-varying linear policy (pilco_rollout_scheduled_*, DESIGN.md section 27): the torch oracle
(tests/action_reward_oracle.py's cascade under step_action) against central differences and, with a constant
schedule, against the cascade under the stationary policy;
and the library side that needs no GPU: exported symbols, the pilco_policy_schedule layout, status codes and their
order on fake descriptors, workspace sizes, the new kernel's register budget, and the Python refusals raised before
any device work."""
import ctypes
import os
import re
import subprocess

import numpy as np
import pytest
import torch

import action_reward_oracle as aro
import particle_grad_oracle as pgo
from oracle import torch_port as tp
from abi_fakes import ERR_DIM, ERR_NULL, ERR_UNSUP, ERR_WS, FAKE, _rollout
from util import CUOBJDUMP, ROOT, make_gp_problem, sass

T = pgo.T


def _problem(Ds=2, U=1, H=3, dims=(), seed=4):
    Dh = Ds + len(dims)
    X, Y, ell, sf2, sn2 = make_gp_problem(30, Dh + U, Ds, seed=seed)
    rng = np.random.RandomState(seed)
    Ws, bs = 0.4 * rng.randn(H, U, Dh), 0.3 * rng.randn(H, U)
    maxa = 0.8 + rng.rand(U)
    B = rng.randn(Ds, Ds)
    terms = [dict(kind=0, coef=1.0, W=np.diag(0.5 + rng.rand(Ds)), t=0.3 * rng.randn(Ds))]
    return aro.dynamics(X, 0.1 * Y, ell, sf2, sn2), Ws, bs, maxa, terms, X[0, :Ds], 0.05 * B @ B.T + 0.02 * np.eye(Ds)


@pytest.mark.parametrize("dims,v", [((), None), ((1,), [0.01, 0.02])])
def test_oracle_gradient_matches_central_differences(dims, v):
    dyn, Ws, bs, maxa, terms, m0, S0 = _problem(dims=dims)
    H = Ws.shape[0]
    Wt, bt = T(Ws).requires_grad_(), T(bs).requires_grad_()
    out = aro.mm_rollout(dyn, aro.step_action(Wt, bt, maxa), terms, m0, S0, H, angle_dims=list(dims) or None, v=v)
    gW, gb = torch.autograd.grad(out["reward"], (Wt, bt))
    f = lambda W, b: float(aro.mm_rollout(dyn, aro.step_action(T(W), T(b), maxa), terms, m0, S0, H,
                                          angle_dims=list(dims) or None, v=v)["reward"])
    h = 1e-6
    for t in range(H):                                    # every step has its own derivative
        e = np.zeros_like(bs); e[t, 0] = h
        fd = (f(Ws, bs + e) - f(Ws, bs - e)) / (2 * h)
        assert abs(fd - float(gb[t, 0])) <= 1e-7 * max(1.0, abs(fd)), (t, fd, float(gb[t, 0]))
        e = np.zeros_like(Ws); e[t, 0, 1] = h
        fd = (f(Ws + e, bs) - f(Ws - e, bs)) / (2 * h)
        assert abs(fd - float(gW[t, 0, 1])) <= 1e-7 * max(1.0, abs(fd)), (t, fd, float(gW[t, 0, 1]))


def test_constant_schedule_is_the_stationary_oracle():
    dyn, Ws, bs, maxa, terms, m0, S0 = _problem()
    H = Ws.shape[0]
    W, b = Ws[0], bs[0]
    sched = aro.mm_rollout(dyn, aro.step_action(T(np.repeat(W[None], H, 0)), T(np.repeat(b[None], H, 0)), maxa), terms,
                           m0, S0, H)
    act = lambda m, s: tp.linear_action(T(W), T(b).reshape(1, -1), m, s, T(maxa)[None])
    ref = aro.mm_rollout(dyn, act, terms, T(m0), T(S0), H)
    for k in ("traj_m", "traj_S", "reward", "step_reward"):
        assert torch.equal(sched[k], ref[k]), k


NEW = ("pilco_rollout_scheduled_workspace_bytes", "pilco_rollout_scheduled_forward",
       "pilco_rollout_scheduled_bwd_workspace_bytes", "pilco_rollout_scheduled_backward")


def test_library_exports_the_entry_points():
    from pilco_b200 import _lib
    for name in NEW:
        assert hasattr(_lib.lib, name) and name in _lib.SIGNATURES
    header = open(os.path.join(ROOT, "include", "pilco_b200.h")).read()
    assert all(name + "(" in header for name in NEW)


def test_schedule_layout(tmp_path):
    from pilco_b200 import _lib
    src = tmp_path / "sch_layout.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "%s"\nint main(void) { printf("%%zu %%zu %%zu\\n", '
                   'sizeof(pilco_policy_schedule), offsetof(pilco_policy_schedule, W_ts), '
                   'offsetof(pilco_policy_schedule, b_ts)); return 0; }\n' % os.path.join(ROOT, "include", "pilco_b200.h"))
    exe = str(tmp_path / "sch_layout")
    subprocess.check_call(["gcc", "-o", exe, str(src)])
    size, ow, ob = map(int, subprocess.check_output([exe], text=True).split())
    assert (ctypes.sizeof(_lib.PolicySchedule), _lib.PolicySchedule.W_ts.offset, _lib.PolicySchedule.b_ts.offset) \
        == (size, ow, ob) == (16, 0, 8)


def test_new_kernel_does_not_spill():
    nvcc = "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not installed")
    res = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas", "-v",
                          "-cubin", "-o", os.devnull, os.path.join(ROOT, "pilco_b200", "csrc", "rollout_bwd.cu")],
                         capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    props = dict(re.findall(r"Function properties for (\S+)\n\s*(.*)", res.stderr))
    name = next(n for n in props if "rb_sched_grad_kernel" in n)
    assert "0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads" in props[name], props[name]
    if os.path.exists(CUOBJDUMP):
        text = sass("rb_sched_grad_kernel")
        assert len(text) == 1 and not any(re.search(r"\b(STL|LDL)\b", t) for t in text.values())


def _sch(W_ts, b_ts):
    from pilco_b200 import _lib
    return _lib.PolicySchedule(W_ts, b_ts)


def test_status_codes_and_their_order():
    """every rejected call returns before it enqueues anything (the fake pointers are never dereferenced): the noisy
    call's description codes, then a negative stride, then an RBF policy under an active schedule, then the workspace"""
    from pilco_b200 import _lib
    lib, C = _lib.lib, ctypes
    g = _lib.RolloutGrad()
    g.gW = g.gb = g.ws = FAKE
    fwd = lambda ro, s: lib.pilco_rollout_scheduled_forward(C.byref(ro), None, None, None, s and C.byref(s), None)
    bwd = lambda ro, s: lib.pilco_rollout_scheduled_backward(C.byref(ro), None, None, None, s and C.byref(s),
                                                             C.byref(g), None)
    active = _sch(3, 1)
    for call in (fwd, bwd):
        nul = _rollout()
        nul.m0 = None
        assert call(nul, _sch(-1, 0)) == ERR_NULL                       # the description first
        assert call(_rollout(), _sch(-1, 0)) == ERR_DIM
        assert call(_rollout(), _sch(0, -1)) == ERR_DIM
        rbf = _rollout()
        rbf.pol.kind = _lib.POLICY_RBF                                  # an RBF description missing its GP fails first
        assert call(rbf, active) == call(rbf, None) not in (ERR_UNSUP, 0)
    ro = _rollout()
    assert fwd(ro, active) == ERR_WS                                    # then the workspace
    assert fwd(ro, None) == ERR_WS and fwd(ro, _sch(0, 0)) == ERR_WS
    ro.ws_bytes = lib.pilco_rollout_scheduled_workspace_bytes(C.byref(ro), None, None, None, C.byref(active))
    g.gW = None                                                         # (so that no call passes validation)
    g.ws_bytes = lib.pilco_rollout_scheduled_bwd_workspace_bytes(C.byref(ro), None, None, None, None)
    assert bwd(ro, None) == ERR_NULL and bwd(ro, active) == ERR_WS      # the per-step slots come after
    g.ws_bytes = lib.pilco_rollout_scheduled_bwd_workspace_bytes(C.byref(ro), None, None, None, C.byref(active))
    assert bwd(ro, active) == ERR_NULL


def test_rbf_policy_under_an_active_schedule_is_unsupported():
    """a valid RBF description: the inactive schedule is the noisy call, an active one PILCO_ERR_UNSUPPORTED before the
    workspace"""
    from pilco_b200 import _lib
    from abi_fakes import _gp
    lib, C = _lib.lib, ctypes
    ro = _rollout()
    ro.pol.kind = _lib.POLICY_RBF
    ro.pol.rbf = _gp(n=20, D=3, E=1, mode=1, iK=None, ldk=0)
    base = lib.pilco_rollout_noisy_forward(C.byref(ro), None, None, None, None)
    assert base == ERR_WS
    assert lib.pilco_rollout_scheduled_forward(C.byref(ro), None, None, None, C.byref(_sch(0, 0)), None) == ERR_WS
    for s in (_sch(3, 0), _sch(0, 1)):
        assert lib.pilco_rollout_scheduled_forward(C.byref(ro), None, None, None, C.byref(s), None) == ERR_UNSUP


def test_workspace_sizes():
    from pilco_b200 import _lib
    lib, C = _lib.lib, ctypes
    ro = _rollout()
    ang = _lib.Angles()
    ang.A, ang.dims[0] = 0, 0
    nz = _lib.ObsNoise()
    ex = _lib.Exploration(0.5, None)
    for a, e, n in ((None, None, None), (None, C.byref(ex), None), (None, None, C.byref(nz)), (C.byref(ang), C.byref(ex), C.byref(nz))):
        fw = lib.pilco_rollout_noisy_workspace_bytes(C.byref(ro), a, e, n)
        bw = lib.pilco_rollout_noisy_bwd_workspace_bytes(C.byref(ro), a, e, n)
        for s in (None, _sch(0, 0)):                                    # inactive: the noisy call's sizes
            assert lib.pilco_rollout_scheduled_workspace_bytes(C.byref(ro), a, e, n, s and C.byref(s)) == fw
            assert lib.pilco_rollout_scheduled_bwd_workspace_bytes(C.byref(ro), a, e, n, s and C.byref(s)) == bw
        s = _sch(3, 1)
        assert lib.pilco_rollout_scheduled_workspace_bytes(C.byref(ro), a, e, n, C.byref(s)) == fw
        R, H, U, Dh = ro.R, ro.H, ro.pol.U, ro.pol.Ds
        pad = lambda k: (k + 1) & ~1
        assert (lib.pilco_rollout_scheduled_bwd_workspace_bytes(C.byref(ro), a, e, n, C.byref(s))
                == bw + 8 * (pad(H * R * U * Dh) + pad(H * R * U)))
        assert lib.pilco_rollout_scheduled_bwd_workspace_bytes(C.byref(ro), a, e, n, C.byref(_sch(-3, 1))) == 0
        assert lib.pilco_rollout_scheduled_workspace_bytes(C.byref(ro), a, e, n, C.byref(_sch(3, -1))) == 0
    for R, H in ((0, 5), (2, -1)):
        ro.R, ro.H = R, H
        assert lib.pilco_rollout_scheduled_workspace_bytes(C.byref(ro), None, None, None, C.byref(_sch(3, 1))) == 0
        assert lib.pilco_rollout_scheduled_bwd_workspace_bytes(C.byref(ro), None, None, None, C.byref(_sch(3, 1))) == 0


def test_python_refusals_before_device_work():
    """the engine and the class refuse a schedule where it does not apply, before any allocation"""
    from pilco_b200 import engine, _lib, controllers
    spec = controllers.TimeVaryingLinearController(3, 1, 4).policy_spec()
    rbf = dict(kind=_lib.POLICY_RBF, Ds=3, U=1, gp=None)
    with pytest.raises(ValueError, match="RBF"):
        engine.RolloutPlan(None, rbf, [], np.zeros(3), np.eye(3), 4, schedule=True)
    with pytest.raises(ValueError, match="fewer than"):
        engine.RolloutPlan(None, spec, [], np.zeros(3), np.eye(3), 5, schedule=True)
    with pytest.raises(ValueError, match="schedule=True"):
        engine.RolloutPlan(None, spec, [], np.zeros(3), np.eye(3), 4)
    with pytest.raises(ValueError, match="ParticlePlan"):
        engine.ParticlePlan(None, spec, [], 10, 4)
    with pytest.raises(ValueError, match="ConsistentGradPlan"):
        engine.ConsistentGradPlan(None, spec, [], 10, 4)
    with pytest.raises(ValueError, match="particles_rollout"):
        engine.particles_rollout(None, spec, [], np.zeros((10, 3)), np.zeros((10, 4, 3)))


def test_controller_flat_layout_and_shift():
    from pilco_b200 import controllers
    np.random.seed(0)
    c = controllers.TimeVaryingLinearController(3, 2, 4, feedback=True)
    assert c.get_flat().shape == (4 * 2 * 3 + 4 * 2,)
    f = np.arange(32.0)
    c.set_flat(f)
    assert np.array_equal(c.get_flat(), f)
    spec = c.policy_spec(np.stack([f, 2 * f]))
    assert spec["W"].shape == (2, 4, 2, 3) and spec["b"].shape == (2, 4, 2) and spec["schedule"]
    c.shift()
    assert np.array_equal(np.asarray(c.b), np.concatenate([f[24:].reshape(4, 2)[1:], f[24:].reshape(4, 2)[-1:]]))
    ol = controllers.TimeVaryingLinearController(3, 2, 4, feedback=False)
    assert ol.get_flat().shape == (8,) and not np.any(np.asarray(ol.W)) and [p.name for p in ol.trainable_parameters] == ["b"]
    ol.randomize()
    assert not np.any(np.asarray(ol.W)) and np.all(np.abs(np.asarray(ol.b)) < 1.0)
    g = ol.flat_grad(np.ones((2, 2, 3)), np.ones((2, 2)))               # a 2-step rollout: steps 2, 3 get 0
    assert np.array_equal(g, np.r_[np.ones(4), np.zeros(4)])
