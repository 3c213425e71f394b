"""CPU tests of the time-varying linear policy in the particle rollouts (pilco_particles_scheduled_*, DESIGN.md section
28): the shared oracles under a schedule (tests/particle_schedule_oracle.py; a constant schedule against the stationary
policy, the torch gradient per step against central differences of the numpy rollout), and the library side that needs no GPU: exported symbols,
status codes and their order on fake descriptors, workspace sizes, the new kernels' register budget, and the Python
refusals raised before any device work."""
import os
import re
import subprocess

import numpy as np
import pytest

import particle_grad_oracle as pgo
import particle_oracle as po
import particle_schedule_oracle as pso
from abi_fakes import ERR_DIM, ERR_NULL, ERR_UNSUP, ERR_WS, FAKE, SAMPLER, _batched, _grad, _particles, entry_call
from particle_cases import _problem, _terms
from pilco_b200 import _lib, engine
from pilco_b200._lib import lib
from util import CUOBJDUMP, ROOT, sass_named

SAMPLERS = [(False, "forward"), (True, "forward"), (False, "pathwise"), (True, "pathwise"), (False, "score"),
            (True, "score"), ("resampled", "forward"), ("resampled", "pathwise")]


def _case(H=3, P=7, seed=3, angle_dims=None):
    """a small host problem (Ds = 3 raw state dimensions, U = 1) with a random schedule W [H,U,Dh], b [H,U]"""
    A = len(angle_dims or ())
    dyn, rng = _problem(seed, Ds=3 + A) if A else _problem(seed)
    if A:                                               # the GP's outputs are the raw state
        dyn = dict(dyn, ell=dyn["ell"][:3], sf2=dyn["sf2"][:3], iK=dyn["iK"][:3], beta=dyn["beta"][:3])
    Dh = 3 + A
    pol = dict(kind=_lib.POLICY_LINEAR, squash=True, maxa=np.array([1.2]), W=0.5 * rng.randn(H, 1, Dh),
               b=rng.randn(H, 1))
    x0, eps, nu = 0.3 * rng.randn(P, 3), rng.randn(P, H, 3), rng.randn(P, H, 3)
    return dyn, pol, _terms(3), x0, eps, nu


def _constant(pol, t=0):
    H = pol["W"].shape[0]
    W, b = pol["W"][t], pol["b"][t]
    return dict(pol, W=np.repeat(W[None], H, 0), b=np.repeat(b[None], H, 0)), dict(pol, W=W, b=b)


@pytest.mark.parametrize("dims,v", [(None, None), ([1], [0.01, 0.02, 0.03])])
def test_constant_schedule_is_the_stationary_oracle(dims, v):
    dyn, pol, terms, x0, eps, nu = _case(angle_dims=dims)
    sched, stat = _constant(pol)
    nu = nu if v is not None else None
    for roll in (po.particle_rollout, po.consistent_rollout):
        with pso.schedule(sched):
            a = roll(dyn, sched, terms, x0, eps, 1.5, angle_dims=dims, nu=nu, v=v)
        b = roll(dyn, stat, terms, x0, eps, 1.5, angle_dims=dims, nu=nu, v=v)
        assert all(np.array_equal(p, q) for p, q in zip(a, b))
    for vg in (pgo.value_and_grad, pgo.consistent_value_and_grad):
        with pso.schedule(sched):
            va, ga = vg(dyn, sched, terms, x0, eps, 1.5, angle_dims=dims, nu=nu, v=v)[:2]
        vb, gb = vg(dyn, stat, terms, x0, eps, 1.5, angle_dims=dims, nu=nu, v=v)[:2]
        assert va == vb
        for k in ("W", "b"):
            s = ga[k].sum(0)
            assert np.max(np.abs(s - gb[k])) <= 1e-13 * max(1.0, np.max(np.abs(gb[k]))), k
    traj = po.particle_rollout(dyn, stat, terms, x0, eps, 1.5, angle_dims=dims, nu=nu, v=v)[0]
    with pso.schedule(sched):
        ga = pgo.score_grad(dyn, sched, terms, traj, eps, 1.5, angle_dims=dims, nu=nu, v=v)
    gb = pgo.score_grad(dyn, stat, terms, traj, eps, 1.5, angle_dims=dims, nu=nu, v=v)
    for k in ("W", "b"):
        assert np.max(np.abs(ga[k].sum(0) - gb[k])) <= 1e-13 * max(1.0, np.max(np.abs(gb[k]))), k


def test_oracle_gradient_matches_central_differences():
    """the torch oracle's per-step gradient against central differences of the numpy rollout's mean return"""
    dyn, pol, terms, x0, eps, _ = _case(H=4)
    H = pol["W"].shape[0]
    with pso.schedule(pol):
        value, g = pgo.value_and_grad(dyn, pol, terms, x0, eps, 1.5)

    def f(p):
        with pso.schedule(p):
            return float(po.particle_rollout(dyn, p, terms, x0, eps, 1.5)[4].mean())
    assert abs(value - f(pol)) <= 1e-12 * max(1.0, abs(value))
    h = 1e-6
    for t in range(H):                                  # every step has its own derivative
        for k, idx in (("b", (t, 0)), ("W", (t, 0, 1))):
            e = np.zeros_like(pol[k]); e[idx] = h
            fd = (f(dict(pol, **{k: pol[k] + e})) - f(dict(pol, **{k: pol[k] - e}))) / (2 * h)
            assert abs(fd - g[k][idx]) <= 1e-7 * max(1.0, abs(fd)), (k, idx, fd, g[k][idx])


def _rows(family):
    """(sampler, call) -> (rollout, size query) of the family's rows of engine.PARTICLE_ENTRY_POINTS, the batched
    forward calls (DESIGN.md sections 31 and 33) left out"""
    return {k[1:]: v for k, v in engine.PARTICLE_ENTRY_POINTS.items() if k[0] == family and k[2] != "batch"}


def test_library_exports_the_entry_points():
    header = open(os.path.join(ROOT, "include", "pilco_b200.h")).read()
    new = [n for pair in _rows("scheduled").values() for n in pair]
    assert len(set(new)) == 16 and set(_rows("scheduled")) == {k for k in _rows("plain") if k[0] != "features"}
    for name in new:
        assert hasattr(lib, name) and name in _lib.SIGNATURES and name + "(" in header


def _rs():
    return _lib.ParticlesResample(FAKE, None, None)


def _call(key, pr, sch, g=None, R=3, scheduled=True, query=False):
    """the row (scheduled or plain, ``key``) of engine.PARTICLE_ENTRY_POINTS with NULL angles, noise and exploration"""
    sampler, kind = key
    return entry_call(("scheduled" if scheduled else "plain", SAMPLER[sampler], kind), query, pr=pr, sch=sch, grad=g,
                      R=R, rs=_rs())


def _desc(key, kind=_lib.POLICY_LINEAR):
    return _particles(kind) if key[1] == "forward" else _batched(kind)


@pytest.mark.parametrize("key", SAMPLERS, ids=lambda k: "%s-%s" % k)
def test_status_codes_and_their_order(key):
    """every rejected call returns before it enqueues anything (the fake pointers are never dereferenced): the call's
    own codes up to its workspace, then a negative stride, then an RBF policy under an active schedule, then the
    workspace; an inactive schedule is the call without it"""
    active, neg = _lib.PolicySchedule(3, 1), (_lib.PolicySchedule(-3, 1), _lib.PolicySchedule(0, -1))
    g = _grad()
    assert _call(key, None, neg[0], g) == ERR_NULL
    for field in ("x0", "traj", "ret"):                 # the description's codes come first
        pr = _desc(key); setattr(pr, field, None)
        for s in (None, active) + neg:
            assert _call(key, pr, s, g) == ERR_NULL
    if key[1] != "forward":
        bad = _grad(); bad.gW = None
        assert _call(key, _desc(key), neg[0], bad) == ERR_NULL
        assert _call(key, _desc(key), active, g, R=0) == _call(key, _desc(key), None, g, R=0, scheduled=False) == ERR_DIM
    for s in neg:
        assert _call(key, _desc(key), s, g) == ERR_DIM
        assert _call(key, _desc(key, _lib.POLICY_RBF), s, g) == ERR_DIM
    base = _call(key, _desc(key), None, g, scheduled=False)
    assert base == ERR_WS
    for s in (None, _lib.PolicySchedule(0, 0), active, _lib.PolicySchedule(0, 1), _lib.PolicySchedule(3, 0)):
        assert _call(key, _desc(key), s, g) == ERR_WS
    rbf = _call(key, _desc(key, _lib.POLICY_RBF), None, g, scheduled=False)
    assert rbf == ERR_WS
    assert _call(key, _desc(key, _lib.POLICY_RBF), _lib.PolicySchedule(0, 0), g) == rbf
    for s in (active, _lib.PolicySchedule(0, 1)):
        assert _call(key, _desc(key, _lib.POLICY_RBF), s, g) == ERR_UNSUP


@pytest.mark.parametrize("key", SAMPLERS, ids=lambda k: "%s-%s" % k)
def test_workspace_sizes_are_the_unscheduled_calls(key):
    for kind in (_lib.POLICY_LINEAR, _lib.POLICY_RBF):
        for P, H in ((1000, 5), (7, 0), (300, 12)):
            pr = _desc(key, kind)
            pr.P, pr.H = P, H
            base = _call(key, pr, None, R=3, scheduled=False, query=True)
            assert base > 0
            for s in (None, _lib.PolicySchedule(0, 0), _lib.PolicySchedule(3, 1), _lib.PolicySchedule(0, 1)):
                assert _call(key, pr, s, R=3, query=True) == base
            for s in (_lib.PolicySchedule(-3, 1), _lib.PolicySchedule(3, -1)):
                assert _call(key, pr, s, R=3, query=True) == 0
    pr = _desc(key)
    pr.P = 0
    assert _call(key, pr, _lib.PolicySchedule(3, 1), R=3, query=True) == 0


NEW_KERNELS = ("pg_sched_kernel", "ps_zbar_sched_kernel")


def test_new_kernels_do_not_spill():
    nvcc = "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not installed")
    res = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas", "-v",
                          "-cubin", "-o", os.devnull, os.path.join(ROOT, "pilco_b200", "csrc", "particles.cu")],
                         capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    props = dict(re.findall(r"Function properties for (\S+)\n\s*(.*)", res.stderr))
    for k in NEW_KERNELS:
        name = next(n for n in props if re.search(r"\d%s\d" % k, n))
        assert "0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads" in props[name], (k, props[name])
    if os.path.exists(CUOBJDUMP):
        text = sass_named([k + "5" if k == "pg_sched_kernel" else k + "7" for k in NEW_KERNELS])
        assert len(text) == 2 and not any(re.search(r"\b(STL|LDL)\b", t) for t in text.values())


def test_engine_refusals_before_allocation():
    """dyn is None: every refusal fires before the engine touches the model or the device"""
    from pilco_b200 import controllers
    spec = controllers.TimeVaryingLinearController(3, 1, 4).policy_spec()
    rbf = dict(kind=_lib.POLICY_RBF, Ds=3, U=1, gp=None)
    x0, eps = np.zeros((10, 3)), np.zeros((10, 4, 3))
    for make, what in ((lambda s, H, **kw: engine.ParticlePlan(None, s, [], 10, H, grad=True, **kw), "ParticlePlan"),
                       (lambda s, H, **kw: engine.ConsistentGradPlan(None, s, [], 10, H, **kw), "ConsistentGradPlan"),
                       (lambda s, H, **kw: engine.particles_rollout(None, s, [], x0[:, :], np.zeros((10, H, 3)), **kw),
                        "particles_rollout")):
        with pytest.raises(ValueError, match="RBF"):
            make(rbf, 4, schedule=True)
        with pytest.raises(ValueError, match="fewer than"):
            make(spec, 5, schedule=True)
        with pytest.raises(ValueError, match=what + ".*schedule=True"):
            make(spec, 4)
    with pytest.raises(ValueError, match="schedule=True"):
        engine.particles_rollout(None, spec, [], x0, eps)


def _mpc_pilco(Dh=2, **kw):
    from pilco.models import PILCO
    from pilco.controllers import TimeVaryingLinearController
    rng = np.random.RandomState(0)
    return PILCO((rng.rand(20, 3), 0.1 * rng.rand(20, 2)), controller=TimeVaryingLinearController(Dh, 1, 4), horizon=4,
                 **kw)


def test_class_plan_refusals_before_device_work(monkeypatch):
    """with num_samples: box terms, angle_dims and measurement noise are refused before any device work (a device
    call would fail loudly here)"""
    import torch
    from pilco.rewards import LinearReward
    from safe_pilco_extension.rewards_safe import RiskOfCollision
    from safe_pilco_extension.safe_pilco import SafePILCO
    from pilco.controllers import TimeVaryingLinearController
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)
    rng = np.random.RandomState(1)
    X, Y = rng.rand(30, 5), 0.1 * rng.rand(30, 4)
    sp = SafePILCO((X, Y), controller=TimeVaryingLinearController(4, 1, 4), horizon=4,
                   reward_add=LinearReward(4, np.ones(4)), reward_mult=RiskOfCollision(4, [0.0, 0.1], [0.6, 0.9]),
                   mu=-4.0)
    flat = sp.controller.get_flat().copy()
    with pytest.raises(ValueError, match="box"):
        sp.plan(np.zeros(4), num_samples=16, seed=0)
    assert np.array_equal(sp.controller.get_flat(), flat)
    with pytest.raises(ValueError, match="measurement_noise"):
        _mpc_pilco(measurement_noise=[0.01, 0.01]).plan(np.zeros(2), num_samples=16, seed=0)
    with pytest.raises(ValueError, match="angle_dims"):
        _mpc_pilco(Dh=3, angle_dims=[0]).plan(np.zeros(2), num_samples=16, seed=0)
    with pytest.raises(ValueError, match="num_samples"):
        _mpc_pilco().plan(np.zeros(2), num_samples=0)
