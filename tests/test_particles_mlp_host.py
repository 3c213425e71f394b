"""CPU tests of tanh MLP policies in the particle rollouts (pilco_particles_mlp_*, DESIGN.md section 29): the oracles'
MLP branch against central differences, MlpController's flat layout and point action, and the library side that needs
no GPU: exported symbols and the struct layout, status codes and their order on fake descriptors, workspace sizes,
the new kernels' register budget, and the engine and class refusals raised before any device work."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest
import torch

import particle_grad_oracle as pgo
import particle_mlp_oracle as pmo
import particle_oracle as po
from abi_fakes import ERR_DIM, ERR_NULL, ERR_UNSUP, ERR_WS, FAKE, SAMPLER, _batched, _grad, _particles, entry_call
from particle_cases import _problem, _terms
from pilco_b200 import _lib, controllers, engine
from pilco_b200._lib import lib
from util import CUOBJDUMP, ROOT, sass_named


@pytest.fixture(autouse=True)
def _mlp_oracle():
    """the shared particle oracles serve MLP policy dicts (tests/particle_mlp_oracle.py)"""
    with pmo.mlp_policies():
        yield


def _pol(hidden, squash, seed=3, Ds=3, U=1):
    rng = np.random.RandomState(seed)
    n = engine.mlp_theta_size(Ds, U, hidden)
    return dict(kind=_lib.POLICY_MLP, squash=squash, maxa=np.array([1.2] * U), Ds=Ds, U=U, hidden=hidden,
                theta=0.6 * rng.randn(n))


@pytest.mark.parametrize("hidden", [(5,), (6, 4)])
@pytest.mark.parametrize("squash", [True, False])
def test_oracle_gradient_matches_central_differences(hidden, squash):
    dyn, rng = _problem(3)
    pol, terms = _pol(hidden, squash), _terms(3)
    P, H = 7, 3
    x0, eps = 0.3 * rng.randn(P, 3), rng.randn(P, H, 3)
    val, g = pgo.value_and_grad(dyn, pol, terms, x0, eps, 1.5)
    assert abs(val - float(po.particle_rollout(dyn, pol, terms, x0, eps, 1.5)[4].mean())) <= 1e-12 * max(1, abs(val))
    d = np.random.RandomState(1).randn(pol["theta"].size)
    f = lambda th: float(po.particle_rollout(dyn, dict(pol, theta=th), terms, x0, eps, 1.5)[4].mean())
    h = 1e-6
    fd = (f(pol["theta"] + h * d) - f(pol["theta"] - h * d)) / (2 * h)
    gd = float(np.asarray(g["theta"]).reshape(-1) @ d)
    assert abs(fd - gd) <= 1e-6 * max(abs(gd), 1e-3), (fd, gd)


def test_controller_flat_round_trip_and_point_action():
    np.random.seed(0)
    c = controllers.MlpController(3, 2, hidden=(5, 4), max_action=[1.0, 2.0])
    n = engine.mlp_theta_size(3, 2, (5, 4))
    flat = c.get_flat()
    assert flat.shape == (n,) == (5 * 4 + 4 * 6 + 2 * 5,)
    assert [tuple(A.shape) for A in c.layers] == [(5, 4), (4, 6), (2, 5)]
    assert all(np.all(np.asarray(A.numpy())[:, -1] == 0.0) for A in c.layers)      # randomize(): zero biases
    new = np.random.RandomState(1).randn(n)
    c.set_flat(new)
    assert np.array_equal(c.get_flat(), new)
    spec = c.policy_spec()
    assert spec["kind"] == _lib.POLICY_MLP and spec["hidden"] == (5, 4) and np.array_equal(spec["theta"], new)
    assert c.policy_spec(np.stack([new, new]))["theta"].shape == (2, n)
    x = np.array([[0.3, -0.2, 0.5]])
    M, S, V = c.compute_action(x)
    ref = pmo.action(dict(kind=_lib.POLICY_MLP, squash=True, maxa=np.array([1.0, 2.0]), Ds=3, U=2,
                                hidden=(5, 4), theta=new), x)
    assert np.allclose(M, ref, rtol=0, atol=1e-15) and M.shape == (1, 2)
    assert np.all(np.asarray(S) == 0) and np.all(np.asarray(V) == 0)
    with pytest.raises(ValueError, match="point"):
        c.compute_action(x, 0.1 * np.eye(3))
    k = c.state_key()
    c.set_flat(new + 1.0)
    assert c.state_key() != k
    with pytest.raises(ValueError, match="hidden"):
        controllers.MlpController(3, 1, hidden=(65,))
    with pytest.raises(ValueError, match="hidden"):
        controllers.MlpController(3, 1, hidden=(4, 4, 4))


NAMES = ["pilco_particles_mlp_" + s for s in ("rollout", "consistent_rollout", "resampled_rollout",
                                              "batch_grad_rollout", "consistent_grad_rollout",
                                              "resampled_grad_rollout")]


def test_library_exports_the_entry_points_and_the_struct_layout():
    header = open(os.path.join(ROOT, "include", "pilco_b200.h")).read()
    sizes = [n.replace("_rollout", "_workspace_bytes") for n in NAMES]
    sizes[0] = "pilco_particles_mlp_workspace_bytes"
    for name in NAMES + sizes:
        assert hasattr(lib, name) and name in _lib.SIGNATURES and name + "(" in header, name
    assert "#define PILCO_POLICY_MLP    2" in header and _lib.POLICY_MLP == 2
    # pilco_mlp { int L, width[2]; const double* theta; long long theta_bs; double* gtheta; } on LP64
    assert C.sizeof(_lib.Mlp) == 40
    assert [getattr(_lib.Mlp, f).offset for f in ("L", "width", "theta", "theta_bs", "gtheta")] == [0, 4, 16, 24, 32]


def _mlp(L=2, widths=(8, 6), theta=FAKE, bs=0, gtheta=FAKE):
    return _lib.Mlp(L, (C.c_int * 2)(*widths), theta, bs, gtheta)


KEYS = [(False, "forward"), (True, "forward"), ("resampled", "forward"),
        (False, "pathwise"), (True, "pathwise"), ("resampled", "pathwise")]


def _rs(xi=FAKE):
    return _lib.ParticlesResample(xi, None, None)


def _call(key, pr, mlp, g=None, R=3, query=False, rs="default", ex=None, family="mlp"):
    """row (``family``, ``key``) of engine.PARTICLE_ENTRY_POINTS"""
    sampler, kind = key
    return entry_call((family, SAMPLER[sampler], kind), query, pr=pr, mlp=mlp, grad=g, R=R, ex=ex,
                      rs=_rs() if rs == "default" else rs)


def _desc(key, kind=_lib.POLICY_MLP):
    return _particles(kind) if key[1] == "forward" else _batched(kind)


@pytest.mark.parametrize("key", KEYS, ids=lambda k: "%s-%s" % k)
def test_status_codes_and_their_order(key):
    """every rejected call returns before it enqueues anything (the fake pointers are never dereferenced): the
    description's codes, the MLP's in place of the policy's, R and the gradient's outputs, the sampler's own, then the
    workspace"""
    fwd = key[1] == "forward"
    g = _grad()
    assert _call(key, None, _mlp(), g) == ERR_NULL
    pr = _desc(key); pr.x0 = None
    assert _call(key, pr, None, g) == ERR_NULL                      # the description first
    pr = _desc(key); pr.dyn.D = 9
    assert _call(key, pr, None, g) == ERR_DIM
    for kind in (_lib.POLICY_LINEAR, _lib.POLICY_RBF):              # the MLP calls need PILCO_POLICY_MLP
        assert _call(key, _desc(key, kind), _mlp(), g) == ERR_UNSUP
    pr = _desc(key); pr.pol.kind = 7
    assert _call(key, pr, _mlp(), g) == ERR_UNSUP
    assert _call(key, _desc(key), None, g) == ERR_NULL
    assert _call(key, _desc(key), _mlp(theta=None), g) == ERR_NULL
    for bad in (_mlp(L=0), _mlp(L=3), _mlp(widths=(0, 6)), _mlp(widths=(65, 6)), _mlp(widths=(8, 0)),
                _mlp(widths=(8, 65)), _mlp(bs=-1)):
        assert _call(key, _desc(key), bad, g) == ERR_DIM
    assert _call(key, _desc(key), _mlp(L=1, widths=(8, 0)), g) == ERR_WS      # width[1] unused at L = 1
    pr = _desc(key); pr.pol.squash, pr.pol.max_action = 1, None
    assert _call(key, pr, _mlp(), g) == ERR_NULL                    # then the squash's max_action
    if fwd:
        assert _call(key, _desc(key), _mlp(bs=40), g) == ERR_UNSUP   # a forward call runs one policy
    else:
        assert _call(key, _desc(key), _mlp(bs=200), g) == ERR_WS
        assert _call(key, _desc(key), _mlp(), g, R=0) == ERR_DIM
        assert _call(key, _desc(key), _mlp(gtheta=None), g) == ERR_NULL
        bad = _grad(); bad.value = None
        assert _call(key, _desc(key), _mlp(), bad) == ERR_NULL
        assert _call(key, _desc(key), _mlp(gtheta=None), g, R=0) == ERR_DIM          # R before the outputs
        bad = _grad(); bad.gW = bad.gb = None                       # the linear fields are ignored
        assert _call(key, _desc(key), _mlp(), bad) == ERR_WS
    if key[0] == "resampled":
        assert _call(key, _desc(key), _mlp(), g, rs=None) == ERR_NULL
        assert _call(key, _desc(key), _mlp(), g, rs=_rs(xi=None)) == ERR_NULL
        pr = _desc(key); pr.P = 1
        assert _call(key, pr, _mlp(), g) == ERR_DIM
    assert _call(key, _desc(key), _mlp(), g) == ERR_WS


@pytest.mark.parametrize("key", KEYS, ids=lambda k: "%s-%s" % k)
def test_existing_calls_refuse_the_mlp_kind(key):
    assert _call(key, _desc(key), None, _grad(), family="plain") == ERR_UNSUP


@pytest.mark.parametrize("key", KEYS, ids=lambda k: "%s-%s" % k)
def test_workspace_sizes(key):
    """forward: the linear call's workspace; gradients: more, growing with the widths; 0 exactly where the call
    fails on sizes"""
    for P, H in ((1000, 5), (7, 0), (300, 12)):
        pr = _desc(key)
        pr.P, pr.H = P, H
        m1, m2, m3 = _call(key, pr, _mlp(L=1, widths=(8, 0)), query=True), _call(key, pr, _mlp(), query=True), \
            _call(key, pr, _mlp(widths=(64, 64)), query=True)
        base = _call(key, pr, None, query=True, family="plain")
        assert base > 0
        if key[1] == "forward":
            assert m1 == m2 == m3 == base
        else:
            assert 0 < m1 < m2 < m3
    pr = _desc(key)
    for bad in (None, _mlp(L=0), _mlp(widths=(65, 6)), _mlp(widths=(8, 0))):
        assert _call(key, pr, bad, query=True) == 0
    pr.P = 0
    assert _call(key, pr, _mlp(), query=True) == 0
    if key[0] == "resampled":
        pr = _desc(key); pr.P = 1
        assert _call(key, pr, _mlp(), query=True) == 0


NEW_KERNELS = ("pm_step_kernel", "pm_refit_kernel", "pm_reverse_kernel", "pm_finish_kernel")


def test_new_kernels_do_not_spill():
    nvcc = "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not installed")
    res = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas", "-v",
                          "-cubin", "-o", os.devnull, os.path.join(ROOT, "pilco_b200", "csrc", "particles_mlp.cu")],
                         capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    props = dict(re.findall(r"Function properties for (\S+)\n\s*(.*)", res.stderr))
    for k in NEW_KERNELS:
        name = next(n for n in props if re.search(r"\d%s" % k, n))
        assert "0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads" in props[name], (k, props[name])
    if os.path.exists(CUOBJDUMP):
        text = sass_named(list(NEW_KERNELS))
        assert len(text) == 4 and not any(re.search(r"\b(STL|LDL)\b", t) for t in text.values())


def _spec(R=None, hidden=(8, 6)):
    n = engine.mlp_theta_size(3, 1, hidden)
    return dict(kind=_lib.POLICY_MLP, Ds=3, U=1, squash=True, max_action=1.0, hidden=hidden,
                theta=np.zeros(n if R is None else (R, n)))


def test_engine_refusals_before_allocation():
    """dyn is None: every refusal fires before the engine touches the model or the device"""
    x0, eps = np.zeros((10, 3)), np.zeros((10, 4, 3))
    spec = _spec()
    for make, what in ((lambda s, **kw: engine.ParticlePlan(None, s, [], 10, 4, grad=True, **kw), "ParticlePlan"),
                       (lambda s, **kw: engine.ConsistentGradPlan(None, s, [], 10, 4, **kw), "ConsistentGradPlan"),
                       (lambda s, **kw: engine.particles_rollout(None, s, [], x0, eps, **kw), "particles_rollout")):
        with pytest.raises(ValueError, match=what + ".*angles"):
            make(spec, angles=[1])
        with pytest.raises(ValueError, match=what + ".*measurement_noise"):
            make(spec, measurement_noise=[0.1, 0.1, 0.1])
        with pytest.raises(ValueError, match=what + ".*schedule"):
            make(spec, schedule=True)
        with pytest.raises(ValueError, match=what + ".*parameters"):
            make(dict(spec, theta=np.zeros(spec["theta"].size + 1)))
        with pytest.raises(ValueError, match=what + ".*hidden"):
            make(dict(spec, hidden=(65,)))
        with pytest.raises(ValueError, match=what + ".*hidden"):
            make(dict(spec, hidden=(4, 4, 4)))
    with pytest.raises(ValueError, match="estimator='score'"):
        engine.ParticlePlan(None, spec, [], 10, 4, grad=True, estimator="score")
    with pytest.raises(ValueError, match="estimator='score'"):
        engine.ConsistentGradPlan(None, spec, [], 10, 4, estimator="score")
    with pytest.raises(ValueError, match=r"theta must be \[3, "):
        engine.ParticlePlan(None, _spec(R=2), [], 10, 4, grad=True, R=3)
    for make, what in ((lambda: engine.RolloutPlan(None, spec, [], np.zeros(3), np.eye(3), 4), "RolloutPlan"),
                       (lambda: engine.PredictPlan(None, spec, [], 3, 4), "PredictPlan"),
                       (lambda: engine.ActionPlan(spec), "ActionPlan")):
        with pytest.raises(ValueError, match=what + ".*particle"):
            make()


def _mlp_pilco(**kw):
    from pilco.models import PILCO
    from pilco.controllers import MlpController
    rng = np.random.RandomState(0)
    return PILCO((rng.rand(20, 3), 0.1 * rng.rand(20, 2)), controller=MlpController(2, 1, hidden=(4,)), horizon=4,
                 **kw)


def test_class_refusals_before_device_work(monkeypatch):
    """the moment-matching methods and the score estimator refuse an MlpController with a TypeError naming
    optimize_policy_sampled, and the particle methods keep their refusals; nothing reaches the device (a device call
    would fail loudly here)"""
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)
    p = _mlp_pilco()
    m, s = np.zeros((1, 2)), 0.01 * np.eye(2)
    for call in (lambda: p.predict(m, s, 3), lambda: p.propagate(m, s), lambda: p.compute_reward(),
                 lambda: p.training_loss(), lambda: p.policy_gradient(), lambda: p.predict_reward_moments(m, s, 3),
                 lambda: p.optimize_policy(maxiter=1), lambda: p.plan(np.zeros(2)),
                 lambda: p.sample_policy_gradient(m, s, 3, num_samples=8, estimator="score")):
        with pytest.raises(TypeError, match="optimize_policy_sampled"):
            call()
    with pytest.raises(ValueError, match="measurement"):
        _mlp_pilco(measurement_noise=[0.01, 0.01]).optimize_policy_sampled(num_samples=8)
    u = np.asarray(p.compute_action(np.array([[0.2, -0.1]])))
    c = p.controller
    ref = pmo.action(dict(kind=_lib.POLICY_MLP, squash=True, maxa=np.array([1.0]), Ds=2, U=1, hidden=(4,),
                                theta=c.get_flat()), np.array([[0.2, -0.1]]))
    assert u.shape == (1, 1) and u.dtype == np.float64 and np.allclose(u, ref, rtol=0, atol=1e-15)
