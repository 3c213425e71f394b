"""CPU tests of the particle rollouts with angular state dimensions (pilco_particles_angles_*, DESIGN.md section 20):
the status codes of the ten angle entry points on fake descriptors (rejected calls only), their workspace sizes against
the calls without angles, the new kernels' registers and SASS, the oracles' angles (tests/particle_oracle.py and
particle_grad_oracle.py) against their calls without angles and against central differences, and the engine's checks
before any device work."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

from pilco_b200 import _lib
from pilco_b200._lib import lib
from abi_fakes import (ERR_DIM, ERR_NULL, ERR_UNSUP, ERR_WS, _FakeGP, _angle_particles, _angles, _batched, _grad,
                       _particles)
from particle_cases import _host_problem, _joint_terms
from particle_grad_oracle import consistent_value_and_grad, score_grad, value_and_grad
from particle_oracle import consistent_rollout, feature_map, particle_rollout
from util import CUOBJDUMP, ROOT, _ref, _round2, sass


# (angle twin, call without angles, takes R and a gradient)
FWD = [("pilco_particles_angles_rollout", "pilco_particles_rollout"),
       ("pilco_particles_angles_consistent_rollout", "pilco_particles_rollout_consistent")]
GRAD = [("pilco_particles_angles_batch_grad_rollout", "pilco_particles_rollout_batch_grad"),
        ("pilco_particles_angles_consistent_grad_rollout", "pilco_particles_rollout_consistent_grad"),
        ("pilco_particles_angles_score_grad_rollout", "pilco_particles_rollout_score_grad")]
WS_FWD = [("pilco_particles_angles_workspace_bytes", "pilco_particles_workspace_bytes"),
          ("pilco_particles_angles_consistent_workspace_bytes", "pilco_particles_consistent_workspace_bytes")]
WS_GRAD = [("pilco_particles_angles_batch_grad_workspace_bytes", "pilco_particles_batch_grad_workspace_bytes"),
           ("pilco_particles_angles_consistent_grad_workspace_bytes", "pilco_particles_consistent_grad_workspace_bytes"),
           ("pilco_particles_angles_score_grad_workspace_bytes", "pilco_particles_score_grad_workspace_bytes")]


def _calls(pr, ang, R=1, g=None):
    """status of every angle rollout entry point on (pr, ang)"""
    g = g if g is not None else _grad()
    out = [getattr(lib, f)(_ref(pr), _ref(ang), None) for f, _ in FWD]
    out += [getattr(lib, f)(_ref(pr), _ref(ang), R, C.byref(g), None) for f, _ in GRAD]
    return out


def test_no_angles_is_the_call_without_angles():
    """ang == NULL and A == 0: the status codes and byte counts of the calls without angles"""
    g = _grad()
    cases = [_particles(), _particles(_lib.POLICY_RBF), _batched(), _particles(H=0), _particles(P=0)]
    nul = _particles(); nul.x0 = None
    cases.append(nul)
    wrong = _particles(); wrong.dyn.E = 4
    cases.append(wrong)
    for pr in cases:
        plain = ([getattr(lib, f)(C.byref(pr), None) for _, f in FWD]
                 + [getattr(lib, f)(C.byref(pr), 2, C.byref(g), None) for _, f in GRAD])
        for ang in (None, _angles()):
            assert _calls(pr, ang, R=2, g=g) == plain
            for f, p in WS_FWD:
                assert getattr(lib, f)(C.byref(pr), _ref(ang)) == getattr(lib, p)(C.byref(pr))
            for f, p in WS_GRAD:
                assert getattr(lib, f)(C.byref(pr), _ref(ang), 2) == getattr(lib, p)(C.byref(pr), 2)
    assert _calls(None, None) == [ERR_NULL] * 5
    assert _calls(None, _angles(0)) == [ERR_NULL] * 5


def test_angle_specific_dimension_errors():
    """every rejection is returned before anything is enqueued (the fake pointers are never dereferenced)"""
    for kind in (_lib.POLICY_LINEAR, _lib.POLICY_RBF):
        assert _calls(_angle_particles(kind), _angles(1)) == [ERR_WS] * 5          # valid: no workspace
        assert _calls(_angle_particles(kind, A=3), _angles(0, 1, 2)) == [ERR_WS] * 5   # every dimension an angle
        assert _calls(_angle_particles(kind, batched=True), _angles(2), R=3) == [ERR_UNSUP] * 2 + [ERR_WS] * 3
        assert _calls(_angle_particles(kind), _angles(3)) == [ERR_DIM] * 5         # out of range
        assert _calls(_angle_particles(kind), _angles(-1)) == [ERR_DIM] * 5
        assert _calls(_angle_particles(kind, A=2), _angles(1, 1)) == [ERR_DIM] * 5  # repeated
        assert _calls(_angle_particles(kind, A=4), _angles(0, 1, 2, 0)) == [ERR_DIM] * 5
        big = _angle_particles(kind, A=4)                                           # A > E
        assert _calls(big, _angles(0, 1, 2, 2)) == [ERR_DIM] * 5
        pr = _angle_particles(kind)
        pr.pol.Ds = 3                                                               # the policy must take Dh = 4
        pr.dyn.D = 4
        assert _calls(pr, _angles(1)) == [ERR_DIM] * 5
        pr = _angle_particles(kind)
        pr.dyn.D = 6                                                                # dyn.D != Dh + U
        assert _calls(pr, _angles(1)) == [ERR_DIM] * 5
        pr = _angle_particles(kind, A=2)
        pr.pol.U, pr.dyn.D = 12, 17                                                 # dyn.D > PILCO_MAX_D
        if kind == _lib.POLICY_RBF:
            pr.pol.rbf.E = 12
        assert _calls(pr, _angles(0, 1)) == [ERR_DIM] * 5
    pr = _angle_particles(_lib.POLICY_RBF)
    pr.pol.rbf.D = 3                                                                # RBF inputs != Dh
    assert _calls(pr, _angles(1)) == [ERR_DIM] * 5
    # everything else: the codes of the calls without angles
    pr = _angle_particles(); pr.x0 = None
    assert _calls(pr, _angles(1)) == [ERR_NULL] * 5
    pr = _angle_particles(); pr.dyn.mode = 1
    assert _calls(pr, _angles(1)) == [ERR_UNSUP] * 5
    pr = _angle_particles(P=0)
    assert _calls(pr, _angles(1)) == [ERR_DIM] * 5
    pr = _angle_particles(batched=True)                                             # batched policy, R = 1 forward
    assert _calls(pr, _angles(1))[:2] == [ERR_UNSUP] * 2
    assert _calls(_angle_particles(), _angles(1), R=0)[2:] == [ERR_DIM] * 3
    g = _grad(); g.value = None
    assert _calls(_angle_particles(), _angles(1), g=g)[2:] == [ERR_NULL] * 3


@pytest.mark.parametrize("kind", [_lib.POLICY_LINEAR, _lib.POLICY_RBF])
def test_workspace_sizes(kind):
    """the angle layouts are those of the calls without angles at the same description, plus the phi history
    [R P,H+1,Dh] for the gradients; the forward-only ones do not grow with H"""
    for P, H, R, A in ((1000, 5, 1, 1), (777, 40, 3, 2), (1, 0, 1, 3)):
        pr, ang = _angle_particles(kind, A=A, P=P, H=H), _angles(*range(A))
        Dh = 3 + A
        for f, p in WS_FWD:
            got = getattr(lib, f)(C.byref(pr), C.byref(ang))
            assert got > 0 and got == getattr(lib, p)(C.byref(pr)), f
        for f, p in WS_GRAD:
            got = getattr(lib, f)(C.byref(pr), C.byref(ang), R)
            assert got == getattr(lib, p)(C.byref(pr), R) + 8 * _round2(R * P * (H + 1) * Dh), f
        assert _ws(pr, ang, "pilco_particles_angles_workspace_bytes") == _ws(
            _angle_particles(kind, A=A, P=P, H=H + 30), ang, "pilco_particles_angles_workspace_bytes")
    # invalid angles: 0
    pr = _angle_particles(kind)
    for f, _ in WS_FWD:
        assert getattr(lib, f)(C.byref(pr), C.byref(_angles(3))) == 0
    for f, _ in WS_GRAD:
        assert getattr(lib, f)(C.byref(pr), C.byref(_angles(1, 1)), 1) == 0
        assert getattr(lib, f)(C.byref(pr), C.byref(_angles(1)), 0) == 0
        assert getattr(lib, f)(None, C.byref(_angles(1)), 1) == 0


def _ws(pr, ang, f):
    return getattr(lib, f)(C.byref(pr), C.byref(ang))


def test_new_kernels_do_not_spill():
    """ptxas of particles_angles.cu: no spill stores or loads and no stack frame"""
    nvcc = "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not installed")
    res = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas", "-v",
                          "-cubin", "-o", os.devnull, os.path.join(ROOT, "pilco_b200", "csrc", "particles_angles.cu")],
                         capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    props = dict(re.findall(r"Function properties for (\S+)\n\s*(.*)", res.stderr))
    pa = {k: v for k, v in props.items() if re.match(r"_Z\d+pa_", k)}
    assert len(pa) == 3, sorted(props)
    for name, p in pa.items():
        assert "0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads" in p, (name, p)


@pytest.mark.skipif(not os.path.exists(CUOBJDUMP), reason="cuobjdump not available")
def test_new_kernels_have_no_local_memory():
    funcs = sass(r"pa_step_kernel|pa_policy_bwd_kernel|pa_state_bwd_kernel")
    assert len(funcs) == 3, sorted(funcs)
    for name, text in funcs.items():
        assert not re.search(r"\b(STL|LDL)\b", text), name


# ---- the oracles ------------------------------------------------------------------------------------------------------
def test_oracle_without_angles_is_the_oracle_without_angles():
    """with angle_dims empty the oracles compute bitwise what they compute without angle_dims: rollouts of both
    samplers, the pathwise and consistent gradients, and the score gradient"""
    dyn, rng = _host_problem(3, 0, 1, seed=1)
    pol = dict(kind=_lib.POLICY_LINEAR, squash=True, maxa=np.array([1.2]), W=rng.randn(1, 3), b=rng.randn(1))
    D = 4
    joint = dict(kind=_lib.REWARD_EXP_SA, coef=0.7, W=np.eye(D) + 0.1, t=0.2 * np.ones(D))
    terms = _joint_terms(3, 1, 1, 0)[1:] + [joint]                 # the state terms and a joint term
    x0, eps = rng.randn(50, 3), rng.randn(50, 4, 3)
    same = lambda a, b: all(np.array_equal(u, v) for u, v in zip(a, b))
    for f in (particle_rollout, consistent_rollout):
        ref = f(dyn, pol, terms, x0, eps, mult_mu=1.5)
        assert same(f(dyn, pol, terms, x0, eps, mult_mu=1.5, angle_dims=[]), ref)
    for f in (value_and_grad, consistent_value_and_grad):
        v0, g0 = f(dyn, pol, terms, x0, eps, 1.5)[:2]
        v1, g1 = f(dyn, pol, terms, x0, eps, 1.5, angle_dims=[])[:2]
        assert v0 == v1 and all(np.array_equal(g0[k], g1[k]) for k in g0)
    traj = particle_rollout(dyn, pol, terms, x0, eps, mult_mu=1.5)[0]
    g0, g1 = score_grad(dyn, pol, terms, traj, eps, 1.5), score_grad(dyn, pol, terms, traj, eps, 1.5, angle_dims=[])
    assert all(np.array_equal(g0[k], g1[k]) for k in g0)
    x = rng.randn(4, 3)
    assert feature_map(x) is x
    np.testing.assert_array_equal(feature_map(x, [1]), np.stack([x[:, 0], x[:, 2], np.sin(x[:, 1]), np.cos(x[:, 1])], 1))


@pytest.mark.parametrize("E,dims", [(4, [1]), (6, [1, 2]), (2, [0, 1])])
def test_oracle_is_periodic(E, dims):
    """x0 + 2 pi e_a: the same actions, rewards (the terms do not read dimension a raw) and return, the trajectory
    shifted by 2 pi in dimension a only.  The rounding of x0 + 2 pi (up to 4.4e-16) is all that differs; the consistent
    sampler's conditioning amplifies it more than the step-wise one (its bar 1e-10)"""
    A, U = len(dims), 1
    dyn, rng = _host_problem(E, A, U, seed=E)
    pol = dict(kind=_lib.POLICY_LINEAR, squash=True, maxa=np.array([1.1]), W=rng.randn(U, E + A), b=rng.randn(U))
    other = next((j for j in range(E) if j not in dims), None)
    terms = _joint_terms(E, A, U, other)[: 3 if other is not None else 1]
    x0, eps = rng.randn(40, E), rng.randn(40, 3, E)
    for f, bar in ((particle_rollout, 1e-12), (consistent_rollout, 1e-10)):
        a = f(dyn, pol, terms, x0, eps, mult_mu=0.7, angle_dims=dims)
        for k, ang in enumerate(dims):
            x1 = x0.copy(); x1[:, ang] += 2.0 * np.pi * (k + 1)
            b = f(dyn, pol, terms, x1, eps, mult_mu=0.7, angle_dims=dims)
            shift = np.zeros(E); shift[ang] = 2.0 * np.pi * (k + 1)
            assert np.max(np.abs(b[0] - a[0] - shift)) <= bar
            for u, v in zip(a[1:], b[1:]):
                assert np.max(np.abs(u - v), initial=0.0) <= bar


def test_oracle_pathwise_gradient_matches_central_differences():
    E, dims, U = 4, [1], 1
    dyn, rng = _host_problem(E, 1, U, seed=11)
    W, b = 0.5 * rng.randn(U, E + 1), rng.randn(U)
    terms = _joint_terms(E, 1, U, 0)
    x0, eps = rng.randn(30, E), rng.randn(30, 5, E)
    pol = lambda W, b: dict(kind=_lib.POLICY_LINEAR, squash=True, maxa=np.array([1.3]), W=W, b=b)
    val = lambda W, b: particle_rollout(dyn, pol(W, b), terms, x0, eps, mult_mu=0.9, angle_dims=dims)[4].mean()
    v, g = value_and_grad(dyn, pol(W, b), terms, x0, eps, mult_mu=0.9, angle_dims=dims)
    assert abs(v - val(W, b)) <= 1e-12 * max(1.0, abs(v))
    h = 1e-5
    for j in range(E + 1):
        dW = np.zeros_like(W); dW[0, j] = h
        fd = (val(W + dW, b) - val(W - dW, b)) / (2 * h)
        assert abs(fd - g["W"][0, j]) <= 1e-7 * max(1.0, abs(fd)), (j, fd, g["W"][0, j])
    fd = (val(W, b + h) - val(W, b - h)) / (2 * h)
    assert abs(fd - g["b"][0]) <= 1e-7 * max(1.0, abs(fd))


def test_engine_checks_before_any_allocation():
    from pilco_b200 import engine
    spec = dict(kind=_lib.POLICY_LINEAR, Ds=4, U=1, W=np.zeros((1, 4)), b=np.zeros(1))
    with pytest.raises(ValueError, match="policy must take 5 inputs"):
        engine.ParticlePlan(_FakeGP(), spec, [], 10, 3, angles=[1])
    with pytest.raises(ValueError, match="policy must take 5 inputs"):
        engine.ConsistentGradPlan(_FakeGP(), spec, [], 10, 3, angles=[1])
    with pytest.raises(ValueError, match="policy must take 5 inputs"):
        engine.ParticlePlan(_FakeGP(), spec, [], 10, 3, grad=True, estimator="score", angles=[1])
    with pytest.raises(ValueError, match="distinct"):
        engine.ParticlePlan(_FakeGP(), dict(spec, Ds=6), [], 10, 3, angles=[1, 1])
    with pytest.raises(ValueError, match="distinct"):
        engine.ParticlePlan(_FakeGP(), dict(spec, Ds=5), [], 10, 3, angles=[4])
