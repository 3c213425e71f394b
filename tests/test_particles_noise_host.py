"""CPU tests of the particle rollouts with measurement noise at the policy's input (pilco_particles_noisy_*, DESIGN.md
section 23): the oracles' measurement noise (tests/particle_oracle.py and particle_grad_oracle.py) against their calls
without it at v = 0, against central differences and against the exact noisy moments of one step; the status codes and
workspace sizes of the ten entry points on fake descriptors; the pilco_particles_noise layout; the new kernels'
registers and SASS; and the engine's checks before any device work."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

from pilco_b200 import _lib
from pilco_b200._lib import lib
from abi_fakes import (ERR_DIM, ERR_NULL, ERR_UNSUP, ERR_WS, _FakeGP, _angle_particles, _angles, _batched, _grad,
                       _noise, _particles)
import action_reward_oracle as aro
import particle_grad_oracle as pgo
import particle_oracle as po
from oracle import torch_port as tp
from particle_cases import _host_problem, _joint_terms, _policy, _rbf_point
from util import CUOBJDUMP, ROOT, _ref, _round2, make_gp_problem, sass

NAMES = ["", "consistent_", "batch_grad_", "consistent_grad_", "score_grad_"]


def _calls(pr, ang, nz, R=1, g=None):
    """status of the five noisy rollouts on (pr, ang, nz)"""
    g = g if g is not None else _grad()
    out = []
    for i, f in enumerate(NAMES):
        fn = getattr(lib, "pilco_particles_noisy_%srollout" % f)
        out.append(fn(_ref(pr), _ref(ang), _ref(nz), None) if i < 2 else
                   fn(_ref(pr), _ref(ang), _ref(nz), R, C.byref(g), None))
    return out


def _angle_calls(pr, ang, R=1, g=None):
    g = g if g is not None else _grad()
    fwd = ["pilco_particles_angles_rollout", "pilco_particles_angles_consistent_rollout"]
    grad = ["pilco_particles_angles_batch_grad_rollout", "pilco_particles_angles_consistent_grad_rollout",
            "pilco_particles_angles_score_grad_rollout"]
    return ([getattr(lib, f)(_ref(pr), _ref(ang), None) for f in fwd]
            + [getattr(lib, f)(_ref(pr), _ref(ang), R, C.byref(g), None) for f in grad])


def _sizes(pr, ang, nz, R=1):
    out = []
    for i, f in enumerate(NAMES):
        fn = getattr(lib, "pilco_particles_noisy_%sworkspace_bytes" % f)
        out.append(fn(_ref(pr), _ref(ang), _ref(nz)) if i < 2 else fn(_ref(pr), _ref(ang), _ref(nz), R))
    return out


def _angle_sizes(pr, ang, R=1):
    out = []
    for i, f in enumerate(NAMES):
        fn = getattr(lib, "pilco_particles_angles_%sworkspace_bytes" % f)
        out.append(fn(_ref(pr), _ref(ang)) if i < 2 else fn(_ref(pr), _ref(ang), R))
    return out


def test_no_noise_is_the_angle_call():
    """nz == NULL: the angle call's status codes and byte counts (ang NULL: the call without angles)"""
    g = _grad()
    cases = [(_particles(), None), (_particles(_lib.POLICY_RBF), None), (_batched(), None), (_particles(H=0), None),
             (_particles(P=0), None), (_angle_particles(), _angles(1)), (_angle_particles(_lib.POLICY_RBF), _angles(1)),
             (_angle_particles(), _angles(3)), (_angle_particles(batched=True), _angles(2))]
    nul = _particles(); nul.x0 = None
    cases.append((nul, None))
    for pr, ang in cases:
        for R in (1, 2):
            assert _calls(pr, ang, None, R=R, g=g) == _angle_calls(pr, ang, R=R, g=g)
            assert _sizes(pr, ang, None, R=R) == _angle_sizes(pr, ang, R=R)
    assert _calls(None, None, None) == [ERR_NULL] * 5
    assert _calls(None, None, _noise()) == [ERR_NULL] * 5
    assert _sizes(None, None, _noise()) == [0] * 5


@pytest.mark.parametrize("angles", [False, True])
def test_status_codes_and_order(angles):
    """the angle call's codes first, then the variances, then nu, then the workspace; a query is 0 exactly where its
    call fails on these checks"""
    def mk(batched=False, **kw):
        if angles:
            return _angle_particles(batched=batched, **kw)
        return (_batched if batched else _particles)(**kw)
    ang = _angles(1) if angles else None
    assert _calls(mk(), ang, _noise()) == [ERR_WS] * 5                      # valid: no workspace
    assert all(s > 0 for s in _sizes(mk(), ang, _noise()))
    for bad in (float("nan"), float("inf"), -1e-300):
        for i in range(3):
            var = [0.01, 0.02, 0.03]; var[i] = bad
            assert _calls(mk(), ang, _noise(var)) == [ERR_DIM] * 5
            assert _sizes(mk(), ang, _noise(var)) == [0] * 5
    var = [0.01, 0.02, 0.03] + [float("nan")] * 13                          # beyond E: not read
    assert _calls(mk(), ang, _noise(var)) == [ERR_WS] * 5
    assert _calls(mk(), ang, _noise(nu=None)) == [ERR_NULL] * 5
    assert _sizes(mk(), ang, _noise(nu=None)) == [0] * 5
    assert _calls(mk(H=0), ang, _noise(nu=None)) == [ERR_WS] * 5           # H = 0 reads no nu
    assert all(s > 0 for s in _sizes(mk(H=0), ang, _noise(nu=None)))
    # the description's codes come first: a NULL input with bad noise is ERR_NULL, a mode-1 model ERR_UNSUP
    pr = mk(); pr.x0 = None
    assert _calls(pr, ang, _noise([float("nan")] * 3, nu=None)) == [ERR_NULL] * 5
    pr = mk(); pr.dyn.mode = 1
    assert _calls(pr, ang, _noise([-1.0] * 3)) == [ERR_UNSUP] * 5
    assert _calls(mk(batched=True), ang, _noise([-1.0] * 3))[:2] == [ERR_UNSUP] * 2
    assert _calls(mk(), ang, _noise([-1.0] * 3), R=0)[2:] == [ERR_DIM] * 3
    g = _grad(); g.value = None
    assert _calls(mk(), ang, _noise([-1.0] * 3), g=g)[2:] == [ERR_NULL] * 3
    if angles:                                                              # the angles before anything else
        assert _calls(mk(), _angles(3), _noise([-1.0] * 3, nu=None)) == [ERR_DIM] * 5
        assert _sizes(mk(), _angles(3), _noise()) == [0] * 5
    # the workspace's codes after the noise's
    pr = mk(); pr.ws_bytes = 1 << 40
    g = _grad(); g.ws_bytes = 1 << 40
    assert _calls(pr, ang, _noise([-1.0] * 3), g=g) == [ERR_DIM] * 5
    assert _calls(pr, ang, _noise(nu=None), g=g) == [ERR_NULL] * 5


@pytest.mark.parametrize("kind", [_lib.POLICY_LINEAR, _lib.POLICY_RBF])
def test_workspace_sizes(kind):
    """forward-only: the angle call's bytes; gradients: the angle layouts with the phi history (also at A = 0), then
    phi(z) [R P,H+1,Dh] and, for the pathwise and consistent gradients, phi_bar_z [R P,Dh]"""
    for P, H, R, A in ((1000, 5, 1, 0), (1000, 5, 1, 1), (777, 40, 3, 2), (1, 0, 1, 0), (1, 0, 1, 3)):
        pr = _angle_particles(kind, A=A, P=P, H=H)
        ang = _angles(*range(A)) if A else None
        Dh = 3 + A
        got = _sizes(pr, ang, _noise(), R=R)
        base = _angle_sizes(pr, ang, R=R)
        assert got[:2] == base[:2] and got[0] > 0
        if A == 0:                                                       # the angle layout's phi history, A = 0
            base = [b + 8 * _round2(R * P * (H + 1) * Dh) for b in _angle_sizes(pr, None, R=R)]
        hist, bar = 8 * _round2(R * P * (H + 1) * Dh), 8 * _round2(R * P * Dh)
        assert got[2] == base[2] + hist + bar
        assert got[3] == base[3] + hist + bar
        assert got[4] == base[4] + hist
        longer = _angle_particles(kind, A=A, P=P, H=H + 30)
        assert _sizes(longer, ang, _noise())[:2] == [lib.pilco_particles_angles_workspace_bytes(C.byref(longer), _ref(ang)),
                                                    lib.pilco_particles_angles_consistent_workspace_bytes(
                                                        C.byref(longer), _ref(ang))]
        assert _sizes(pr, ang, _noise())[0] == _sizes(longer, ang, _noise())[0]


def test_noise_struct_layout(tmp_path):
    """offsets and size of pilco_particles_noise against the ctypes mirror (compiled by the host C compiler)"""
    src = tmp_path / "layout.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "pilco_b200.h"\n'
                   'int main(void) { printf("%zu %zu %zu\\n", offsetof(pilco_particles_noise, v), '
                   'offsetof(pilco_particles_noise, nu), sizeof(pilco_particles_noise)); return 0; }\n')
    exe = tmp_path / "layout"
    res = subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)],
                         capture_output=True, text=True)
    if res.returncode != 0 and "not found" in res.stderr:
        pytest.skip("no C compiler")
    assert res.returncode == 0, res.stderr
    got = [int(x) for x in subprocess.run([str(exe)], capture_output=True, text=True).stdout.split()]
    M = _lib.ParticlesNoise
    assert got == [M.v.offset, M.nu.offset, C.sizeof(M)]
    for f in NAMES:
        assert hasattr(lib, "pilco_particles_noisy_%sworkspace_bytes" % f)
        assert hasattr(lib, "pilco_particles_noisy_%srollout" % f)


def test_new_kernels_do_not_spill():
    """ptxas of particles_noise.cu: the three pn_ kernels have no stack frame and no spills"""
    nvcc = "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not installed")
    res = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas", "-v",
                          "-cubin", "-o", os.devnull, os.path.join(ROOT, "pilco_b200", "csrc", "particles_noise.cu")],
                         capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    props = dict(re.findall(r"Function properties for (\S+)\n\s*(.*)", res.stderr))
    pn = {k: v for k, v in props.items() if re.match(r"_Z\d+pn_", k)}
    assert len(pn) == 3, sorted(props)
    for name, p in pn.items():
        assert "0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads" in p, (name, p)


@pytest.mark.skipif(not os.path.exists(CUOBJDUMP), reason="cuobjdump not available")
def test_new_kernels_have_no_local_memory():
    funcs = sass(r"pn_step_kernel|pn_policy_bwd_kernel|pn_state_bwd_kernel")
    assert len(funcs) == 3, sorted(funcs)
    for name, text in funcs.items():
        assert not re.search(r"\b(STL|LDL)\b", text), name


# ---- the oracle -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dims", [[], [1]])
def test_zero_noise_is_the_angle_oracle_bitwise(dims):
    """v = 0 (and v None): both samplers, the pathwise, consistent and score gradients are the oracles' without v"""
    E, A, U = 3, len(dims), 1
    dyn, rng = _host_problem(E, A, U, seed=3)
    pol = _policy("linear", rng, U, E + A)
    terms = _joint_terms(E, A, U, 0) if A else _joint_terms(3, 1, 1, 0)[1:]
    x0, eps, nu = rng.randn(40, E), rng.randn(40, 4, E), rng.randn(40, 4, E)
    same = lambda a, b: all(np.array_equal(u, w) for u, w in zip(a, b))
    for v in (None, np.zeros(E)):
        for f in (po.particle_rollout, po.consistent_rollout):
            assert same(f(dyn, pol, terms, x0, eps, 1.5, angle_dims=dims, nu=nu, v=v),
                        f(dyn, pol, terms, x0, eps, 1.5, angle_dims=dims))
        for f in (pgo.value_and_grad, pgo.consistent_value_and_grad):
            v1, g1 = f(dyn, pol, terms, x0, eps, 1.5, angle_dims=dims, nu=nu, v=v)[:2]
            v0, g0 = f(dyn, pol, terms, x0, eps, 1.5, angle_dims=dims)[:2]
            assert v0 == v1 and all(np.array_equal(g0[k], g1[k]) for k in g0)
        traj = po.particle_rollout(dyn, pol, terms, x0, eps, 1.5, angle_dims=dims)[0]
        g0 = pgo.score_grad(dyn, pol, terms, traj, eps, 1.5, angle_dims=dims)
        g1 = pgo.score_grad(dyn, pol, terms, traj, eps, 1.5, angle_dims=dims, nu=nu, v=v)
        assert all(np.array_equal(g0[k], g1[k]) for k in g0)
    # with noise the actions move, the first state does not
    a = po.particle_rollout(dyn, pol, terms, x0, eps, 1.5, angle_dims=dims, nu=nu, v=0.05 * np.ones(E))
    b = po.particle_rollout(dyn, pol, terms, x0, eps, 1.5, angle_dims=dims)
    assert np.array_equal(a[0][:, 0], b[0][:, 0]) and not np.array_equal(a[1], b[1])


@pytest.mark.parametrize("kind,dims", [("linear", []), ("linear", [1]), ("rbf", []), ("rbf", [2])])
def test_oracle_pathwise_gradient_matches_central_differences(kind, dims):
    E, U = 4, 1
    A = len(dims)
    dyn, rng = _host_problem(E, A, U, seed=13)
    pol = _policy(kind, rng, U, E + A)
    terms = _joint_terms(E, A, U, 0) if A else [dict(kind=_lib.REWARD_EXP_SA, coef=0.7, W=np.eye(E + U), t=0.2 * np.ones(E + U)),
                                              dict(kind=_lib.REWARD_LINEAR, coef=0.2, channel=_lib.CHANNEL_MULT,
                                                   W=np.eye(E)[0], t=None)]
    x0, eps, nu = rng.randn(30, E), rng.randn(30, 4, E), rng.randn(30, 4, E)
    v = np.array([0.03, 0.0, 0.05, 0.02])
    key = "W" if kind == "linear" else "Xc"
    gkey = "W" if kind == "linear" else "X"
    val = lambda p: po.particle_rollout(dyn, p, terms, x0, eps, 0.9, angle_dims=dims, nu=nu, v=v)[4].mean()
    value, g = pgo.value_and_grad(dyn, pol, terms, x0, eps, 0.9, angle_dims=dims, nu=nu, v=v)
    assert abs(value - val(pol)) <= 1e-12 * max(1.0, abs(value))
    h = 1e-5
    for j in range(E + A):
        lo, hi = dict(pol), dict(pol)
        lo[key], hi[key] = pol[key].copy(), pol[key].copy()
        lo[key][0, j] -= h; hi[key][0, j] += h
        if kind == "rbf":                                  # po's RBF policy reads C and beta: refactorise
            lo, hi = _rbf_point(lo), _rbf_point(hi)
        fd = (val(hi) - val(lo)) / (2 * h)
        assert abs(fd - g[gkey][0, j]) <= 1e-7 * max(1.0, abs(fd)), (j, fd, g[gkey][0, j])


def test_one_step_matches_the_noisy_moments():
    """H = 1, a linear unsquashed policy, no angles: x_1's sample moments over 2 10^5 particles match
    the moment-matching oracle's exact noisy step moments; without the noise they do not"""
    E, U = 3, 2
    X, Y, ell, sf2, sn2 = make_gp_problem(40, E + U, E, seed=7)
    Y = 0.1 * Y
    rng = np.random.RandomState(8)
    W, b = 0.5 * rng.randn(U, E), 0.3 * rng.randn(U)
    v = np.array([0.05, 0.02, 0.08])
    B = rng.randn(E, E)
    m0, S0 = X[0, :E], 0.03 * B @ B.T + 0.02 * np.eye(E)
    terms = [dict(kind=1, coef=1.0, W=np.ones(E), t=None)]
    T = pgo.T
    ref = aro.problem_rollout("linear", [T(W), T(b)], X, Y, ell, sf2, sn2, None, terms, T(m0), T(S0), 1, v=v)
    bare = aro.problem_rollout("linear", [T(W), T(b)], X, Y, ell, sf2, sn2, None, terms, T(m0), T(S0), 1,
                               v=np.zeros(E))
    iK, beta = tp.calculate_factorizations(T(X), T(Y), T(ell), T(sf2), T(sn2))
    dyn = dict(C=X, ell=ell, sf2=sf2, iK=iK.numpy(), beta=beta.numpy())
    pol = dict(kind=_lib.POLICY_LINEAR, squash=False, maxa=np.ones(U), W=W, b=b)
    N = 200000
    x0 = rng.multivariate_normal(m0, S0, size=N)
    traj = po.particle_rollout(dyn, pol, terms, x0, rng.randn(N, 1, E), nu=rng.randn(N, 1, E), v=v)[0]
    worst = po.moment_check(traj[:, 1], ref["traj_m"][1].numpy(), ref["traj_S"][1].numpy())
    assert worst < 5.0, worst
    assert po.moment_check(traj[:, 1], bare["traj_m"][1].numpy(), bare["traj_S"][1].numpy()) > 5.0


def test_engine_checks_before_any_allocation():
    from pilco_b200 import engine
    spec = dict(kind=_lib.POLICY_LINEAR, Ds=4, U=1, W=np.zeros((1, 4)), b=np.zeros(1))
    for bad, msg in (([0.1] * 3, "expected 4 variances"), ([0.1, 0.1, float("nan"), 0.1], "finite"),
                     ([0.1, -0.1, 0.1, 0.1], ">= 0"), ([0.1] * 5, "expected 4 variances")):
        with pytest.raises(ValueError, match=msg):
            engine.ParticlePlan(_FakeGP(), spec, [], 10, 3, measurement_noise=bad)
        with pytest.raises(ValueError, match=msg):
            engine.ConsistentGradPlan(_FakeGP(), spec, [], 10, 3, measurement_noise=bad)
        with pytest.raises(ValueError, match=msg):
            engine.ParticlePlan(_FakeGP(), dict(spec, Ds=5), [], 10, 3, grad=True, estimator="score", angles=[1],
                                measurement_noise=bad)
