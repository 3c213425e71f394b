"""CPU tests of PILCO's exploration objective in the particle rollouts (pilco_particles_explore_*,
pilco_particles_reward_moments, DESIGN.md section 24): the exploration bonus of tests/particle_grad_oracle.py at b = 0
against the call without it, against central differences and, at step 0, against the closed-form reward variance;
the status codes, their order and the workspace sizes on fake descriptors; the new kernels' registers and SASS; and
the engine's checks before any device work."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

from pilco_b200 import _lib
from pilco_b200._lib import lib
from abi_fakes import (ERR_DIM, ERR_NULL, ERR_UNSUP, ERR_WS, FAKE, _FakeGP, _angle_particles, _angles, _batched, _grad,
                       _noise, _particles)
import action_reward_oracle as aro
import particle_grad_oracle as pgo
import particle_oracle as po
from particle_cases import _host_problem, _policy, _rbf_point
from util import CUOBJDUMP, ROOT, _ref, _round2, sass

GRADS = ["batch_grad_", "consistent_grad_"]
BOX_MULT = dict(kind=_lib.REWARD_BOX, coef=0.4, channel=_lib.CHANNEL_MULT,
                W=np.array([1.0, 0.0, 0.0, 0.0, -2.0, 2.0]), t=None)


def _ex(b=0.5, step_var=FAKE):
    return _lib.Exploration(b, step_var)


def _calls(pr, ang, nz, ex, R=1, g=None):
    g = g if g is not None else _grad()
    return [getattr(lib, "pilco_particles_explore_%srollout" % f)(_ref(pr), _ref(ang), _ref(nz), _ref(ex), R,
                                                                  C.byref(g), None) for f in GRADS]


def _noisy_calls(pr, ang, nz, R=1, g=None):
    g = g if g is not None else _grad()
    return [getattr(lib, "pilco_particles_noisy_%srollout" % f)(_ref(pr), _ref(ang), _ref(nz), R, C.byref(g), None)
            for f in GRADS]


def _sizes(pr, ang, nz, ex, R=1):
    return [getattr(lib, "pilco_particles_explore_%sworkspace_bytes" % f)(_ref(pr), _ref(ang), _ref(nz), _ref(ex), R)
            for f in GRADS]


def _noisy_sizes(pr, ang, nz, R=1):
    return [getattr(lib, "pilco_particles_noisy_%sworkspace_bytes" % f)(_ref(pr), _ref(ang), _ref(nz), R)
            for f in GRADS]


def test_inactive_exploration_is_the_noisy_call():
    """ex == NULL, and b = 0 with step_var NULL: the noisy call's status codes and byte counts"""
    g = _grad()
    cases = [(_particles(), None, None), (_particles(_lib.POLICY_RBF), None, None), (_batched(), None, None),
             (_particles(H=0), None, None), (_particles(P=1), None, None), (_particles(P=0), None, None),
             (_angle_particles(), _angles(1), None), (_angle_particles(), _angles(1), _noise()),
             (_particles(), None, _noise()), (_angle_particles(), _angles(3), None),
             (_particles(reward_kind=_lib.REWARD_BOX), None, None)]
    nul = _particles(); nul.x0 = None
    cases.append((nul, None, None))
    for pr, ang, nz in cases:
        for R in (1, 2):
            for ex in (None, _ex(0.0, None)):
                assert _calls(pr, ang, nz, ex, R=R, g=g) == _noisy_calls(pr, ang, nz, R=R, g=g)
                assert _sizes(pr, ang, nz, ex, R=R) == _noisy_sizes(pr, ang, nz, R=R)
    assert _calls(None, None, None, _ex()) == [ERR_NULL] * 2
    assert _sizes(None, None, None, _ex()) == [0] * 2


@pytest.mark.parametrize("feature", ["plain", "angles", "noise"])
def test_status_codes_and_order(feature):
    """the noisy call's codes first, then b, the additive box and P, then the workspace; a query is 0 exactly where its
    call fails on the exploration checks"""
    def mk(**kw):
        return _angle_particles(**kw) if feature == "angles" else _particles(**kw)
    ang = _angles(1) if feature == "angles" else None
    nz = _noise() if feature == "noise" else None
    for ex in (_ex(0.5), _ex(-0.5, None), _ex(0.0)):                         # valid: no workspace
        assert _calls(mk(), ang, nz, ex) == [ERR_WS] * 2
        assert all(s > 0 for s in _sizes(mk(), ang, nz, ex))
    for bad in (float("nan"), float("inf"), -float("inf")):
        assert _calls(mk(), ang, nz, _ex(bad)) == [ERR_DIM] * 2
        assert _sizes(mk(), ang, nz, _ex(bad)) == [0] * 2
    box = mk(reward_kind=_lib.REWARD_BOX)
    assert _calls(box, ang, nz, _ex()) == [ERR_UNSUP] * 2
    assert _sizes(box, ang, nz, _ex()) == [0] * 2
    assert _calls(mk(reward_kind=_lib.REWARD_BOX, channel=_lib.CHANNEL_MULT), ang, nz, _ex()) == [ERR_WS] * 2
    assert _calls(mk(P=1), ang, nz, _ex()) == [ERR_DIM] * 2
    assert _sizes(mk(P=1), ang, nz, _ex()) == [0] * 2
    assert _calls(mk(H=0), ang, nz, _ex()) == [ERR_WS] * 2                # H = 0: a zero bonus
    # the order: b before the box before P; the description's codes before all three
    assert _calls(mk(P=1, reward_kind=_lib.REWARD_BOX), ang, nz, _ex(float("nan"))) == [ERR_DIM] * 2
    assert _calls(mk(P=1, reward_kind=_lib.REWARD_BOX), ang, nz, _ex()) == [ERR_UNSUP] * 2
    pr = mk(reward_kind=_lib.REWARD_BOX); pr.x0 = None
    assert _calls(pr, ang, nz, _ex(float("nan"))) == [ERR_NULL] * 2
    pr = mk(P=1); pr.dyn.mode = 1
    assert _calls(pr, ang, nz, _ex()) == [ERR_UNSUP] * 2
    g = _grad(); g.value = None
    assert _calls(mk(P=1), ang, nz, _ex(), g=g) == [ERR_NULL] * 2
    assert _calls(mk(P=1), ang, nz, _ex(), R=0) == [ERR_DIM] * 2
    if feature == "noise":                                                  # the noise's checks before b's
        assert _calls(mk(), ang, _noise([-1.0] * 3), _ex(float("nan"))) == [ERR_DIM] * 2
        assert _calls(mk(reward_kind=_lib.REWARD_BOX), ang, _noise(nu=None), _ex()) == [ERR_NULL] * 2
    if feature == "angles":
        assert _calls(mk(), _angles(3), nz, _ex()) == [ERR_DIM] * 2
        assert _sizes(mk(), _angles(3), nz, _ex()) == [0] * 2
    # the workspace's codes after the exploration's
    g = _grad(); g.ws_bytes = 1 << 40
    assert _calls(mk(P=1), ang, nz, _ex(), g=g) == [ERR_DIM] * 2
    g.ws = None
    assert _calls(mk(), ang, nz, _ex(), g=g) == [ERR_NULL] * 2


@pytest.mark.parametrize("kind", [_lib.POLICY_LINEAR, _lib.POLICY_RBF])
def test_workspace_sizes(kind):
    """the noisy / angle / plain gradient layout, then sigma_t [R,H] and the table [R,H,K,2]"""
    for P, H, R, A, noise, K in ((1000, 5, 1, 0, False, 1), (1000, 5, 1, 1, False, 1), (777, 40, 3, 2, True, 1),
                                 (2, 0, 1, 0, False, 1), (500, 7, 2, 0, True, 3)):
        pr = _angle_particles(kind, A=A, P=P, H=H)
        pr.n_rewards = K
        for k in range(K):
            pr.rewards[k].kind, pr.rewards[k].coef, pr.rewards[k].W, pr.rewards[k].t = _lib.REWARD_EXP, 1.0, FAKE, FAKE
        ang = _angles(*range(A)) if A else None
        nz = _noise() if noise else None
        base = _noisy_sizes(pr, ang, nz, R=R)
        extra = 8 * (_round2(R * H) + _round2(R * H * K * 2))
        assert _sizes(pr, ang, nz, _ex(), R=R) == [b + extra for b in base] and base[0] > 0


def test_reward_moments_status_codes():
    def mk(**kw):
        pr = _particles(**kw)
        return pr
    call = lambda pr, ang=None, R=1: lib.pilco_particles_reward_moments(_ref(pr), _ref(ang), R, None, None, None)
    assert call(None) == ERR_NULL
    assert call(mk(P=1)) == ERR_DIM
    assert call(mk(), R=0) == ERR_DIM and call(mk(), R=65536) == ERR_DIM
    assert call(mk(reward_kind=_lib.REWARD_BOX)) == ERR_UNSUP
    assert call(mk(reward_kind=9)) == ERR_UNSUP
    pr = mk(); pr.rewards[0].t = None
    assert call(pr) == ERR_NULL
    pr = mk(); pr.traj = None
    assert call(pr) == ERR_NULL
    pr = mk(H=0); pr.traj = pr.act = None
    assert call(pr) == 0                                                     # H = 0: nothing to read or launch
    assert call(mk(), _angles(1)) == ERR_DIM                                 # pol.Ds must be E + A
    pr = _angle_particles(A=1, H=0)
    assert call(pr, _angles(1)) == 0
    assert call(pr, _angles(5)) == ERR_DIM


def test_new_symbols_and_kernels_do_not_spill():
    for f in GRADS:
        assert hasattr(lib, "pilco_particles_explore_%sworkspace_bytes" % f)
        assert hasattr(lib, "pilco_particles_explore_%srollout" % f)
    assert hasattr(lib, "pilco_particles_reward_moments")
    nvcc = "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not installed")
    res = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas", "-v",
                          "-cubin", "-o", os.devnull, os.path.join(ROOT, "pilco_b200", "csrc", "particles_explore.cu")],
                         capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    props = dict(re.findall(r"Function properties for (\S+)\n\s*(.*)", res.stderr))
    px = {k: v for k, v in props.items() if re.match(r"_Z\d+px_", k)}
    assert len(px) == 3, sorted(props)
    for name, p in px.items():
        assert "0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads" in p, (name, p)


@pytest.mark.skipif(not os.path.exists(CUOBJDUMP), reason="cuobjdump not available")
def test_new_kernels_have_no_local_memory():
    funcs = sass(r"px_moments_kernel|px_bonus_kernel|px_value_kernel")
    assert len(funcs) == 3, sorted(funcs)
    for name, text in funcs.items():
        assert not re.search(r"\b(STL|LDL)\b", text), name


# ---- the oracle -------------------------------------------------------------------------------------------------------
def _terms(E, A, U):
    """EXP + LINEAR state terms, an EXP_SA joint term and a MULT box (D = E + A + U)"""
    D = E + A + U
    return [dict(kind=_lib.REWARD_EXP, coef=0.8, W=0.5 * np.eye(E), t=0.2 * np.ones(E)),
            dict(kind=_lib.REWARD_LINEAR, coef=0.3, W=np.linspace(-1.0, 1.0, E), t=None),
            dict(kind=_lib.REWARD_EXP_SA, coef=0.6, W=0.4 * np.eye(D), t=0.1 * np.ones(D)),
            BOX_MULT]


@pytest.mark.parametrize("dims,noisy", [([], False), ([1], False), ([], True), ([1], True)])
def test_zero_b_is_the_noise_oracle_bitwise(dims, noisy):
    E, A, U = 4, len(dims), 1
    dyn, rng = _host_problem(E, A, U, seed=5)
    pol = _policy("linear", rng, U, E + A)
    x0, eps, nu = rng.randn(30, E), rng.randn(30, 4, E), rng.randn(30, 4, E)
    v = 0.02 * np.ones(E) if noisy else None
    for f in (pgo.value_and_grad, pgo.consistent_value_and_grad):
        out = f(dyn, pol, _terms(E, A, U), x0, eps, 1.5, angle_dims=dims, nu=nu, v=v, b=0.0)
        (v1, g1), sv = out[:2], out[-1]
        v0, g0 = f(dyn, pol, _terms(E, A, U), x0, eps, 1.5, angle_dims=dims, nu=nu, v=v)[:2]
        assert v0 == v1 and all(np.array_equal(g0[k], g1[k]) for k in g0)
        assert sv.shape == (4,) and np.all(sv > 0.0)


@pytest.mark.parametrize("kind", ["linear", "rbf"])
@pytest.mark.parametrize("b", [0.5, -0.5])
def test_oracle_gradient_matches_central_differences(kind, b):
    E, A, U = 4, 0, 1
    dyn, rng = _host_problem(E, A, U, seed=17)
    pol = _policy(kind, rng, U, E)
    terms = _terms(E, A, U)
    x0, eps = rng.randn(25, E), rng.randn(25, 3, E)
    key, gkey = ("W", "W") if kind == "linear" else ("Xc", "X")
    val = lambda p: pgo.value_and_grad(dyn, p, terms, x0, eps, mult_mu=0.9, b=b)[0]
    value, g, _ = pgo.value_and_grad(dyn, pol, terms, x0, eps, mult_mu=0.9, b=b)
    h = 1e-5
    for j in range(E):
        lo, hi = dict(pol), dict(pol)
        lo[key], hi[key] = pol[key].copy(), pol[key].copy()
        lo[key][0, j] -= h; hi[key][0, j] += h
        if kind == "rbf":
            lo, hi = _rbf_point(lo), _rbf_point(hi)
        fd = (val(hi) - val(lo)) / (2 * h)
        assert abs(fd - g[gkey][0, j]) <= 1e-7 * max(1.0, abs(fd)), (j, fd, g[gkey][0, j])


def test_step0_variance_matches_the_closed_form():
    """sigma_0^2 over 10^6 draws of x0 ~ N(m0, S0) against the closed-form Var at (m0, S0): exact for
    the state terms, and for the joint term under a linear unsquashed policy (then [x, u] is Gaussian)"""
    E, U = 3, 1
    rng = np.random.RandomState(23)
    B = rng.randn(E, E)
    m0, S0 = 0.3 * rng.randn(E), 0.2 * B @ B.T + 0.05 * np.eye(E)
    W, bb = 0.5 * rng.randn(U, E), 0.2 * rng.randn(U)
    terms = _terms(E, 0, U)
    N = 1000000
    x0 = rng.multivariate_normal(m0, S0, size=N)
    u = x0 @ W.T + bb
    traj, act = np.stack([x0, x0], 1), u[:, None]
    got = po.sample_moments(terms, traj, act)[1][0]
    mj = np.concatenate([m0, W @ m0 + bb])
    J = np.vstack([np.eye(E), W])
    Sj = J @ S0 @ J.T
    T = pgo.T
    want = 0.0
    q = np.zeros(N)                                          # per-draw sum_k c_k^2 (r_k - mean_k)^2: its spread is the SE
    for term in terms[:3]:
        joint = term["kind"] == _lib.REWARD_EXP_SA
        m, s = (mj, Sj) if joint else (m0, S0)
        c = term["coef"]
        want += c * c * float(aro.term_var(term, T(m).reshape(1, -1), T(s)))
        r = po.point_value(term, x0, u)
        q += c * c * (r - r.mean()) ** 2
    se = q.std() / np.sqrt(N)
    assert abs(got - want) < 5.0 * se, (got, want, se)
    assert abs(got - want) > 0.0


def test_engine_checks_before_any_allocation():
    from pilco_b200 import engine
    spec = dict(kind=_lib.POLICY_LINEAR, Ds=4, U=1, W=np.zeros((1, 4)), b=np.zeros(1))
    terms = [dict(kind=_lib.REWARD_LINEAR, coef=1.0, W=np.ones(4), t=None)]
    for kw, msg in ((dict(exploration=float("nan")), "finite"), (dict(exploration=float("inf")), "finite"),
                    (dict(exploration=0.5, P=1), "P >= 2")):
        P = kw.pop("P", 10)
        with pytest.raises(ValueError, match=msg):
            engine.ParticlePlan(_FakeGP(), spec, terms, P, 3, grad=True, **kw)
        with pytest.raises(ValueError, match=msg):
            engine.ConsistentGradPlan(_FakeGP(), spec, terms, P, 3, **kw)
    box = [dict(kind=_lib.REWARD_BOX, coef=1.0, W=np.zeros(6), t=None)]
    with pytest.raises(ValueError, match="additive box"):
        engine.ParticlePlan(_FakeGP(), spec, box, 10, 3, grad=True, exploration=0.0)
    for kw in (dict(grad=True, estimator="score"), dict(grad=False)):
        with pytest.raises(ValueError, match="pathwise"):
            engine.ParticlePlan(_FakeGP(), spec, terms, 10, 3, exploration=0.5, **kw)
    with pytest.raises(ValueError, match="P >= 2"):
        engine.particle_reward_moments(terms, np.zeros((1, 4, 4)), np.zeros((1, 3, 1)))
