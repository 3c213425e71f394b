"""CPU tests of the Gaussian-resampled particle rollouts (pilco_particles_resampled_*, engine.ParticlePlan(resample=
True), DESIGN.md section 26): the refit's Cholesky and its reverse as the device runs them (resample_math.cuh built by
the host compiler) against the torch oracle, degenerate columns included; the oracle's gradient against central
differences; the oracle's fitted moments against the moment-matching trajectory (oracle/python_port.py); the status
codes, their order and the workspace sizes of the C entry points on fake descriptors; the new kernels' registers and
SASS; and the engine's checks before any allocation."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest
import torch

from oracle import python_port as pp
from pilco_b200 import _lib, engine
from pilco_b200._lib import lib
from abi_fakes import ERR_ALIGN, ERR_DIM, ERR_NULL, ERR_UNSUP, ERR_WS, FAKE, PT_MAX_P, _batched, _grad, _particles
from particle_cases import _problem, _terms
import particle_oracle as po
import particle_grad_oracle as pgo
from util import CUOBJDUMP, ROOT, _ref, sass_named

NEW_KERNELS = ["pr_close_kernel", "pr_moments_kernel", "pr_step_kernel", "pr_adjoint_kernel", "pr_scatter_kernel"]


# ---- the refit's Cholesky and its reverse, host-compiled ---------------------------------------------------------------
@pytest.fixture(scope="module")
def chol_host(tmp_path_factory):
    d = tmp_path_factory.mktemp("resample_harness")
    src = d / "h.cpp"
    src.write_text('#include "%s"\nextern "C" void chol(const double* S, double* L, int n) { pr_chol(S, L, n); }\n'
                   'extern "C" void chol_bwd(const double* L, double* Lb, double* Sb, int n) { pr_chol_bwd(L, Lb, Sb, n); }\n'
                   % os.path.join(ROOT, "pilco_b200", "csrc", "resample_math.cuh"))
    so = str(d / "h.so")
    res = subprocess.run(["g++", "-O2", "-ffp-contract=off", "-shared", "-fPIC", "-o", so, str(src)],
                         capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    h = C.CDLL(so)
    dp = C.POINTER(C.c_double)
    h.chol.argtypes = [dp, dp, C.c_int]
    h.chol_bwd.argtypes = [dp, dp, dp, C.c_int]
    p = lambda a: a.ctypes.data_as(dp)

    def run(S, Lb):
        n = S.shape[0]
        S = np.ascontiguousarray(S, dtype=np.float64)
        L, Sb, Lb = np.zeros((n, n)), np.zeros((n, n)), np.ascontiguousarray(np.tril(Lb), dtype=np.float64).copy()
        h.chol(p(S), p(L), n)
        h.chol_bwd(p(L), p(Lb), p(Sb), n)
        return L, Sb
    return run


def _spd(rng, n, rank=None):
    A = rng.randn(n, rank or n)
    return A @ A.T + (0.0 if rank else 0.1 * np.eye(n))


@pytest.mark.parametrize("n,rank", [(1, None), (4, None), (12, None), (16, None), (6, 3), (16, 9)])
def test_host_cholesky_and_adjoint_are_the_oracle(chol_host, n, rank):
    rng = np.random.RandomState(n + (rank or 0))
    S = _spd(rng, n, rank)
    if rank is None and n > 2:
        S[2] = S[:, 2] = 0.0                                    # a zero variance: a degenerate column in the middle
    Lb = rng.randn(n, n)
    L, Sb = chol_host(S, Lb)
    Lr, Sbr = pgo.chol_np(S), pgo.chol_bwd_np(S, np.tril(Lb))
    scale = max(np.abs(Sbr).max(), 1e-300)
    print("n=%d rank=%s: factor %.1e, adjoint %.1e of scale, degenerate columns %d" % (
        n, rank, np.abs(L - Lr).max() / np.abs(Lr).max(), np.abs(Sb - Sbr).max() / scale, int((np.diag(L) == 0).sum())))
    assert np.abs(L - Lr).max() <= 1e-13 * np.abs(Lr).max()
    assert np.abs(Sb - Sbr).max() <= 1e-13 * scale
    if rank is not None or n > 2:
        assert (np.diag(L) == 0.0).any() and np.array_equal(np.diag(L) == 0.0, np.diag(Lr) == 0.0)
    np.testing.assert_allclose(L @ L.T, S, atol=1e-12 * np.abs(S).max())


# ---- the oracle ---------------------------------------------------------------------------------------------------------
def _linear(rng, Ds, squash=True):
    return dict(kind=_lib.POLICY_LINEAR, squash=squash, maxa=np.array([1.2]), W=0.6 * rng.randn(1, Ds),
                b=0.2 * rng.randn(1))


def test_oracle_gradient_is_a_central_difference():
    dyn, rng = _problem(71)
    pol = _linear(rng, 3)
    terms = _terms(3)
    P, H = 40, 5
    x0, eps, xi = 0.5 + 0.2 * rng.randn(P, 3), rng.randn(P, H, 3), rng.randn(P, H, 3)
    ref = pgo.resampled_rollout(dyn, pol, terms, x0, eps, xi, mult_mu=1.5)
    v = {"W": rng.randn(1, 3), "b": rng.randn(1)}
    gv = sum(float((ref["grad"][k].reshape(v[k].shape) * v[k]).sum()) for k in v)
    h = 1e-6
    val = lambda s: pgo.resampled_rollout(dyn, dict(pol, W=pol["W"] + s * v["W"], b=pol["b"] + s * v["b"]), terms, x0,
                                          eps, xi, mult_mu=1.5)["value"]
    cd = (val(h) - val(-h)) / (2 * h)
    print("oracle: central difference %.12e, g'v %.12e" % (cd, gv))
    assert abs(cd - gv) <= 1e-7 * max(abs(gv), 1.0)


def test_oracle_is_the_step_wise_sampler_at_one_step():
    dyn, rng = _problem(72)
    pol = _linear(rng, 3)
    P = 30
    x0, eps, xi = 0.5 + 0.2 * rng.randn(P, 3), rng.randn(P, 1, 3), rng.randn(P, 1, 3)
    ref = pgo.resampled_rollout(dyn, pol, _terms(3), x0, eps, xi, mult_mu=1.5)
    plain = po.particle_rollout(dyn, pol, _terms(3), x0, eps, mult_mu=1.5)
    np.testing.assert_allclose(ref["ret"], plain[4], rtol=1e-13, atol=1e-13)
    np.testing.assert_allclose(ref["xp"][0], plain[0][:, 1], rtol=1e-13, atol=1e-13)


def test_oracle_moments_are_the_moment_matching_trajectory():
    """linear unsquashed policy, H = 3, P = 2^14: the fitted moments of every step lie within 5 standard errors"""
    dyn, rng = _problem(73)
    pol = _linear(rng, 3, squash=False)
    terms = [dict(kind=_lib.REWARD_EXP, coef=1.0, W=np.eye(3), t=np.zeros(3))]
    P, H = 1 << 14, 3
    m0, S0 = np.array([0.5, 0.4, 0.6]), 0.02 * np.eye(3)
    x0 = m0[None] + rng.randn(P, 3) @ np.linalg.cholesky(S0).T
    eps, xi = rng.randn(P, H, 3), rng.randn(P, H, 3)
    ref = pgo.resampled_rollout(dyn, pol, terms, x0, eps, xi)
    m, s = m0[None], S0
    C_, ell, sf2 = dyn["C"], dyn["ell"], dyn["sf2"]
    worst = po.moment_check(x0, m[0], s)
    for t in range(H):
        m, s = pp.propagate(m, s, lambda mm, ss: pp.linear_action(pol["W"], pol["b"][None], mm, ss, squash=False),
                            lambda mm, ss: pp.predict_given_factorizations(C_, ell, sf2, mm, ss, dyn["iK"], dyn["beta"]))
        worst = max(worst, po.moment_check(ref["xp"][t], m[0], s))
    print("oracle moments vs moment matching at H=%d, P=%d: worst %.2f standard errors" % (H, P, worst))
    assert worst <= 5.0


# ---- the C entry points on fake descriptors -----------------------------------------------------------------------------
def _rs(xi=FAKE):
    r = _lib.ParticlesResample()
    r.xi, r.step_mean, r.step_cov = xi, None, None
    return r


def _fwd(pr, rs):
    return lib.pilco_particles_resampled_rollout(_ref(pr), _ref(rs), None)


def _grad_call(pr, rs, R, g):
    return lib.pilco_particles_resampled_grad_rollout(_ref(pr), _ref(rs), R, _ref(g), None)


def _ws(pr, rs):
    return lib.pilco_particles_resampled_workspace_bytes(_ref(pr), _ref(rs))


def _gws(pr, rs, R):
    return lib.pilco_particles_resampled_grad_workspace_bytes(_ref(pr), _ref(rs), R)


def _plain_cases():
    """(pr, R, g) that the calls without resampling reject: every description defect of abi_fakes"""
    out = []
    for kind in (_lib.POLICY_LINEAR, _lib.POLICY_RBF):
        for mutate in (lambda p: setattr(p, "x0", None), lambda p: setattr(p, "P", 0), lambda p: setattr(p, "H", -1),
                       lambda p: setattr(p.dyn, "mode", 1), lambda p: setattr(p.dyn, "D", 17),
                       lambda p: setattr(p, "n_rewards", 0), lambda p: setattr(p.rewards[0], "kind", 99),
                       lambda p: setattr(p.dyn, "iK", FAKE + 8), lambda p: setattr(p, "P", PT_MAX_P + 1)):
            pr = _particles(kind)
            mutate(pr)
            out.append((pr, 1, _grad()))
        out.append((_batched(kind), 0, _grad()))
        g = _grad(); g.value = None
        out.append((_batched(kind), 3, g))
    out.append((None, 1, _grad()))
    return out


def test_status_codes_and_their_order():
    """the call without resampling's codes first (the same status on every case it rejects), then rs / xi NULL, then
    P < 2, then the workspace"""
    seen = set()
    for i, (pr, R, g) in enumerate(_plain_cases()):
        want = lib.pilco_particles_rollout_batch_grad(_ref(pr), R, _ref(g), None)
        assert want != 0, i
        for rs in (_rs(), None, _rs(None)):
            assert _grad_call(pr, rs, R, g) == want, i
        if R == 1 and (pr is None or pr.pol.W_bs == 0):
            want_f = lib.pilco_particles_rollout(_ref(pr), None)
            assert _fwd(pr, _rs()) == want_f and _fwd(pr, None) == want_f, i
        seen.add(want)
    assert seen >= {ERR_NULL, ERR_DIM, ERR_UNSUP, ERR_ALIGN}
    for pr in (_particles(), _batched()):
        R = 1 if pr.pol.W_bs == 0 else 3
        assert _grad_call(pr, None, R, _grad()) == ERR_NULL
        assert _grad_call(pr, _rs(None), R, _grad()) == ERR_NULL
        pr.P = 1
        assert _grad_call(pr, None, R, _grad()) == ERR_NULL                 # NULL before P < 2
        assert _grad_call(pr, _rs(), R, _grad()) == ERR_DIM
        pr.P = 1000
        assert _grad_call(pr, _rs(), R, _grad()) == ERR_WS                  # the fake workspace holds 0 bytes
    pr = _particles(H=0)
    assert _fwd(pr, _rs(None)) == ERR_WS                                    # H = 0 reads no xi
    assert _fwd(_particles(), _rs(None)) == ERR_NULL and _fwd(_particles(), None) == ERR_NULL
    assert _fwd(_batched(), _rs()) == ERR_UNSUP                             # the forward is unbatched


def test_workspace_query_is_zero_exactly_where_the_call_fails_on_sizes():
    for P, H, R in ((1, 5, 1), (2, 5, 1), (1000, 0, 2), (PT_MAX_P, 3, 1), (PT_MAX_P // 2 + 1, 3, 2), (1000, 5, 0),
                    (1000, 5, 65536), (3, 40, 7)):
        pr = _batched(P=P, H=H)
        g = _grad(); g.ws_bytes = (1 << 62)
        need = _gws(pr, _rs(), R)
        rc = _grad_call(pr, _rs(), R, g)
        assert (need == 0) == (rc == ERR_DIM), (P, H, R, need, rc)
        if need:
            g.ws_bytes = need - 8
            assert _grad_call(pr, _rs(), R, g) == ERR_WS
    pr = _particles(P=1)
    assert _ws(pr, _rs()) == 0 and _ws(_particles(P=2), None) > 0


def _even(k):
    return k + (k & 1)


@pytest.mark.parametrize("kind", [_lib.POLICY_LINEAR, _lib.POLICY_RBF])
def test_workspace_bytes_are_the_stated_layout(kind):
    """the call without resampling's layout, then x' [H,T,Ds], mu^ [H,R,Ds], L^ [H,R,Ds,Ds] and (gradient) the
    reverse scratch [R,Ds+Ds^2]"""
    Ds = 3
    for P, H, R in ((1000, 5, 1), (1000, 5, 2), (777, 12, 3), (2, 0, 1), (2, 1, 4)):
        pr = (_batched if R > 1 else _particles)(kind, P=P, H=H)
        T = R * P
        extra = _even(H * T * Ds) + _even(H * R * Ds) + _even(H * R * Ds * Ds)
        base = lib.pilco_particles_batch_grad_workspace_bytes(_ref(pr), R)
        assert _gws(pr, _rs(), R) == base + 8 * (extra + _even(R * (Ds + Ds * Ds))), (P, H, R)
        if R == 1:
            assert _ws(pr, _rs()) == lib.pilco_particles_workspace_bytes(_ref(pr)) + 8 * extra, (P, H)


def test_symbols_are_exported():
    names = ["pilco_particles_resampled_workspace_bytes", "pilco_particles_resampled_rollout",
             "pilco_particles_resampled_grad_workspace_bytes", "pilco_particles_resampled_grad_rollout"]
    header = open(os.path.join(ROOT, "include", "pilco_b200.h")).read()
    for f in names:
        assert hasattr(lib, f) and f in _lib.SIGNATURES and f + "(" in header
    assert "typedef struct pilco_particles_resample" in header


def test_new_kernels_do_not_spill():
    """ptxas of particles_resample.cu: no stack frame and no spills in any of its kernels; their register arrays have
    PILCO_MAX_D compile-time entries, so this one compile covers every D <= 16"""
    nvcc = "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not installed")
    res = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas", "-v",
                          "-cubin", "-o", os.devnull, os.path.join(ROOT, "pilco_b200", "csrc", "particles_resample.cu")],
                         capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    props = dict(re.findall(r"Function properties for (\S+)\n\s*(.*)", res.stderr))
    pr = {k: v for k, v in props.items() if re.match(r"_Z\d+pr_", k)}
    assert len(pr) == len(NEW_KERNELS), sorted(props)
    for name, p in pr.items():
        assert "0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads" in p, (name, p)


@pytest.mark.skipif(not os.path.exists(CUOBJDUMP), reason="cuobjdump not available")
def test_new_kernels_have_no_local_memory():
    sass = sass_named(NEW_KERNELS)
    assert set(sass) == set(NEW_KERNELS)
    for name, text in sass.items():
        assert not re.search(r"\b(STL|LDL)\b", text), name


# ---- the engine ---------------------------------------------------------------------------------------------------------
def test_engine_refuses_before_any_allocation(monkeypatch):
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)
    for kw, what in ((dict(consistent=True), "consistent"), (dict(estimator="score", grad=True), "score"),
                     (dict(angles=[0]), "angles"), (dict(measurement_noise=[0.1, 0.1, 0.1]), "measurement_noise"),
                     (dict(exploration=0.0, grad=True), "exploration")):
        with pytest.raises(ValueError, match=what):
            engine.ParticlePlan(None, None, None, 10, 3, resample=True, **kw)
    with pytest.raises(ValueError, match="P >= 2"):
        engine.ParticlePlan(None, None, None, 1, 3, resample=True)
    with pytest.raises(ValueError, match="resample"):
        engine.particles_rollout(None, None, None, np.zeros((4, 3)), np.zeros((4, 2, 3)), consistent=True,
                                 resample=True, xi=np.zeros((4, 2, 3)))
    with pytest.raises(ValueError, match="xi"):
        engine.particles_rollout(None, None, None, np.zeros((4, 3)), np.zeros((4, 2, 3)), resample=True)
