"""CPU tests of function samples from random-feature draws (pilco_particles_features_*, DESIGN.md section 30): the
sampler's closed forms (the update identity, sin^2 + cos^2, the conditional-on-omega variance against Monte Carlo),
the oracle's autograd gradient against central differences, and the library side that needs no GPU: exported symbols
and the struct layout, status codes and their order on fake descriptors, workspace sizes, the new kernels' register
budget, and the engine's refusals raised before any device work."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

import particle_features_oracle as pfo
import particle_grad_oracle as pgo
import particle_oracle as po
from abi_fakes import ERR_DIM, ERR_NULL, ERR_UNSUP, ERR_WS, FAKE, _batched, _gp, _grad, _particles, entry_call
from particle_cases import _problem, _terms
from pilco_b200 import _lib, engine
from pilco_b200._lib import lib
from util import CUOBJDUMP, ROOT, sass_named


def _normals(dyn, P, F, seed):
    rng = np.random.RandomState(seed)
    E, D = dyn["ell"].shape
    n = dyn["C"].shape[0]
    return rng.randn(E, F, D), rng.randn(P, E, 2 * F), rng.randn(P, E, n)


def _K(A, B, ell, sf2):
    return po.se_k(A, B, ell, sf2)


def test_update_identity_gives_the_posterior_covariance():
    """with an exact joint prior draw g in place of phi' w, f = g + k_xX (beta - iK (g(X) + sqrt(sn2) eps)) has
    covariance k - k_xX iK k_Xx: k - 2 k iK k + k iK (K + sn2 I) iK k"""
    rng = np.random.RandomState(0)
    n, D, sf2, sn2 = 30, 3, 0.7, 1e-2
    X, Xs, ell = rng.rand(n, D), rng.rand(6, D), 0.4 + rng.rand(D)
    K = _K(X, X, ell, sf2)
    iK = np.linalg.inv(K + sn2 * np.eye(n))
    kxX, kxx = _K(Xs, X, ell, sf2), _K(Xs, Xs, ell, sf2)
    A = kxX @ iK
    cov = kxx - A @ kxX.T - kxX @ A.T + A @ (K + sn2 * np.eye(n)) @ A.T
    assert np.abs(cov - (kxx - kxX @ iK @ kxX.T)).max() <= 1e-12 * sf2


@pytest.mark.parametrize("F", [1, 7, 64])
def test_features_have_the_prior_variance_far_from_the_data(F):
    dyn, _ = _problem(1)
    zeta, _, _ = _normals(dyn, 1, F, 2)
    omega = zeta / dyn["ell"][:, None, :]
    far = 50.0 + np.random.RandomState(3).rand(5, dyn["C"].shape[1])
    for e in range(dyn["ell"].shape[0]):
        phi = pfo.features(far, omega[e], dyn["sf2"][e])
        assert np.abs((phi * phi).sum(1) - dyn["sf2"][e]).max() <= 1e-15 * 4
    var = pfo.conditional_variance(dyn, 1e-3 * np.ones(3), omega, far)
    assert np.abs(var - dyn["sf2"][None]).max() <= 1e-12 * dyn["sf2"].max()


def test_conditional_variance_against_monte_carlo():
    """given omega, Var f(x~) over (w, eps_y) is |phi(x~) - k iK Phi(X)|^2 + sn2 |iK k|^2 (5 standard errors, seeded);
    the mean is the posterior mean k iK y"""
    dyn, rng = _problem(2, n=15)
    sn2 = 1e-3 * np.ones(3)
    P, F = 40000, 16
    zeta, w, eps_y = _normals(dyn, P, F, 4)
    omega, v = pfo.draw(dyn, sn2, zeta, w, eps_y)
    x = np.tile(dyn["C"][3] + 0.05, (P, 1))
    f = pfo.evaluate(dyn, omega, w, v, x)
    var = pfo.conditional_variance(dyn, sn2, omega, x[:1])[0]
    sv = f.var(0, ddof=1)
    se = var * np.sqrt(2.0 / (P - 1))
    assert np.all(np.abs(sv - var) <= 5 * se), (sv, var)
    mu = po.gp_latent(dyn, x[:1])[0][0]
    assert np.all(np.abs(f.mean(0) - mu) <= 5 * np.sqrt(var / P))


def test_oracle_gradient_matches_central_differences():
    dyn, rng = _problem(3)
    P, H, F = 6, 4, 8
    zeta, w, eps_y = _normals(dyn, P, F, 5)
    omega, v = pfo.draw(dyn, 1e-3 * np.ones(3), zeta, w, eps_y)
    W, b = 0.4 * rng.randn(1, 3), 0.1 * rng.randn(1)
    pol = dict(kind=_lib.POLICY_LINEAR, squash=True, maxa=np.array([1.5]), W=W, b=b)
    terms, x0 = _terms(3), 0.3 * rng.randn(P, 3)
    val, g, hist = pfo.value_and_grad(dyn, omega, w, v, pol, terms, x0, H, 1.5)
    ref = pfo.rollout(dyn, omega, w, v, pol, terms, x0, H, 1.5)
    assert abs(val - float(ref[4].mean())) <= 1e-12 * max(1.0, abs(val))
    assert np.abs(hist["traj"] - ref[0]).max() <= 1e-12
    dW = np.random.RandomState(1).randn(*W.shape)
    f = lambda Wx: float(pfo.rollout(dyn, omega, w, v, dict(pol, W=Wx), terms, x0, H, 1.5)[4].mean())
    h = 1e-6
    fd = (f(W + h * dW) - f(W - h * dW)) / (2 * h)
    gd = float((np.asarray(g["W"]) * dW).sum())
    assert abs(fd - gd) <= 1e-6 * max(abs(gd), 1e-3), (fd, gd)


# ---- the library: exports, layout, status codes, sizes, kernels --------------------------------------------------------
NAMES = ["pilco_particles_features_draw", "pilco_particles_features_rollout", "pilco_particles_features_grad_rollout",
         "pilco_particles_mlp_features_rollout", "pilco_particles_mlp_features_grad_rollout"]


def test_library_exports_the_entry_points_and_the_struct_layout(tmp_path):
    header = open(os.path.join(ROOT, "include", "pilco_b200.h")).read()
    for name in NAMES:
        size = name.replace("_rollout", "_workspace_bytes") if name.endswith("_rollout") else name + "_workspace_bytes"
        for s in (name, size):
            assert hasattr(lib, s) and s in _lib.SIGNATURES and s + "(" in header, s
    assert "#define PILCO_MAX_FEATURES 8192" in header and _lib.MAX_FEATURES == 8192
    assert lib.pilco_version() == _lib.ABI_VERSION == 3
    offs = [getattr(_lib.FeatureDraws, f).offset for f in ("F", "omega", "w", "v")]
    assert C.sizeof(_lib.FeatureDraws) == 32 and offs == [0, 8, 16, 24]
    cc = "/usr/bin/cc"
    if not os.path.exists(cc):
        pytest.skip("no C compiler")
    src = tmp_path / "layout.c"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "pilco_b200.h"\nint main(void) {\n'
                   '  printf("%zu %zu %zu %zu %zu\\n", sizeof(pilco_feature_draws), offsetof(pilco_feature_draws, F),\n'
                   '         offsetof(pilco_feature_draws, omega), offsetof(pilco_feature_draws, w),\n'
                   '         offsetof(pilco_feature_draws, v));\n  return 0;\n}\n')
    exe = tmp_path / "layout"
    res = subprocess.run([cc, "-I", os.path.join(ROOT, "include"), "-I", "/usr/local/cuda/include", str(src), "-o",
                          str(exe)], capture_output=True, text=True)
    if res.returncode != 0:
        pytest.skip("the header does not compile here: " + res.stderr[:200])
    out = subprocess.run([str(exe)], capture_output=True, text=True).stdout.split()
    assert [int(x) for x in out] == [32] + offs


def _fd(F=64, omega=FAKE, w=FAKE, v=FAKE):
    return _lib.FeatureDraws(F, omega, w, v)


KEYS = [("lin", "forward"), ("lin", "pathwise"), ("mlp", "forward"), ("mlp", "pathwise")]


def _mlp(theta=FAKE, gtheta=FAKE):
    return _lib.Mlp(1, (C.c_int * 2)(8, 0), theta, 0, gtheta)


def _call(key, pr, fd, g=None, R=3, query=False, ang=None, nz=None, ex=None, mlp="default"):
    """row (plain (lin) or mlp, "features", kind) of engine.PARTICLE_ENTRY_POINTS"""
    pol, kind = key
    return entry_call(("plain" if pol == "lin" else "mlp", "features", kind), query, pr=pr, ang=ang, nz=nz,
                      mlp=_mlp() if mlp == "default" else mlp, ex=ex, fd=fd, grad=g, R=R)


def _desc(key):
    kind = _lib.POLICY_MLP if key[0] == "mlp" else _lib.POLICY_LINEAR
    pr = _particles(kind) if key[1] == "forward" else _batched(kind)
    if key[0] == "mlp" and key[1] != "forward":
        pr.pol.W_bs = pr.pol.b_bs = 0
    return pr


@pytest.mark.parametrize("key", KEYS, ids=lambda k: "%s-%s" % k)
def test_status_codes_and_their_order(key):
    """the mirrored consistent call's codes (pr->eps excepted), then the draws' NULL and F, then the workspace; every
    rejected call returns before it enqueues anything"""
    g = _grad()
    assert _call(key, None, _fd(), g) == ERR_NULL
    pr = _desc(key); pr.x0 = None
    assert _call(key, pr, None, g) == ERR_NULL                       # the description before the draws
    pr = _desc(key); pr.dyn.D = 9
    assert _call(key, pr, None, g) == ERR_DIM
    pr = _desc(key); pr.dyn.mode = 1
    assert _call(key, pr, _fd(F=0), g) == ERR_UNSUP
    pr = _desc(key); pr.eps = None
    assert _call(key, pr, _fd(), g) == ERR_WS                        # eps is not read
    if key[1] != "forward":
        assert _call(key, _desc(key), None, g, R=0) == ERR_DIM        # R before the draws
        bad = _grad(); bad.value = None
        assert _call(key, _desc(key), None, bad) == ERR_NULL
        assert _call(key, _desc(key), _fd(F=0), bad) == ERR_NULL      # the outputs before F
    for fd in (None, _fd(omega=None), _fd(w=None), _fd(v=None), _fd(F=0, w=None)):
        assert _call(key, _desc(key), fd, g) == ERR_NULL
    for F in (0, -1, 8193):
        assert _call(key, _desc(key), _fd(F=F), g) == ERR_DIM
    assert _call(key, _desc(key), _fd(F=8192), g) == ERR_WS
    assert _call(key, _desc(key), _fd(F=1), g) == ERR_WS
    if key[0] == "lin":
        a = _lib.Angles(); a.A = 1; a.dims[0] = 7                    # the angles' map before the draws
        assert _call(key, _desc(key), None, g, ang=a) == ERR_DIM
    else:
        assert _call(key, _desc(key), _fd(F=0), g, mlp=_mlp(theta=None)) == ERR_NULL


@pytest.mark.parametrize("key", KEYS, ids=lambda k: "%s-%s" % k)
def test_workspace_sizes(key):
    """no predict workspace and nothing of size n or F: the same for every F and n, growing with H; 0 exactly where
    the call fails on sizes"""
    for P, H in ((1000, 5), (7, 0), (300, 12)):
        pr = _desc(key)
        pr.P, pr.H = P, H
        sizes = {_call(key, pr, _fd(F=F), query=True) for F in (1, 64, 8192)}
        assert len(sizes) == 1 and min(sizes) > 0
        pr.dyn.n = 4000
        assert _call(key, pr, _fd(), query=True) == min(sizes)
        pr.H = H + 1
        assert _call(key, pr, _fd(), query=True) > min(sizes)
    pr = _desc(key)
    for bad in (None, _fd(F=0), _fd(F=8193)):
        assert _call(key, pr, bad, query=True) == 0
    pr.P = 0
    assert _call(key, pr, _fd(), query=True) == 0


def test_draw_status_codes_and_workspace():
    args = lambda **kw: [kw.get(k, d) for k, d in (("dyn", C.byref(_gp())), ("sn2", FAKE), ("P", 100), ("F", 64),
                                                    ("zeta", FAKE), ("w", FAKE), ("eps", FAKE), ("omega", FAKE),
                                                    ("v", FAKE), ("ws", FAKE), ("wsb", 0), ("st", None))]
    draw = lambda **kw: lib.pilco_particles_features_draw(*args(**kw))
    for k in ("dyn", "sn2", "zeta", "w", "eps", "omega", "v", "ws"):
        assert draw(**{k: None}) == ERR_NULL, k
    assert draw(dyn=C.byref(_gp(mode=1))) == ERR_UNSUP
    assert draw(dyn=C.byref(_gp(iK=None))) == ERR_UNSUP
    assert draw(dyn=C.byref(_gp(bs=5))) == ERR_UNSUP
    for kw in (dict(P=0), dict(F=0), dict(F=8193), dict(dyn=C.byref(_gp(D=17))), dict(dyn=C.byref(_gp(ldk=32)))):
        assert draw(**kw) == ERR_DIM, kw
    assert draw(F=0, sn2=None) == ERR_NULL                             # NULL before sizes
    g = _gp()
    need = lib.pilco_particles_features_draw_workspace_bytes(C.byref(g), 100, 64)
    assert need == 8 * (3 * 50 * 128 + 100 * 3 * 50)
    assert draw(wsb=need - 1) == ERR_WS
    assert lib.pilco_particles_features_draw_workspace_bytes(C.byref(g), 100, 8193) == 0
    assert lib.pilco_particles_features_draw_workspace_bytes(C.byref(g), 0, 64) == 0
    assert lib.pilco_particles_features_draw_workspace_bytes(None, 100, 64) == 0


NEW_KERNELS = ("pf_eval_kernel", "pf_vjp_kernel", "pf_omega_kernel", "pf_phi_kernel", "pf_prep_kernel")


def test_new_kernels_do_not_spill():
    nvcc = "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not installed")
    res = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas", "-v",
                          "-cubin", "-o", os.devnull, os.path.join(ROOT, "pilco_b200", "csrc", "particles_features.cu")],
                         capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    props = dict(re.findall(r"Function properties for (\S+)\n\s*(.*)", res.stderr))
    for k in NEW_KERNELS:
        name = next(n for n in props if re.search(r"\d%s" % k, n))
        assert "0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads" in props[name], (k, props[name])
    if os.path.exists(CUOBJDUMP):
        text = sass_named(list(NEW_KERNELS))
        assert len(text) == len(NEW_KERNELS) and not any(re.search(r"\b(STL|LDL)\b", t) for t in text.values())


class _Fitc:
    """a model as fitc_factorize returns it: no sn2"""
    mode, iK, batched, n, D, E = 0, object(), False, 10, 4, 3


class _Exact(_Fitc):
    sn2 = object()


def _spec():
    return dict(kind=_lib.POLICY_LINEAR, Ds=3, U=1, squash=True, max_action=1.0, W=np.zeros((1, 3)), b=np.zeros(1))


def test_engine_refusals_before_allocation():
    """the models are host stand-ins: every refusal fires before the engine touches the device"""
    spec = _spec()
    with pytest.raises(ValueError, match="FITC"):
        engine.feature_draws(_Fitc(), 10, 8, None, None, None)
    for F in (0, 8193):
        with pytest.raises(ValueError, match="num_features"):
            engine.feature_draws(_Exact(), 10, F, None, None, None)
    with pytest.raises(ValueError, match="zeta"):
        engine.feature_draws(_Exact(), 10, 8, np.zeros((3, 8, 3)), np.zeros((10, 3, 16)), np.zeros((10, 3, 10)))
    with pytest.raises(ValueError, match="w must be"):
        engine.feature_draws(_Exact(), 10, 8, np.zeros((3, 8, 4)), np.zeros((10, 3, 8)), np.zeros((10, 3, 10)))
    with pytest.raises(ValueError, match="consistent=False"):
        engine.ParticlePlan(_Exact(), spec, [], 10, 4, num_features=8)
    with pytest.raises(ValueError, match="estimator='score'"):
        engine.ConsistentGradPlan(_Exact(), spec, [], 10, 4, estimator="score", num_features=8)
    with pytest.raises(ValueError, match="resample"):
        engine.ParticlePlan(_Exact(), spec, [], 10, 4, consistent=True, resample=True, num_features=8)
    with pytest.raises(ValueError, match="FITC"):
        engine.ConsistentGradPlan(_Fitc(), spec, [], 10, 4, num_features=8)
    draws = engine.FeatureDraws(8, np.zeros((3, 8, 4)), np.zeros((10, 3, 16)), np.zeros((10, 3, 10)))
    with pytest.raises(ValueError, match="consistent=False"):
        engine.particles_rollout(_Exact(), spec, [], np.zeros((10, 3)), None, features=draws, horizon=4)
    with pytest.raises(ValueError, match="schedule"):
        engine.particles_rollout(_Exact(), spec, [], np.zeros((10, 3)), None, consistent=True, features=draws,
                                 horizon=4, schedule=True)
    with pytest.raises(ValueError, match="horizon"):
        engine.particles_rollout(_Exact(), spec, [], np.zeros((10, 3)), None, consistent=True, features=draws)
    with pytest.raises(ValueError, match="x0 must be"):
        engine.particles_rollout(_Exact(), spec, [], np.zeros((9, 3)), None, consistent=True, features=draws,
                                 horizon=4)
    with pytest.raises(ValueError, match="FeatureDraws"):                # omega must be [E,F,D]
        engine.FeatureDraws(8, np.zeros((3, 7, 4)), np.zeros((10, 3, 16)), np.zeros((10, 3, 10)))


def _pilco(**kw):
    from pilco.models import PILCO
    rng = np.random.RandomState(0)
    return PILCO((rng.rand(20, 3), 0.1 * rng.rand(20, 2)), horizon=4, **kw)


def test_class_refusals_before_device_work(monkeypatch):
    """num_features needs consistent=True, the exact GP and the pathwise estimator, and 1 <= F <= 8192; every refusal
    fires before anything reaches the device (a device call would fail loudly here)"""
    import torch
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)
    p = _pilco()
    m, s = np.zeros((1, 2)), 0.01 * np.eye(2)
    calls = {"sample_trajectories": lambda **kw: p.sample_trajectories(m, s, 3, num_samples=8, **kw),
             "sample_reward_moments": lambda **kw: p.sample_reward_moments(m, s, 3, num_samples=8, **kw),
             "sample_policy_gradient": lambda **kw: p.sample_policy_gradient(m, s, 3, num_samples=8, **kw),
             "optimize_policy_sampled": lambda **kw: p.optimize_policy_sampled(num_samples=8, **kw)}
    for what, call in calls.items():
        with pytest.raises(ValueError, match=what + ".*consistent=False"):
            call(num_features=16)
        for F in (0, 8193):
            with pytest.raises(ValueError, match=what + ".*num_features must be"):
                call(num_features=F, consistent=True)
    with pytest.raises(ValueError, match="estimator='score'"):
        p.sample_policy_gradient(m, s, 3, num_samples=8, consistent=True, estimator="score", num_features=16)
    sp = _pilco(num_induced_points=10)
    with pytest.raises(ValueError, match="SMGPR"):
        sp.sample_trajectories(m, s, 3, num_samples=8, consistent=True, num_features=16)
    with pytest.raises(ValueError, match="SMGPR"):
        sp.optimize_policy_sampled(num_samples=8, consistent=True, num_features=16)
