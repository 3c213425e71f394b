"""CPU tests of the batched forward-only rollouts of stationary policies and the cross-entropy method over policy
parameters (pilco_particles_{,consistent_,mlp_,mlp_consistent_}batch_rollout, engine.ParticleBatchPlan,
policy_opt.CemPolicySearch, PILCO.optimize_policy_sampled(optimizer="cem"); DESIGN.md section 33): exported symbols,
status codes and their order on fake descriptors against the gradient calls', workspace sizes against the layout,
every kernel's SASS against the previous library's, a host build of the update at H = 1, U = n_theta with unbounded
candidates against the numpy oracle, and the engine's and the class's refusals before any device work."""
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import cem_oracle as co
from abi_fakes import (ERR_ALIGN, ERR_DIM, ERR_NULL, ERR_WS, FAKE, PT_MAX_P, _FakeGP, _angles, _batched,
                       _grad, _noise, _particles, entry_call)
from pilco_b200 import _lib, controllers, engine
from pilco_b200._lib import lib
from util import CUOBJDUMP, ROOT

CALLS = ["pilco_particles_batch_rollout", "pilco_particles_consistent_batch_rollout"]
MLP_CALLS = ["pilco_particles_mlp_batch_rollout", "pilco_particles_mlp_consistent_batch_rollout"]
GRAD = ["pilco_particles_explore_batch_grad_rollout", "pilco_particles_explore_consistent_grad_rollout"]
N_THETA = 8 * 4 + 6 * 9 + 1 * 7                       # _mlp(): Ds = 3, widths (8, 6), U = 1


def _size(name):
    return name.replace("_rollout", "_workspace_bytes")


def test_library_exports_the_entry_points():
    header = open(os.path.join(ROOT, "include", "pilco_b200.h")).read()
    for name in CALLS + MLP_CALLS:
        for s in (name, _size(name)):
            assert hasattr(lib, s) and s in _lib.SIGNATURES and s + "(" in header, s
    assert lib.pilco_version() == 3
    assert sorted(v for k, v in engine.PARTICLE_ENTRY_POINTS.items() if k[0] != "scheduled" and k[2] == "batch") == \
        sorted((n, _size(n)) for n in CALLS + MLP_CALLS)


# ---- status codes ------------------------------------------------------------------------------------------------------
ref = lambda s: C.byref(s) if s is not None else None


def _mlp(theta=FAKE, bs=N_THETA, L=2, widths=(8, 6)):
    return _lib.Mlp(L, (C.c_int * 2)(*widths), theta, bs, FAKE)


def _row(family, consistent, call):
    return family, "consistent" if consistent else "step", call


def _fwd(consistent, pr, R=3, value=FAKE, ang=None, nz=None, query=False):
    return entry_call(_row("plain", consistent, "batch"), query, pr=pr, ang=ang, nz=nz, R=R, value=value)


def _grad_call(consistent, pr, R=3, g="default", ang=None, nz=None):
    return entry_call(_row("plain", consistent, "pathwise"), pr=pr, ang=ang, nz=nz, R=R,
                      grad=_grad() if g == "default" else g)


def _mfwd(consistent, pr, mlp, R=3, value=FAKE, query=False):
    return entry_call(_row("mlp", consistent, "batch"), query, pr=pr, mlp=mlp, R=R, value=value)


def _mgrad(consistent, pr, mlp, R=3, g="default"):
    return entry_call(_row("mlp", consistent, "pathwise"), pr=pr, mlp=mlp, R=R, grad=_grad() if g == "default" else g)


def _broken():
    """(description, R, angles, noise) of calls that fail before their workspace"""
    out = [(None, 3, None, None)]
    for f in ("x0", "eps", "traj", "ret"):
        pr = _batched(); setattr(pr, f, None)
        out.append((pr, 3, None, None))
    pr = _batched(); pr.dyn.D = 9
    out.append((pr, 3, None, None))
    pr = _batched(); pr.dyn.mode = 1
    out.append((pr, 3, None, None))
    pr = _batched(); pr.pol.W_bs = -1
    out.append((pr, 3, None, None))
    pr = _batched(_lib.POLICY_RBF); pr.pol.rbf.mode = 0
    out.append((pr, 3, None, None))
    out += [(_batched(_lib.POLICY_MLP), 3, None, None), (_batched(), 0, None, None), (_batched(), 65536, None, None),
            (_batched(P=1000), PT_MAX_P // 1000 + 1, None, None), (_batched(), 3, _angles(7), None),
            (_batched(), 3, None, _noise(var=(-1.0, 0.0, 0.0))), (_batched(), 3, None, _noise(nu=None)),
            (_batched(), 3, None, _noise(var=(np.nan, 0.0, 0.0)))]
    return out


@pytest.mark.parametrize("consistent", [False, True], ids=["stepwise", "consistent"])
def test_status_codes_are_the_gradient_calls(consistent):
    """every description the gradient call (ex NULL) rejects before its workspace, the forward rejects with the same
    code; value NULL where the gradient's outputs are checked; then the workspace's codes.  No rejected call enqueues"""
    for pr, R, ang, nz in _broken():
        want = _grad_call(consistent, pr, R, ang=ang, nz=nz)
        assert want not in (0, ERR_WS)
        assert _fwd(consistent, pr, R, ang=ang, nz=nz) == want, (R, ang, nz)
        pr2 = _lib.Particles.from_buffer_copy(pr) if pr is not None else None
        if want != ERR_NULL and nz is None:                           # the description, R and angles before value
            assert _fwd(consistent, pr2, R, value=None, ang=ang, nz=nz) == want
    assert _fwd(consistent, _batched(), value=None) == _grad_call(consistent, _batched(), g=None) == ERR_NULL
    assert _fwd(consistent, _batched(), value=None, nz=_noise(var=(-1.0, 0.0, 0.0))) == ERR_NULL   # before the noise
    for pr, kw in ((_batched(), {}), (_particles(), dict(R=1)), (_batched(_lib.POLICY_RBF), {}),
                   (_batched(), dict(ang=_angles(), nz=_noise())), (_particles(H=0), {})):
        assert _fwd(consistent, pr, **kw) == ERR_WS == _grad_call(consistent, pr, **kw)
    pr = _batched(); pr.ws = None
    assert _fwd(consistent, pr) == ERR_NULL
    pr = _batched(); pr.ws = FAKE + 8
    assert _fwd(consistent, pr) == ERR_ALIGN
    # ang with A = 0 and NULL are the same call, for the codes and the sizes
    for pr in (_batched(), _particles(P=0)):
        assert _fwd(consistent, pr, ang=_angles()) == _fwd(consistent, pr)
        assert _fwd(consistent, pr, ang=_angles(), query=True) == _fwd(consistent, pr, query=True)


@pytest.mark.parametrize("consistent", [False, True], ids=["stepwise", "consistent"])
def test_mlp_status_codes_are_the_gradient_calls(consistent):
    call = lambda pr, mlp, **kw: _mfwd(consistent, pr, mlp, **kw)
    grad = lambda pr, mlp, **kw: _mgrad(consistent, pr, mlp, **kw)
    mk = lambda: _batched(_lib.POLICY_MLP)
    cases = [(None, _mlp(), 3), (mk(), None, 3), (mk(), _mlp(theta=None), 3), (mk(), _mlp(L=3), 3),
             (mk(), _mlp(widths=(65, 6)), 3), (mk(), _mlp(bs=-1), 3), (_batched(), _mlp(), 3), (mk(), _mlp(), 0),
             (mk(), _mlp(), 65536)]
    pr = mk(); pr.pol.max_action = None
    cases.append((pr, _mlp(), 3))
    for pr, m, R in cases:
        want = grad(pr, m, R=R)
        assert want not in (0, ERR_WS)
        assert call(pr, m, R=R) == want
    assert call(mk(), _mlp(), value=None) == grad(mk(), _mlp(), g=None) == ERR_NULL
    assert call(mk(), _mlp(), R=0, value=None) == ERR_DIM                   # R before value
    assert call(mk(), _mlp()) == ERR_WS == grad(mk(), _mlp())
    assert call(_particles(_lib.POLICY_MLP), _mlp(bs=0), R=1) == ERR_WS
    pr = mk(); pr.ws = FAKE + 8
    assert call(pr, _mlp()) == ERR_ALIGN


# ---- workspace sizes ---------------------------------------------------------------------------------------------------
def _ev(x):
    return x + (x & 1)


def _layout(consistent, P, H, R, n=50, D=4, E=3):
    """DESIGN.md section 33's forward-only layouts in bytes, each slot rounded up to an even count of doubles"""
    T = R * P
    pb = int(lib.pilco_gp_predict_workspace_bytes(n, D, E, T, 0))
    if not consistent:                     # x~ [T,D], the step closure's mean and var [T,E], one predict workspace
        return 8 * (_ev(T * D) + 2 * _ev(T * E) + _ev(pb // 8))
    np_ = engine.pad_n(n)                  # x~ [H,T,D], mu, s2, mean, var [T,E], W_t [T,E,np], K* [H,T,E,np], L, predict
    return 8 * (_ev(H * T * D) + 4 * _ev(T * E) + _ev(T * E * np_) + _ev(H * T * E * np_) + _ev(H * (H + 1) // 2 * T * E)
                + _ev(pb // 8))


@pytest.mark.parametrize("consistent", [False, True], ids=["stepwise", "consistent"])
def test_workspace_sizes_follow_the_layout(consistent):
    for P, H, R in ((1000, 5, 3), (37, 2, 1), (100, 40, 7), (1, 1, 1)):
        pr = _batched(P=P, H=H)
        want = _layout(consistent, P, H, R)
        assert _fwd(consistent, pr, R=R, query=True) == want, (P, H, R)
        assert _fwd(consistent, _batched(_lib.POLICY_RBF, P=P, H=H), R=R, query=True) == want
        mp = _batched(_lib.POLICY_MLP, P=P, H=H)
        assert _mfwd(consistent, mp, _mlp(), R=R, query=True) == want            # no MLP slots without a gradient
        assert _fwd(consistent, pr, R=R, nz=_noise(), query=True) == want        # the noise adds none either
        grad = getattr(lib, _size(GRAD[consistent]))(ref(pr), None, None, None, R)
        assert 0 < want < grad
    if not consistent:                                                           # does not grow with H
        assert len({_fwd(False, _batched(H=H), query=True) for H in (1, 5, 40, 400)}) == 1
    else:
        assert _fwd(True, _batched(H=40), query=True) > _fwd(True, _batched(H=5), query=True)


@pytest.mark.parametrize("consistent", [False, True], ids=["stepwise", "consistent"])
def test_size_query_is_zero_exactly_where_the_call_fails_on_sizes(consistent):
    bad = []
    for f, v in (("P", 0), ("P", PT_MAX_P + 1), ("H", -1)):
        pr = _batched(); setattr(pr, f, v)
        bad.append((pr, 3, {}))
    pr = _batched(); pr.dyn.D = 65
    bad += [(pr, 3, {}), (_batched(), 0, {}), (_batched(), 65536, {}), (_batched(P=1000), PT_MAX_P // 1000 + 1, {}),
            (_batched(), 3, dict(ang=_angles(7))), (_batched(), 3, dict(nz=_noise(var=(np.nan, 0.0, 0.0))))]
    for pr, R, kw in bad:
        assert _fwd(consistent, pr, R=R, query=True, **kw) == 0
        assert _fwd(consistent, pr, R=R, **kw) == ERR_DIM
    assert _fwd(consistent, None, query=True) == 0
    for pr, R, kw in ((_batched(), 3, {}), (_batched(_lib.POLICY_RBF), 2, {}), (_batched(H=0), 1, {}),
                      (_batched(), 3, dict(nz=_noise()))):
        assert _fwd(consistent, pr, R=R, query=True, **kw) > 0 and _fwd(consistent, pr, R=R, **kw) == ERR_WS
    mk = lambda: _batched(_lib.POLICY_MLP)
    for m, R in ((_mlp(L=0), 3), (_mlp(widths=(8, 65)), 3), (_mlp(), 0), (None, 3)):
        assert _mfwd(consistent, mk(), m, R=R, query=True) == 0
        assert _mfwd(consistent, mk(), m, R=R) in (ERR_DIM, ERR_NULL)
    assert _mfwd(consistent, mk(), _mlp(L=1, widths=(8, 0)), query=True) > 0      # width[1] unused at L = 1


# ---- the kernels -------------------------------------------------------------------------------------------------------
SASS_GOLDEN = os.path.join(ROOT, "tests", "golden", "kernel_sass.json")


@pytest.mark.skipif(not os.path.exists(CUOBJDUMP), reason="cuobjdump not available")
def test_every_kernel_is_unchanged():
    """the batched forwards are host orchestration over existing kernels: the library has the same kernels, each with
    the same SASS, as the one kernel_sass.json was recorded from (tests/golden/make_kernel_sass.py)"""
    sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
    from make_kernel_sass import kernel_hashes
    with open(SASS_GOLDEN) as f:
        golden = json.load(f)
    got = kernel_hashes(os.path.join(ROOT, "pilco_b200", "libpilco_b200.so"))
    assert sorted(got) == sorted(golden)
    changed = [k for k in golden if got[k] != golden[k]]
    assert not changed, changed


# ---- the update at H = 1, U = n_theta, unbounded: a host build against the oracle --------------------------------------
HARNESS = r'''
#include "%s"
#include <vector>

extern "C" void cem_update_host(int K, int n, int ke, double alpha, double lo, double hi, const double* value,
                                double* cand, const double* xi, double* mean, double* std, double* best_value,
                                double* best, double* trace, int* order) {
    int N = 1;
    while (N < K) N <<= 1;
    std::vector<double> v(N);
    std::vector<int> ix(N);
    for (int i = 0; i < N; ++i) { v[i] = i < K ? value[i] : NAN; ix[i] = i; }
    for (int k = 2; k <= N; k <<= 1)
        for (int j = k >> 1; j > 0; j >>= 1)
            for (int i = 0; i < N; ++i) cem_bitonic_step(v.data(), ix.data(), i, j, k);
    for (int i = 0; i < K; ++i) order[i] = ix[i];
    double s = 0.0;
    for (int q = 0; q < ke; ++q) s = cem_add(s, value[order[q]]);
    trace[0] = value[order[0]]; trace[1] = s / ke;
    const bool up = value[order[0]] > *best_value;
    if (up) *best_value = value[order[0]];
    for (int e = 0; e < n; ++e) {
        if (up) best[e] = cand[(size_t)order[0] * n + e];
        cem_refit(cand, order, ke, (size_t)n, (size_t)e, alpha, mean + e, std + e);
    }
    if (xi)
        for (size_t q = 0; q < (size_t)K * n; ++q) {
            const int k = (int)(q / n);
            cand[q] = cem_draw(k, mean[q %% n], std[q %% n], k ? xi[q] : 0.0, lo, hi);
        }
}
'''


@pytest.fixture(scope="module")
def host(tmp_path_factory):
    d = tmp_path_factory.mktemp("cem_policy")
    src, so = d / "cem_policy_harness.cpp", str(d / "cem_policy_harness.so")
    src.write_text(HARNESS % os.path.join(ROOT, "pilco_b200", "csrc", "cem_math.cuh"))
    res = subprocess.run(["g++", "-O2", "-ffp-contract=off", "-shared", "-fPIC", "-o", so, str(src)],
                         capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    h = C.CDLL(so)
    dp, ip = C.POINTER(C.c_double), C.POINTER(C.c_int)
    h.cem_update_host.argtypes = [C.c_int, C.c_int, C.c_int, C.c_double, C.c_double, C.c_double] + [dp] * 8 + [ip]
    return h


def _p(a, t=C.c_double):
    return a.ctypes.data_as(C.POINTER(t))


@pytest.mark.parametrize("K,ke,n,kind", [(40, 5, 77, "random"), (400, 40, 5153, "nans"), (64, 8, 13, "ties"),
                                         (9, 9, 4, "all_nan"), (1, 1, 6, "random")])
def test_host_update_over_policy_parameters_matches_the_oracle(host, K, ke, n, kind):
    """H = 1, U = n_theta, lo = -inf, hi = +inf: clip is the identity, row 0 of the next population is the mean exactly,
    a NaN value ranks last and never becomes the best, ties go to the lower index"""
    rng = np.random.RandomState(K + n)
    value = rng.randn(K) if kind != "ties" else rng.randint(0, 3, K) * 0.5
    if kind == "nans":
        value[rng.rand(K) < 0.3] = np.nan
        value[0] = np.nan
    if kind == "all_nan":
        value[:] = np.nan
    cand = 3.0 * rng.randn(K, 1, n)
    mean, std, xi = rng.randn(1, n), 0.1 + rng.rand(1, n), 5.0 * rng.randn(K, 1, n)
    lo, hi = -np.inf, np.inf
    ref = co.update(cand, value, mean, std, ke, 0.1, lo, hi, -np.inf, mean.copy(), xi)
    got = dict(cand=cand.copy(), mean=mean.copy(), std=std.copy(), best=mean.copy(), bv=np.array([-np.inf]),
               trace=np.zeros(2), order=np.zeros(K, dtype=np.int32))
    host.cem_update_host(K, n, ke, 0.1, lo, hi, _p(value), _p(got["cand"]), _p(xi), _p(got["mean"]), _p(got["std"]),
                         _p(got["bv"]), _p(got["best"]), _p(got["trace"]), _p(got["order"], C.c_int))
    assert np.array_equal(got["order"], ref["order"])
    for k in ("cand", "mean", "std", "best", "trace"):
        assert np.array_equal(got[k], ref[k], equal_nan=True), k
    assert np.array_equal(got["cand"][0], got["mean"])                  # row 0 is the mean exactly
    assert np.array_equal(got["cand"][1:], got["mean"][None] + got["std"][None] * xi[1:])   # no clipping
    finite = np.isfinite(value)
    if finite.any():
        top = int(np.flatnonzero(value == value[finite].max())[0])       # the lowest index among ties
        assert got["order"][0] == top and got["bv"][0] == value[top] and np.array_equal(got["best"], cand[top])
        assert not np.isin(got["order"][:finite.sum()], np.flatnonzero(~finite)).any()      # NaNs last
    else:
        assert got["bv"][0] == -np.inf and np.array_equal(got["best"], mean)               # never a NaN best


# ---- refusals before device work ---------------------------------------------------------------------------------------
def _linear_spec(R=4, Ds=3, U=1, **kw):
    return dict(kind=_lib.POLICY_LINEAR, Ds=Ds, U=U, squash=True, max_action=1.0, W=np.zeros((R, U, Ds)),
                b=np.zeros((R, U)), **kw)


def _mlp_spec(R=4, Ds=3, U=1, hidden=(8,)):
    n = engine.mlp_theta_size(Ds, U, hidden)
    return dict(kind=_lib.POLICY_MLP, Ds=Ds, U=U, squash=True, max_action=1.0, hidden=hidden, theta=np.zeros((R, n)))


class _Rbf:
    def __init__(self, batched=True, R=4, n=10, D=3, E=1):
        self.batched, self.n, self.D, self.E = batched, n, D, E
        self.X = np.zeros((R, n, D) if batched else (n, D))


def test_engine_refusals_before_allocation(monkeypatch):
    import torch
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)
    gp = _FakeGP(n=40, D=4, E=3)
    make = lambda spec=None, P=16, H=4, R=4, **kw: engine.ParticleBatchPlan(gp, _linear_spec() if spec is None else spec,
                                                                           [], P, H, R, **kw)
    for kw, what in ((dict(R=0), "R >= 1"), (dict(P=0), "P >= 1"), (dict(H=0), "H >= 1")):
        with pytest.raises(ValueError, match=what):
            make(**kw)
    with pytest.raises(ValueError, match="schedule"):
        make(dict(controllers.TimeVaryingLinearController(3, 1, 4).policy_spec(np.zeros((4, 16))), schedule=True))
    for kw, what in ((dict(num_features=16), "num_features"), (dict(resample=True), "resample"),
                     (dict(exploration=0.5), "exploration"), (dict(exploration=0.0), "exploration")):
        with pytest.raises(ValueError, match=what):
            make(**kw)
    with pytest.raises(ValueError, match="an MLP policy does not combine with angles"):
        make(_mlp_spec(Ds=4), angles=[0])
    with pytest.raises(ValueError, match="an MLP policy does not combine with measurement_noise"):
        make(_mlp_spec(), measurement_noise=[0.1, 0.1, 0.1])
    with pytest.raises(ValueError, match="parameters"):
        make(dict(_mlp_spec(), theta=np.zeros((4, 7))))
    with pytest.raises(ValueError, match="W"):
        make(_linear_spec(R=3))
    with pytest.raises(ValueError, match="leading R"):
        make(dict(kind=_lib.POLICY_RBF, Ds=3, U=1, gp=_Rbf(batched=False)))
    with pytest.raises(ValueError, match="leading R"):
        make(dict(kind=_lib.POLICY_RBF, Ds=3, U=1, gp=_Rbf(R=3)))
    with pytest.raises(ValueError, match="inputs"):
        make(_linear_spec(Ds=4))
    with pytest.raises(ValueError, match="measurement_noise"):
        make(measurement_noise=[0.1, -1.0, 0.0])
    with pytest.raises(ValueError, match="reward terms"):
        engine.ParticleBatchPlan(gp, _linear_spec(), [{}] * 9, 16, 4, 4)
    with pytest.raises(ValueError, match="max_ws_bytes"):
        make(max_ws_bytes=1024)
    with pytest.raises(RuntimeError, match="CUDA device"):                  # everything passed: the first allocation
        make(max_ws_bytes=1 << 40)


def _pilco(controller="linear", **kw):
    from pilco.models import PILCO
    rng = np.random.RandomState(0)
    Dh = 2 + len(kw.get("angle_dims") or [])
    c = {"linear": lambda: controllers.LinearController(Dh, 1),
         "rbf": lambda: controllers.RbfController(Dh, 1, 5),
         "mlp": lambda: controllers.MlpController(Dh, 1, (4,)),
         "tvl": lambda: controllers.TimeVaryingLinearController(Dh, 1, 4)}[controller]()
    return PILCO((rng.rand(20, 3), 0.1 * rng.rand(20, 2)), controller=c, horizon=4, **kw)


def test_class_refusals_before_device_work(monkeypatch):
    import torch
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)
    cem = lambda p, **kw: p.optimize_policy_sampled(**dict(dict(optimizer="cem", num_samples=8, seed=0, maxiter=2,
                                                                population=16, elites=4), **kw))
    cases = [(_pilco("tvl"), {}, "plan"), (_pilco("mlp", angle_dims=[0]), {}, "MLP policy does not combine with angles"),
             (_pilco("mlp", measurement_noise="model"), {}, "MLP policy does not combine with measurement_noise")]
    p = _pilco()
    cases += [(p, dict(exploration=0.5), "exploration"), (p, dict(resample=True), "resample"),
              (p, dict(num_features=16, consistent=True), "num_features"), (p, dict(restarts=2), "restarts=1"),
              (p, dict(restarts=0), "restarts=1")]
    for kw in (dict(population=0), dict(population=8193), dict(elites=0), dict(population=10, elites=11),
               dict(maxiter=0)):
        cases.append((p, kw, "population"))
    n = p.controller.get_flat().size
    for std in (0.0, -1.0, np.nan, np.inf, np.ones(n + 1), np.r_[np.ones(n - 1), 0.0]):
        cases.append((p, dict(cem_std=std), "cem_std"))
    cases.append((p, dict(num_samples=0), "num_samples"))
    for q, kw, what in cases:
        flat = q.controller.get_flat().copy()
        with pytest.raises(ValueError, match=what):
            cem(q, **kw)
        assert np.array_equal(q.controller.get_flat(), flat)
    with pytest.raises(ValueError, match="'cem'"):
        p.optimize_policy_sampled(optimizer="sgd")


def test_cem_branches_before_the_gradient_optimisers_refusals(monkeypatch):
    """what the gradient optimisers refuse (box terms, angles, measurement noise) reaches the device with CEM, and the
    default optimizer still refuses it with its own message"""
    import torch
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)
    from safe_pilco_extension.rewards_safe import RiskOfCollision
    from safe_pilco_extension.safe_pilco import SafePILCO
    from pilco.rewards import LinearReward
    rng = np.random.RandomState(0)
    sp = SafePILCO((rng.rand(20, 3), 0.1 * rng.rand(20, 2)), horizon=4, reward_add=LinearReward(2, np.ones(2)),
                   reward_mult=RiskOfCollision(2, [-0.1], [0.1]), mu=-4.0)
    for p, what in ((sp, "box"), (_pilco(angle_dims=[0]), "angle_dims"), (_pilco(measurement_noise="model"),
                                                                           "measurement_noise"),
                    (_pilco("rbf", angle_dims=[1]), "angle_dims")):
        with pytest.raises(ValueError, match=what):
            p.optimize_policy_sampled(num_samples=8, seed=0)
        with pytest.raises(RuntimeError, match="CUDA device"):
            p.optimize_policy_sampled(optimizer="cem", num_samples=8, seed=0, population=16, elites=4, maxiter=1)
