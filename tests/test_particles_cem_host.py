"""CPU tests of the batched forward-only rollouts and the cross-entropy method (pilco_particles_scheduled_*batch_rollout,
pilco_cem_update / pilco_cem_draw, engine.CemPlan, PILCO.plan(optimizer="cem"); DESIGN.md section 31): exported
symbols and the pilco_cem layout, status codes and their order on fake descriptors, workspace sizes, a host build of
the update's rank / refit / draw code against the numpy oracle bit for bit, the new kernels' registers and SASS, and
the engine's and the class's refusals before any device work."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

import cem_oracle as co
from abi_fakes import (ERR_ALIGN, ERR_DIM, ERR_NULL, ERR_UNSUP, ERR_WS, FAKE, PT_MAX_P, _FakeGP, _angles, _batched,
                       _noise, _particles)
from pilco_b200 import _lib, controllers, engine
from pilco_b200._lib import lib
from util import CUOBJDUMP, ROOT, sass_named

BATCH = ["pilco_particles_scheduled_batch_rollout", "pilco_particles_scheduled_consistent_batch_rollout"]
CEM_FIELDS = ("K", "H", "U", "n_elite", "alpha", "lo", "hi", "value", "cand", "xi", "mean", "std", "best_value",
              "best", "trace")


def test_library_exports_the_entry_points_and_the_cem_layout(tmp_path):
    header = open(os.path.join(ROOT, "include", "pilco_b200.h")).read()
    for name in BATCH + ["pilco_cem_update", "pilco_cem_draw", "pilco_cem_update_workspace_bytes"]:
        names = (name, name.replace("_rollout", "_workspace_bytes")) if name in BATCH else (name,)
        for s in names:
            assert hasattr(lib, s) and s in _lib.SIGNATURES and s + "(" in header, s
    offs = [getattr(_lib.Cem, f).offset for f in CEM_FIELDS]
    assert C.sizeof(_lib.Cem) == 104 and offs == [0, 4, 8, 12] + list(range(16, 104, 8))
    cc = "/usr/bin/cc"
    if not os.path.exists(cc):
        pytest.skip("no C compiler")
    src = tmp_path / "layout.c"
    body = ", ".join("offsetof(pilco_cem, %s)" % f for f in CEM_FIELDS)
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "pilco_b200.h"\nint main(void) {\n'
                   '  size_t o[] = {sizeof(pilco_cem), %s};\n'
                   '  for (int i = 0; i < %d; ++i) printf("%%zu ", o[i]);\n  return 0;\n}\n' % (body, len(CEM_FIELDS) + 1))
    exe = tmp_path / "layout"
    res = subprocess.run([cc, "-I", os.path.join(ROOT, "include"), "-I", "/usr/local/cuda/include", str(src), "-o",
                          str(exe)], capture_output=True, text=True)
    if res.returncode != 0:
        pytest.skip("the header does not compile here: " + res.stderr[:200])
    out = subprocess.run([str(exe)], capture_output=True, text=True).stdout.split()
    assert [int(x) for x in out] == [104] + offs


# ---- the batched forward: status codes and sizes ----------------------------------------------------------------------
def _sch(W_ts=3, b_ts=1):
    return _lib.PolicySchedule(W_ts, b_ts)


def _batch(consistent, pr, R=3, sch="default", value=FAKE, ang=None, nz=None, query=False):
    ref = lambda s: C.byref(s) if s is not None else None
    sch = _sch() if sch == "default" else sch
    name = BATCH[consistent]
    if query:
        return getattr(lib, name.replace("_rollout", "_workspace_bytes"))(ref(pr), ref(ang), ref(nz), ref(sch), R)
    return getattr(lib, name)(ref(pr), ref(ang), ref(nz), ref(sch), R, value, None)


def _grad_query(consistent, pr, R=3, sch="default", ang=None, nz=None):
    ref = lambda s: C.byref(s) if s is not None else None
    sch = _sch() if sch == "default" else sch
    name = "pilco_particles_scheduled_%sgrad_workspace_bytes" % ("consistent_" if consistent else "batch_")
    return getattr(lib, name)(ref(pr), ref(ang), ref(nz), None, ref(sch), R)


@pytest.mark.parametrize("consistent", [False, True], ids=["stepwise", "consistent"])
def test_batch_rollout_status_codes_and_their_order(consistent):
    """the gradient call's codes with value NULL in place of its gradient outputs, then the workspace's; every rejected
    call returns before it enqueues anything"""
    call = lambda pr, **kw: _batch(consistent, pr, **kw)
    assert call(None) == ERR_NULL
    pr = _batched(); pr.x0 = None
    assert call(pr, value=None) == ERR_NULL
    pr = _batched(); pr.dyn.D = 9
    assert call(pr, value=None) == ERR_DIM                           # the description before value
    pr = _batched(); pr.dyn.mode = 1
    assert call(pr) == ERR_UNSUP
    for R in (0, -1, 65536):
        assert call(_batched(), R=R, value=None) == ERR_DIM          # R before value
    assert call(_batched(P=1000), R=PT_MAX_P // 1000 + 1) == ERR_DIM
    assert call(_batched(), value=None) == ERR_NULL
    assert call(_batched(), value=None, nz=_noise(var=(-1.0, 0.0, 0.0))) == ERR_NULL   # value before the noise
    assert call(_batched(), nz=_noise(var=(-1.0, 0.0, 0.0))) == ERR_DIM
    assert call(_batched(), nz=_noise(nu=None)) == ERR_NULL
    assert call(_batched(), ang=_angles(7)) == ERR_DIM                # the angles' map
    assert call(_batched(), sch=_sch(-1, 1)) == ERR_DIM               # a negative stride after everything else
    assert call(_batched(), value=None, sch=_sch(-1, 1)) == ERR_NULL
    assert call(_batched(_lib.POLICY_RBF)) == ERR_UNSUP               # an active schedule with an RBF policy
    assert call(_batched(_lib.POLICY_MLP)) == ERR_UNSUP
    for pr, kw in ((_batched(), {}), (_batched(), dict(sch=None)), (_particles(), dict(R=1)),
                   (_batched(_lib.POLICY_RBF), dict(sch=None)),
                   (_batched(), dict(ang=_angles(), nz=_noise())), (_particles(H=0), {})):
        assert call(pr, **kw) == ERR_WS                               # valid: the workspace (0 bytes) is short
    pr = _batched(); pr.ws = None
    assert call(pr) == ERR_NULL
    pr = _batched(); pr.ws = FAKE + 8
    assert call(pr) == ERR_ALIGN


@pytest.mark.parametrize("consistent", [False, True], ids=["stepwise", "consistent"])
def test_batch_rollout_workspace_sizes(consistent):
    """the forward-only layout at T = R P: at R = 1 the single scheduled forward's, below the gradient call's at every
    R (no histories), growing with R; 0 exactly where the call fails on sizes"""
    single = "pilco_particles_scheduled_%sworkspace_bytes" % ("consistent_" if consistent else "")
    pr = _batched()
    one = _batch(consistent, pr, R=1, query=True)
    assert one > 0 and one == getattr(lib, single)(C.byref(pr), None, None, C.byref(_sch()))
    sizes = [_batch(consistent, pr, R=R, query=True) for R in (1, 2, 7)]
    assert sizes[0] < sizes[1] < sizes[2]
    for R in (1, 2, 7):
        assert 0 < _batch(consistent, pr, R=R, query=True) < _grad_query(consistent, pr, R=R)
    assert _batch(consistent, pr, R=2, ang=_angles(), nz=_noise(), query=True) > 0
    for R in (0, 65536):
        assert _batch(consistent, pr, R=R, query=True) == 0
    assert _batch(consistent, pr, sch=_sch(0, -1), query=True) == 0
    assert _batch(consistent, pr, ang=_angles(7), query=True) == 0
    assert _batch(consistent, pr, nz=_noise(var=(np.nan, 0.0, 0.0)), query=True) == 0
    bad = _batched(); bad.P = 0
    assert _batch(consistent, bad, query=True) == 0
    assert _batch(consistent, None, query=True) == 0


# ---- the update: status codes and sizes --------------------------------------------------------------------------------
def _cem(**kw):
    c = _lib.Cem(*[kw.get(f, d) for f, d in zip(CEM_FIELDS, (64, 5, 1, 8, 0.1, -1.5, 1.5) + (FAKE,) * 8)])
    return c


def _update(c, ws=FAKE, wsb=0):
    return lib.pilco_cem_update(C.byref(c) if c is not None else None, ws, wsb, None)


def _draw(c):
    return lib.pilco_cem_draw(C.byref(c) if c is not None else None, None)


def test_cem_status_codes_and_their_order():
    assert _update(None) == ERR_NULL and _draw(None) == ERR_NULL
    for f in ("value", "cand", "mean", "std", "best_value", "best"):
        assert _update(_cem(**{f: None, "K": 0})) == ERR_NULL, f        # NULL before the sizes
    for f in ("cand", "xi", "mean", "std"):
        assert _draw(_cem(**{f: None, "K": 0})) == ERR_NULL, f
    bad = [dict(K=0), dict(K=8193), dict(K=-1), dict(H=0), dict(U=0), dict(H=1 << 12, U=1 << 13), dict(n_elite=0),
           dict(n_elite=65), dict(alpha=-0.1), dict(alpha=1.0), dict(alpha=np.nan), dict(alpha=np.inf),
           dict(lo=1.5, hi=1.5), dict(lo=2.0, hi=1.0), dict(lo=np.nan), dict(hi=np.nan)]
    for kw in bad:
        assert _update(_cem(**kw), ws=None) == ERR_DIM, kw               # the sizes before the workspace
    for kw in (dict(K=0), dict(H=0), dict(lo=2.0, hi=1.0)):
        assert _draw(_cem(**kw)) == ERR_DIM, kw
    # the draw reads neither n_elite, alpha nor the update's outputs (its valid calls would enqueue: not made here)
    need = lib.pilco_cem_update_workspace_bytes(64)
    assert _update(_cem(), ws=None, wsb=need) == ERR_NULL
    assert _update(_cem(), ws=FAKE + 8, wsb=need) == ERR_ALIGN
    assert _update(_cem(), wsb=need - 1) == ERR_WS
    assert _update(_cem(xi=None, trace=None), wsb=0) == ERR_WS          # xi and trace may be NULL


def test_cem_workspace_bytes():
    """the rank order [K] and one flag, rounded up to 16 bytes; 0 exactly for K outside 1 .. 8192"""
    for K in (1, 3, 4, 64, 1000, 8192):
        assert lib.pilco_cem_update_workspace_bytes(K) == -(-4 * (K + 1) // 16) * 16
    for K in (0, -1, 8193):
        assert lib.pilco_cem_update_workspace_bytes(K) == 0


# ---- a host build of the update against the numpy oracle ---------------------------------------------------------------
HARNESS = r'''
#include "%s"
#include <vector>

// the kernels' flow on the host: the bitonic network sequentially, then each element's refit and draw
extern "C" void cem_rank_host(int K, const double* value, int* order) {
    int N = 1;
    while (N < K) N <<= 1;
    std::vector<double> v(N);
    std::vector<int> ix(N);
    for (int i = 0; i < N; ++i) { v[i] = i < K ? value[i] : NAN; ix[i] = i; }
    for (int k = 2; k <= N; k <<= 1)
        for (int j = k >> 1; j > 0; j >>= 1)
            for (int i = 0; i < N; ++i) cem_bitonic_step(v.data(), ix.data(), i, j, k);
    for (int i = 0; i < K; ++i) order[i] = ix[i];
}

extern "C" void cem_update_host(int K, int HU, int ke, double alpha, double lo, double hi, const double* value,
                                double* cand, const double* xi, double* mean, double* std, double* best_value,
                                double* best, double* trace, int* order) {
    cem_rank_host(K, value, order);
    const double top = value[order[0]];
    double s = 0.0;
    for (int q = 0; q < ke; ++q) s = cem_add(s, value[order[q]]);
    trace[0] = top; trace[1] = s / ke;
    const bool up = top > *best_value;
    if (up) *best_value = top;
    for (int e = 0; e < HU; ++e) {
        if (up) best[e] = cand[(size_t)order[0] * HU + e];
        cem_refit(cand, order, ke, (size_t)HU, (size_t)e, alpha, mean + e, std + e);
    }
    if (xi)
        for (size_t q = 0; q < (size_t)K * HU; ++q) {
            const int k = (int)(q / HU);
            cand[q] = cem_draw(k, mean[q %% HU], std[q %% HU], k ? xi[q] : 0.0, lo, hi);
        }
}
'''


@pytest.fixture(scope="module")
def host(tmp_path_factory):
    d = tmp_path_factory.mktemp("cem")
    src, so = d / "cem_harness.cpp", str(d / "cem_harness.so")
    src.write_text(HARNESS % os.path.join(ROOT, "pilco_b200", "csrc", "cem_math.cuh"))
    res = subprocess.run(["g++", "-O2", "-ffp-contract=off", "-shared", "-fPIC", "-o", so, str(src)],
                         capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    h = C.CDLL(so)
    dp, ip = C.POINTER(C.c_double), C.POINTER(C.c_int)
    h.cem_rank_host.argtypes = [C.c_int, dp, ip]
    h.cem_update_host.argtypes = [C.c_int, C.c_int, C.c_int, C.c_double, C.c_double, C.c_double, dp, dp, dp, dp, dp,
                                  dp, dp, dp, ip]
    return h


def _p(a, t=C.c_double):
    return a.ctypes.data_as(C.POINTER(t))


def _host_update(h, cand, value, mean, std, ke, alpha, lo, hi, best_value, best, xi):
    K, H, U = cand.shape
    cand, mean, std, best = cand.copy(), mean.copy(), std.copy(), best.copy()
    bv, trace, order = np.array([best_value]), np.zeros(2), np.zeros(K, dtype=np.int32)
    h.cem_update_host(K, H * U, ke, alpha, lo, hi, _p(np.ascontiguousarray(value)), _p(cand),
                      _p(xi) if xi is not None else None, _p(mean), _p(std), _p(bv), _p(best), _p(trace),
                      _p(order, C.c_int))
    return dict(order=order, mean=mean, std=std, best_value=bv[0], best=best, trace=trace, cand=cand)


def _values(kind, K, rng):
    if kind == "random":
        return rng.randn(K)
    if kind == "ties":
        return rng.randint(0, 4, K).astype(np.float64) * 0.5
    if kind == "nans":
        v = rng.randn(K)
        v[rng.rand(K) < 0.3] = np.nan
        v[0] = np.nan
        return v
    if kind == "all_nan":
        return np.full(K, np.nan)
    if kind == "equal":
        return np.full(K, 0.25)
    if kind == "signed_zeros":
        return np.where(rng.rand(K) < 0.5, 0.0, -0.0)
    raise ValueError(kind)


CASES = [  # values, K, k_e, alpha, std scale (large: both bounds clip)
    ("random", 37, 5, 0.1, 0.5), ("random", 64, 1, 0.0, 0.3), ("random", 1000, 1000, 0.3, 3.0),
    ("ties", 100, 10, 0.1, 0.5), ("ties", 8, 8, 0.0, 5.0), ("nans", 50, 7, 0.2, 0.5), ("nans", 16, 16, 0.1, 0.5),
    ("all_nan", 9, 3, 0.1, 0.5), ("equal", 33, 4, 0.5, 2.0), ("equal", 1, 1, 0.0, 0.5),
    ("signed_zeros", 20, 6, 0.1, 0.5), ("random", 8192, 400, 0.1, 1.0),
]


@pytest.mark.parametrize("kind,K,ke,alpha,scale", CASES)
def test_host_build_matches_the_oracle_bitwise(host, kind, K, ke, alpha, scale):
    """the rank order, mean, std, best, trace and next candidates of the host build equal the oracle's bit for bit:
    ties, NaNs, k_e = 1 and k_e = K, all-equal values, clipping at both bounds, alpha = 0"""
    rng = np.random.RandomState(K + ke)
    H, U, lo, hi = 6, 2, -np.pi / 2, np.pi / 2
    value = _values(kind, K, rng)
    cand = co.clip(scale * rng.randn(K, H, U), lo, hi)
    mean, std = 0.3 * rng.randn(H, U), scale * (0.1 + rng.rand(H, U))
    xi = rng.randn(K, H, U)
    best = rng.randn(H, U)
    order = np.zeros(K, dtype=np.int32)
    host.cem_rank_host(K, _p(value), _p(order, C.c_int))
    assert np.array_equal(order, co.rank(value))
    for best_value, x in ((-np.inf, xi), (0.1, None)):
        ref = co.update(cand, value, mean, std, ke, alpha, lo, hi, best_value, best, x)
        got = _host_update(host, cand, value, mean, std, ke, alpha, lo, hi, best_value, best, x)
        for k in ("order", "mean", "std", "best", "trace", "cand"):
            assert np.array_equal(np.asarray(got[k]), np.asarray(ref[k]), equal_nan=True), (k, kind)
        assert got["best_value"] == ref["best_value"] or (np.isnan(got["best_value"]) and np.isnan(ref["best_value"]))
    nxt = co.draw(mean, std, xi, lo, hi)
    if scale >= 2.0:
        assert (nxt == lo).any() and (nxt == hi).any()                  # both bounds reached


def test_oracle_rank_rules():
    v = np.array([1.0, np.nan, 3.0, 3.0, -np.inf, np.nan, 1.0])
    assert list(co.rank(v)) == [2, 3, 0, 6, 4, 1, 5]
    assert list(co.rank(np.array([-0.0, 0.0]))) == [0, 1]


NEW_KERNELS = ("cem_rank_kernel", "cem_refit_kernel", "cem_draw_kernel")


def test_new_kernels_do_not_spill():
    nvcc = "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not installed")
    res = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas", "-v",
                          "-cubin", "-o", os.devnull, os.path.join(ROOT, "pilco_b200", "csrc", "particles_cem.cu")],
                         capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    props = dict(re.findall(r"Function properties for (\S+)\n\s*(.*)", res.stderr))
    for k in NEW_KERNELS:
        name = next(n for n in props if re.search(r"\d%s" % k, n))
        assert "0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads" in props[name], (k, props[name])
    if os.path.exists(CUOBJDUMP):
        text = sass_named(list(NEW_KERNELS))
        assert len(text) == len(NEW_KERNELS) and not any(re.search(r"\b(STL|LDL)\b", t) for t in text.values())


# ---- refusals before device work ---------------------------------------------------------------------------------------
def _spec(H=4, Ds=3, U=1, **kw):
    return dict(controllers.TimeVaryingLinearController(Ds, U, H, feedback=False).policy_spec(), **kw)


def test_engine_refusals_before_allocation(monkeypatch):
    import torch
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)
    gp, spec = _FakeGP(n=40, D=4, E=3), _spec()
    make = lambda s=spec, **kw: engine.CemPlan(gp, s, [], 16, 4, kw.pop("K", 64), kw.pop("ke", 8), kw.pop("it", 3),
                                               **kw)
    with pytest.raises(ValueError, match="RBF"):
        make(dict(kind=_lib.POLICY_RBF, Ds=3, U=1, gp=None))
    with pytest.raises(ValueError, match="MLP"):
        make(dict(kind=_lib.POLICY_MLP, Ds=3, U=1, hidden=(8,), theta=np.zeros(41)))
    with pytest.raises(ValueError, match="num_features"):
        make(num_features=16)
    with pytest.raises(ValueError, match="resample"):
        make(resample=True)
    with pytest.raises(ValueError, match="estimator"):
        make(estimator="score")
    for kw, what in ((dict(K=0), "population"), (dict(K=8193), "population"), (dict(ke=0), "elites"),
                     (dict(ke=65), "elites"), (dict(it=0), "iters"), (dict(alpha=1.0), "alpha"),
                     (dict(alpha=-0.5), "alpha")):
        with pytest.raises(ValueError, match=what):
            make(**kw)
    with pytest.raises(ValueError, match="fewer than"):
        engine.CemPlan(gp, spec, [], 16, 5, 64, 8, 3)
    with pytest.raises(ValueError, match="leading batch"):
        make(dict(spec, W=np.zeros((2, 4, 1, 3)), b=np.zeros((2, 4, 1))))
    with pytest.raises(ValueError, match="squash"):
        make(dict(spec, squash=False))
    with pytest.raises(ValueError, match="inputs"):
        make(_spec(Ds=4))
    with pytest.raises(ValueError, match="measurement_noise"):
        make(measurement_noise=[0.1, -1.0, 0.0])


def _mpc_pilco(Dh=2, **kw):
    from pilco.models import PILCO
    rng = np.random.RandomState(0)
    return PILCO((rng.rand(20, 3), 0.1 * rng.rand(20, 2)),
                 controller=controllers.TimeVaryingLinearController(Dh, 1, 4), horizon=4, **kw)


def test_class_refusals_before_device_work(monkeypatch):
    import torch
    from pilco.models import PILCO
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)
    p = _mpc_pilco()
    flat = p.controller.get_flat().copy()
    x = np.zeros(2)
    with pytest.raises(ValueError, match="num_samples"):
        p.plan(x, optimizer="cem")
    with pytest.raises(ValueError, match="num_samples"):
        p.plan(x, optimizer="cem", num_samples=0)
    with pytest.raises(ValueError, match="restarts=1"):
        p.plan(x, optimizer="cem", num_samples=8, restarts=2)
    for kw in (dict(population=0), dict(population=8193), dict(elites=0), dict(population=10, elites=11),
               dict(maxiter=0)):
        with pytest.raises(ValueError, match="population"):
            p.plan(x, optimizer="cem", num_samples=8, **kw)
    with pytest.raises(ValueError, match="optimizer"):
        p.plan(x, optimizer="adam", num_samples=8)
    assert np.array_equal(p.controller.get_flat(), flat)
    rng = np.random.RandomState(0)
    stationary = PILCO((rng.rand(20, 3), 0.1 * rng.rand(20, 2)), horizon=4)
    with pytest.raises(TypeError, match="TimeVaryingLinearController"):
        stationary.plan(x, optimizer="cem", num_samples=8)
    mlp = PILCO((rng.rand(20, 3), 0.1 * rng.rand(20, 2)), controller=controllers.MlpController(2, 1, (4,)), horizon=4)
    with pytest.raises(TypeError, match="MlpController"):
        mlp.plan(x, optimizer="cem", num_samples=8)
