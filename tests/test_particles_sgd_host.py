"""CPU tests of the stochastic policy optimiser (pilco_normals, pilco_adam_update, engine.normals / AdamState,
policy_opt.StochasticEvaluator, PILCO.optimize_policy_sampled(optimizer="adam"); DESIGN.md section 32): Philox4x32-10
against Random123's known answers, a host build of sgd_math.cuh against the numpy oracle (the uniforms and the Adam step
bit for bit, the normals to 1e-15), exported symbols and the pilco_adam layout, status codes and their order, the new
kernels' registers and SASS, and the engine's and the class's refusals before any device work."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

import sgd_oracle as so
from abi_fakes import ERR_DIM, ERR_NULL, FAKE
from particle_cases import _safe_pilco
from pilco_b200 import _lib, controllers, engine
from pilco_b200._lib import lib
from util import CUOBJDUMP, ROOT, sass_named

ADAM_FIELDS = ("R", "n", "lr", "b1", "b2", "eps", "max_norm", "theta", "ld_theta", "packed", "ld_packed", "m", "v",
               "t", "b1t", "b2t", "iter", "trace", "ok", "trace_rows")
# Random123's known-answer vectors of Philox4x32-10: (counter, key, output)
KAT = [((0, 0, 0, 0), (0, 0), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
       ((0xffffffff,) * 4, (0xffffffff,) * 2, (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
       ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0),
        (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1))]


def test_library_exports_the_entry_points_and_the_adam_layout(tmp_path):
    header = open(os.path.join(ROOT, "include", "pilco_b200.h")).read()
    for s in ("pilco_normals", "pilco_adam_update"):
        assert hasattr(lib, s) and s in _lib.SIGNATURES and s + "(" in header, s
    offs = [getattr(_lib.Adam, f).offset for f in ADAM_FIELDS]
    assert C.sizeof(_lib.Adam) == 152
    assert offs == [0, 4, 8, 16, 24, 32, 40, 48, 56, 64, 72, 80, 88, 96, 104, 112, 120, 128, 136, 144]
    assert lib.pilco_version() == 3
    cc = "/usr/bin/cc"
    if not os.path.exists(cc):
        pytest.skip("no C compiler")
    src = tmp_path / "layout.c"
    body = ", ".join("offsetof(pilco_adam, %s)" % f for f in ADAM_FIELDS)
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "pilco_b200.h"\nint main(void) {\n'
                   '  size_t o[] = {sizeof(pilco_adam), %s};\n'
                   '  for (int i = 0; i < %d; ++i) printf("%%zu ", o[i]);\n  return 0;\n}\n' % (body, len(ADAM_FIELDS) + 1))
    exe = tmp_path / "layout"
    res = subprocess.run([cc, "-I", os.path.join(ROOT, "include"), "-I", "/usr/local/cuda/include", str(src), "-o",
                          str(exe)], capture_output=True, text=True)
    if res.returncode != 0:
        pytest.skip("the header does not compile here: " + res.stderr[:200])
    out = subprocess.run([str(exe)], capture_output=True, text=True).stdout.split()
    assert [int(x) for x in out] == [152] + offs


# ---- status codes ------------------------------------------------------------------------------------------------------
def _adam(**kw):
    d = dict(R=3, n=10, lr=1e-3, b1=0.9, b2=0.999, eps=1e-8, max_norm=0.0, theta=FAKE, ld_theta=10, packed=FAKE,
             ld_packed=12, m=FAKE, v=FAKE, t=FAKE, b1t=FAKE, b2t=FAKE, iter=FAKE, trace=FAKE, ok=FAKE, trace_rows=5)
    d.update(kw)
    return _lib.Adam(*[d[f] for f in ADAM_FIELDS])


def _update(a):
    return lib.pilco_adam_update(C.byref(a) if a is not None else None, None)


def test_normals_status_codes():
    assert lib.pilco_normals(1, 0, None, 10, FAKE, None) == ERR_NULL
    assert lib.pilco_normals(1, 0, FAKE, 10, None, None) == ERR_NULL
    assert lib.pilco_normals(1, 0, None, -1, FAKE, None) == ERR_NULL          # NULL before the size
    assert lib.pilco_normals(1, 0, FAKE, -1, FAKE, None) == ERR_DIM


def test_adam_status_codes_and_their_order():
    """every rejected call returns before it enqueues anything: NULL, then sizes, then hyper-parameters"""
    assert _update(None) == ERR_NULL
    for f in ("theta", "packed", "m", "v", "t", "b1t", "b2t", "iter", "trace", "ok"):
        assert _update(_adam(**{f: None, "R": 0, "lr": -1.0})) == ERR_NULL, f
    assert _update(_adam(trace=None, ok=None, trace_rows=0, R=0)) == ERR_DIM    # trace and ok unread at 0 rows
    bad = [dict(R=0), dict(R=-1), dict(n=0), dict(ld_theta=9), dict(ld_packed=11), dict(trace_rows=-1),
           dict(lr=0.0), dict(lr=-1e-3), dict(lr=np.inf), dict(lr=np.nan), dict(b1=1.0), dict(b1=-0.1),
           dict(b1=np.nan), dict(b2=1.0), dict(b2=-1e-9), dict(eps=0.0), dict(eps=-1e-8), dict(eps=np.nan),
           dict(max_norm=-1.0), dict(max_norm=np.nan)]
    for kw in bad:
        assert _update(_adam(**kw)) == ERR_DIM, kw


# ---- a host build against the oracle -----------------------------------------------------------------------------------
HARNESS = r'''
#include "%s"

extern "C" void philox_host(const uint32_t* ctr, const uint32_t* key, uint32_t* out) {
    uint32_t c[4] = {ctr[0], ctr[1], ctr[2], ctr[3]};
    sgd_philox(c, key[0], key[1]);
    for (int i = 0; i < 4; ++i) out[i] = c[i];
}

// the normals kernel's flow over all pairs, with the uniforms
extern "C" void normals_host(unsigned long long seed, unsigned stream, unsigned it, long long n, double* out,
                             double* u) {
    for (long long j = 0; j < (n + 1) / 2; ++j) {
        double u1, u2, z0, z1;
        sgd_pair_uniforms(seed, stream, it, (uint64_t)j, &u1, &u2);
        u[2 * j] = u1; u[2 * j + 1] = u2;
        sgd_box_muller(u1, u2, &z0, &z1);
        out[2 * j] = z0;
        if (2 * j + 1 < n) out[2 * j + 1] = z1;
    }
}

// the Adam kernel's flow, one restart after another, then the counter
extern "C" void adam_host(int R, int n, double lr, double b1, double b2, double eps, double max_norm, double* theta,
                          const double* packed, double* m, double* v, long long* t, double* b1t, double* b2t,
                          long long* iter, double* trace, int* ok, int trace_rows) {
    const long long k = *iter;
    for (int r = 0; r < R; ++r) {
        const double* row = packed + (size_t)r * (n + 2);
        const double* g = row + 2;
        double red[SGD_LANES];
        bool fin = true;
        for (int l = 0; l < SGD_LANES; ++l) { bool f; red[l] = sgd_lane_sumsq(g, n, l, &f); fin = fin && f; }
        for (int half = SGD_LANES / 2; half > 0; half >>= 1)
            for (int l = 0; l < half; ++l) sgd_tree_step(red, l, half);
        const bool good = row[1] == 0.0 && isfinite(row[0]) && fin;
        if (good) {
            const double scale = sgd_clip_scale(red[0], max_norm);
            const double nb1t = sgd_mul(b1t[r], b1), nb2t = sgd_mul(b2t[r], b2);
            for (int i = 0; i < n; ++i)
                sgd_adam_elem(g[i], scale, lr, b1, b2, eps, nb1t, nb2t, m + (size_t)r * n + i, v + (size_t)r * n + i,
                              theta + (size_t)r * n + i);
            t[r] += 1; b1t[r] = nb1t; b2t[r] = nb2t;
        }
        if (k >= 0 && k < trace_rows) { trace[k * R + r] = -row[0]; ok[k * R + r] = good; }
    }
    *iter = k + 1;
}
'''


@pytest.fixture(scope="module")
def host(tmp_path_factory):
    d = tmp_path_factory.mktemp("sgd")
    src, so_ = d / "sgd_harness.cpp", str(d / "sgd_harness.so")
    src.write_text(HARNESS % os.path.join(ROOT, "pilco_b200", "csrc", "sgd_math.cuh"))
    res = subprocess.run(["g++", "-O2", "-ffp-contract=off", "-shared", "-fPIC", "-o", so_, str(src)],
                         capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    h = C.CDLL(so_)
    dp, lp, ip, up = C.POINTER(C.c_double), C.POINTER(C.c_longlong), C.POINTER(C.c_int), C.POINTER(C.c_uint32)
    h.philox_host.argtypes = [up, up, up]
    h.normals_host.argtypes = [C.c_ulonglong, C.c_uint, C.c_uint, C.c_longlong, dp, dp]
    h.adam_host.argtypes = [C.c_int, C.c_int] + [C.c_double] * 5 + [dp, dp, dp, dp, lp, dp, dp, lp, dp, ip, C.c_int]
    return h


def _p(a, t=C.c_double):
    return a.ctypes.data_as(C.POINTER(t))


@pytest.mark.parametrize("case", range(len(KAT)))
def test_philox_known_answers(host, case):
    ctr, key, want = KAT[case]
    assert [int(x) for x in so.philox(np.array(ctr), np.array(key))] == list(want)
    out = np.zeros(4, dtype=np.uint32)
    host.philox_host(_p(np.array(ctr, dtype=np.uint32), C.c_uint32), _p(np.array(key, dtype=np.uint32), C.c_uint32),
                     _p(out, C.c_uint32))
    assert list(out) == list(want)


@pytest.mark.parametrize("seed,stream,it,n", [(0, 0, 0, 1), (12345, 1, 0, 1001), (2 ** 64 - 1, 2 ** 32 - 1, 7, 4096),
                                              (0x243f6a8885a308d3, 16, 2 ** 32 - 1, 333)])
def test_host_normals_match_the_oracle(host, seed, stream, it, n):
    """uniforms bitwise, in (0, 1); normals within 1e-15 of the oracle's Box-Muller relative to their radius r (an
    element near a zero of sin or cos is small, but its error is that of r's rounding and the angle's)"""
    out, u = np.zeros(n + 1), np.zeros(n + 1)
    host.normals_host(seed, stream, it, n, _p(out), _p(u))
    u1, u2 = so.pair_uniforms(seed, stream, it, (n + 1) // 2)
    got_u = u[:2 * ((n + 1) // 2)].reshape(-1, 2)
    assert np.array_equal(got_u[:, 0], u1) and np.array_equal(got_u[:, 1], u2)
    assert (u1 > 0).all() and (u1 < 1).all() and (u2 > 0).all() and (u2 < 1).all()
    ref = so.normals(seed, stream, it, n)
    r = np.repeat(np.sqrt(-2.0 * np.log(u1)), 2)[:n]
    assert np.all(np.abs(out[:n] - ref) <= 1e-15 * r)
    naive = np.stack([r[::2] * np.cos(2 * np.pi * u2), r[::2] * np.sin(2 * np.pi * u2)], -1).reshape(-1)[:n]
    assert np.all(np.abs(out[:n] - naive) <= 4e-15 * r)                   # numpy's Box-Muller with sin(2 pi u)
    assert np.array_equal(so.normals(seed, stream, it, n // 2), ref[:n // 2])
    assert out[n] == 0.0                                                  # an odd n writes n elements only


def test_sincospi_reduction_is_exact_at_the_quarter_points():
    s, c = so.sincospi(np.array([0.0, 0.5, 1.0, 1.5, 0.25, 1.75]))
    assert list(s[:4]) == [0.0, 1.0, 0.0, -1.0] and list(c[:4]) == [1.0, 0.0, -1.0, 0.0]
    assert abs(s[4] - np.sqrt(0.5)) < 2e-16 and abs(c[5] - np.sqrt(0.5)) < 2e-16


def _host_adam(h, st, packed, k, hyper, trace_rows):
    theta, m, v = st["theta"].copy(), st["m"].copy(), st["v"].copy()
    t, b1t, b2t = st["t"].copy(), st["b1t"].copy(), st["b2t"].copy()
    R, n = theta.shape
    trace, ok = np.full((max(trace_rows, 1), R), np.nan), np.zeros((max(trace_rows, 1), R), dtype=np.int32)
    it = np.array([k], dtype=np.int64)
    h.adam_host(R, n, *hyper, _p(theta), _p(np.ascontiguousarray(packed)), _p(m), _p(v), _p(t, C.c_longlong),
                _p(b1t), _p(b2t), _p(it, C.c_longlong), _p(trace), _p(ok, C.c_int), trace_rows)
    return dict(theta=theta, m=m, v=v, t=t, b1t=b1t, b2t=b2t, trace=trace, ok=ok, iter=int(it[0]))


def _state(R, n, rng, steps=None):
    st = dict(theta=rng.randn(R, n), m=np.zeros((R, n)), v=np.zeros((R, n)), t=np.zeros(R, dtype=np.int64),
              b1t=np.ones(R), b2t=np.ones(R))
    if steps is not None:                                             # per-restart step counts that differ
        st["t"] = np.asarray(steps, dtype=np.int64)
        st["b1t"], st["b2t"] = 0.9 ** st["t"], 0.999 ** st["t"]
        st["m"], st["v"] = 0.1 * rng.randn(R, n), 0.01 * rng.rand(R, n)
    return st


def _packed(R, n, rng, scale=1.0):
    p = np.zeros((R, n + 2))
    p[:, 0] = rng.randn(R)
    p[:, 2:] = scale * rng.randn(R, n)
    return p


ADAM_CASES = ["first_step", "skipped", "clip_above", "clip_at", "no_clip", "steps_differ", "zero_grad",
              "trace_beyond", "large_n"]


@pytest.mark.parametrize("case", ADAM_CASES)
def test_host_adam_matches_the_oracle_bitwise(host, case):
    rng = np.random.RandomState(ADAM_CASES.index(case))
    R, n, k, rows = 4, 37, 2, 5
    lr, b1, b2, eps, max_norm = 1e-2, 0.9, 0.999, 1e-8, 0.0
    st, packed = _state(R, n, rng), _packed(R, n, rng)
    if case == "skipped":                                            # a status, a NaN loss, an inf gradient entry
        packed[0, 1] = 1.0
        packed[1, 0] = np.nan
        packed[2, 5] = np.inf
        st = _state(R, n, rng, steps=[3, 4, 5, 6])
    elif case == "clip_above":
        max_norm = 0.5 * np.sqrt(so.sumsq(packed[1, 2:]))
    elif case == "clip_at":                                          # exactly at the bound: no clip
        max_norm = np.sqrt(so.sumsq(packed[1, 2:]))
    elif case == "no_clip":
        max_norm = 1e6
    elif case == "steps_differ":
        st = _state(R, n, rng, steps=[0, 1, 7, 100])
    elif case == "zero_grad":
        packed[:, 2:] = 0.0
        packed[3, 2:] = -0.0
        st = _state(R, n, rng, steps=[0, 2, 3, 4])
    elif case == "trace_beyond":
        k = rows + 3
    elif case == "large_n":
        n = 4545
        st, packed = _state(R, n, rng, steps=[1, 2, 3, 4]), _packed(R, n, rng, 1e3)
        max_norm = 10.0
    hyper = (lr, b1, b2, eps, max_norm)
    got = _host_adam(host, st, packed, k, hyper, rows)
    trace0, ok0 = np.full((rows, R), np.nan), np.zeros((rows, R), dtype=np.int32)
    ref = so.adam(st["theta"], packed, st["m"], st["v"], st["t"], st["b1t"], st["b2t"], k, trace0, ok0, *hyper)
    for key in ("theta", "m", "v", "t", "b1t", "b2t", "trace", "ok", "iter"):
        assert np.array_equal(np.asarray(got[key]), np.asarray(ref[key]), equal_nan=True), key
    if case == "skipped":
        for r in range(3):
            assert np.array_equal(got["theta"][r], st["theta"][r]) and got["t"][r] == st["t"][r]
            assert not got["ok"][k, r]
        assert got["ok"][k, 3] and got["t"][3] == 7
    if case == "first_step":                                         # bias-corrected: each step is about lr in size
        assert np.allclose(np.abs(got["theta"] - st["theta"]), lr, rtol=1e-4)
    if case == "trace_beyond":
        assert np.isnan(got["trace"]).all() and got["iter"] == k + 1
    if case == "zero_grad":
        assert np.array_equal(got["m"], 0.9 * st["m"]) and (got["t"] == st["t"] + 1).all()


# ---- the kernels -------------------------------------------------------------------------------------------------------
NEW_KERNELS = ("sgd_normals_kernel", "sgd_adam_kernel", "sgd_tick_kernel")


def test_new_kernels_do_not_spill():
    nvcc = "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not installed")
    res = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas", "-v",
                          "-cubin", "-o", os.devnull, os.path.join(ROOT, "pilco_b200", "csrc", "particles_sgd.cu")],
                         capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    props = dict(re.findall(r"Function properties for (\S+)\n\s*(.*)", res.stderr))
    for k in NEW_KERNELS:
        name = next(n for n in props if re.search(r"\d%s" % k, n))
        assert "0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads" in props[name], (k, props[name])
    if os.path.exists(CUOBJDUMP):
        text = sass_named(list(NEW_KERNELS))
        assert len(text) == len(NEW_KERNELS) and not any(re.search(r"\b(STL|LDL)\b", t) for t in text.values())
        assert not any(re.search(r"\s(ATOMG?|ATOMS|RED)\.", t) for t in text.values())   # no atomics


# ---- refusals before device work ---------------------------------------------------------------------------------------
def test_engine_refusals_before_device_work(monkeypatch):
    import torch
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)
    for kw, what in ((dict(lr=0.0), "learning_rate"), (dict(lr=np.inf), "learning_rate"),
                     (dict(betas=(1.0, 0.9)), "betas"), (dict(betas=(0.9, -0.1)), "betas"), (dict(eps=0.0), "eps"),
                     (dict(max_norm=-1.0), "max_grad_norm"), (dict(max_norm=np.nan), "max_grad_norm")):
        with pytest.raises(ValueError, match=what):
            engine.AdamState(2, 5, **kw)
    for R, n, rows in ((0, 5, 0), (2, 0, 0), (2, 5, -1)):
        with pytest.raises(ValueError, match="R >= 1"):
            engine.AdamState(R, n, trace_rows=rows)
    assert engine.adam_hyperparameters(1e-3, (0.9, 0.999), 1e-8, None) == (1e-3, 0.9, 0.999, 1e-8, 0.0)
    cpu = torch.zeros(4, dtype=torch.float64)
    it = torch.zeros(1, dtype=torch.int64)
    with pytest.raises(ValueError, match="out"):
        engine.normals(cpu, 1, 0, it)
    with pytest.raises(ValueError, match="out"):
        engine.normals(np.zeros(4), 1, 0, it)


def _pilco(controller=None, **kw):
    from pilco.models import PILCO
    rng = np.random.RandomState(0)
    return PILCO((rng.rand(20, 3), 0.1 * rng.rand(20, 2)), controller=controller, horizon=4, **kw)


def test_class_refusals_before_device_work(monkeypatch):
    import torch
    from pilco_b200 import policy_opt
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)
    p = _pilco()
    flat = p.controller.get_flat().copy()
    adam = lambda q=p, **kw: q.optimize_policy_sampled(**dict(dict(maxiter=5, num_samples=8, optimizer="adam"), **kw))
    with pytest.raises(ValueError, match="optimizer"):
        p.optimize_policy_sampled(optimizer="sgd")
    with pytest.raises(ValueError, match="maxiter"):
        adam(maxiter=0)
    for kw, what in ((dict(learning_rate=0.0), "learning_rate"), (dict(learning_rate=-1.0), "learning_rate"),
                     (dict(learning_rate=np.nan), "learning_rate"), (dict(betas=(0.9, 1.0)), "betas"),
                     (dict(eps=0.0), "eps"), (dict(max_grad_norm=-0.5), "max_grad_norm")):
        with pytest.raises(ValueError, match=what):
            adam(**kw)
    with pytest.raises(ValueError, match="num_samples"):
        adam(num_samples=0)
    with pytest.raises(ValueError, match="resample"):
        adam(resample=True, consistent=True)
    with pytest.raises(ValueError, match="exploration"):
        adam(exploration=0.5, num_samples=1)
    with pytest.raises(ValueError, match="consistent"):
        adam(num_features=16)
    with pytest.raises(ValueError, match="measurement_noise"):
        adam(_pilco(measurement_noise=[0.1, 0.1]))
    with pytest.raises((ValueError, TypeError), match="TimeVaryingLinearController"):
        adam(_pilco(controllers.TimeVaryingLinearController(2, 1, 4)))
    with pytest.raises(ValueError, match="box"):
        adam(_safe_pilco())
    with pytest.raises(ValueError, match="box"):
        policy_opt.StochasticEvaluator(_safe_pilco(), 2, np.zeros((2, 5)), 8, 0, np.zeros(4), np.eye(4))
    with pytest.raises(ValueError, match="learning_rate"):
        policy_opt.StochasticEvaluator(p, 2, np.zeros((2, flat.size)), 8, 0, np.zeros(2), np.eye(2), lr=0.0)
    with pytest.raises(ValueError, match="maxiter"):
        policy_opt.optimize_stochastic(p, 0, 2, 8, 0)
    assert np.array_equal(p.controller.get_flat(), flat)
    assert not hasattr(p, "adam_trace")
