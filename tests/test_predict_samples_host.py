"""CPU tests of posterior function samples at deterministic inputs (pilco_gp_predict_samples, GPRModel.predict_f_samples):
the numpy oracle's statistics, the workspace sizes, host-side argument validation of the C entry point (fake non-null
pointers as in test_abi_errors.py: only rejected calls are made), the GPflow method surface, the no-GPU failure, and the
SASS of the new kernels."""
import ctypes as C
import inspect
import os
import re

import numpy as np
import pytest
import torch

from pilco_b200._lib import lib
from predict_samples_oracle import predict_f_samples
from abi_fakes import ERR_ALIGN, ERR_DIM, ERR_NULL, ERR_UNSUP, ERR_WS, FAKE, _gp
from util import CUOBJDUMP, make_gp_problem, sass

WSB = lambda *a: int(lib.pilco_gp_predict_samples_workspace_bytes(*a))
PRED = lambda *a: int(lib.pilco_gp_predict_workspace_bytes(*a))


@pytest.mark.parametrize("Z", [False, True])
def test_oracle_draws_have_the_posterior_moments(Z):
    X, Y, ell, sf2, sn2 = make_gp_problem(120, 2, 1, seed=3)
    Zs = np.random.RandomState(4).rand(20, 2) if Z else None
    Xs = np.random.RandomState(5).rand(12, 2) * 1.4 - 0.2
    S = 200000
    eps = np.random.RandomState(6).randn(S, 12)
    smp, mean, cov = predict_f_samples(X, Y[:, 0], ell[0], sf2[0], sn2[0], Xs, eps, Z=Zs)
    target = cov + 1e-6 * np.eye(12)
    emp = np.cov(smp.T)
    # entrywise standard error of a sample covariance: sqrt((c_ii c_jj + c_ij^2) / S)
    se = np.sqrt((np.outer(np.diag(target), np.diag(target)) + target ** 2) / S)
    assert np.max(np.abs(emp - target) / se) < 5.5
    assert np.max(np.abs(smp.mean(0) - mean) / np.sqrt(np.diag(target) / S)) < 5.5
    smp_d, mean_d, var = predict_f_samples(X, Y[:, 0], ell[0], sf2[0], sn2[0], Xs, eps, full_cov=False, Z=Zs)
    assert np.allclose(var, np.diag(cov), rtol=0, atol=1e-10 * sf2[0]) and np.array_equal(mean_d, mean)
    se_v = var * np.sqrt(2.0 / S)
    assert np.max(np.abs(smp_d.var(0) - var) / se_v) < 5.5
    # independent points: no correlation between the marginal draws
    assert np.max(np.abs(np.corrcoef(smp_d.T) - np.eye(12))) < 5.5 / np.sqrt(S)


def test_oracle_negative_variance_gives_the_mean():
    mean, var = np.array([1.0, 2.0]), np.array([-1e-18, 4.0])
    from predict_samples_oracle import draw
    out = draw(mean, var, np.ones((1, 2)), full_cov=False)
    assert np.array_equal(out, [[1.0, 4.0]])


def test_workspace_bytes():
    n, D = 300, 12
    # diagonal path: O(T) and independent of S
    for T in (1, 1000, 100000, 65535 * 32):
        for E in (1, 10):
            b = WSB(n, D, E, T, 1, 0)
            assert b == WSB(n, D, E, T, 1 << 20, 0)
            assert b == ((PRED(n, D, E, T, 0) + 15) & ~15) + 2 * T * E * 8
            assert b <= 8 * E * (T + 32) * 16                                # O(T): no [T,T] or [T,n] array
    # full covariance: max(predict workspace, eps' and L eps) + covariance + mean
    for E, T, S in ((1, 64, 1), (3, 1100, 256), (2, 4096, 1), (1, 1024, 1 << 14)):
        pb = PRED(n, D, E, T, 1)
        assert WSB(n, D, E, T, S, 1) == max(pb, 2 * S * T * E * 8) + 8 * E * T * T + 8 * T * E, (E, T, S)
    assert WSB(2000, 12, 1, 64, 1, 1) == 2 * 64 * 2048 * 8 + 8 * 64 * 64 + 8 * 64
    # unsupported arguments and the GEMM leading dimension ne*S overflowing an int
    for args in ((0, D, 1, 10, 1, 1), (n, 0, 1, 10, 1, 1), (n, 17, 1, 10, 1, 0), (n, D, 0, 10, 1, 1), (n, D, 17, 10, 1, 0),
                 (n, D, 1, 0, 1, 1), (n, D, 1, 10, 0, 0), (n, D, 1, 10, 0, 1), (n, D, 1, 65535 * 8 + 1, 1, 1),
                 (n, D, 1, 65535 * 32 + 1, 1, 0), (n, D, 2, 10, 2 ** 30, 1), (n, D, 16, 10, 2 ** 27, 1)):
        assert WSB(*args) == 0, args
    assert WSB(n, D, 16, 10, 2 ** 27 - 1, 1) > 0


def _call(g=None, e0=0, ne=2, T=10, S=4, Xs=FAKE, eps=FAKE, out=FAKE, full_cov=1, jitter=1e-6, info=FAKE, ws=FAKE,
          wsb=1 << 40, gp=True):
    g = _gp() if g is None and gp else g
    return lib.pilco_gp_predict_samples(C.byref(g) if g is not None else None, e0, ne, T, S, Xs, eps, out, full_cov,
                                        jitter, info, ws, wsb, None)


def test_argument_validation():
    assert _call(gp=False) == ERR_NULL
    for k in ("Xs", "eps", "out", "info", "ws"):
        assert _call(**{k: None}) == ERR_NULL, k
    assert _call(_gp(mode=1)) == ERR_UNSUP
    assert _call(_gp(iK=None)) == ERR_UNSUP
    for fc in (0, 1):
        assert _call(full_cov=fc, T=0) == ERR_DIM
        assert _call(full_cov=fc, S=0) == ERR_DIM
        assert _call(full_cov=fc, ne=0) == ERR_DIM
        assert _call(full_cov=fc, e0=-1) == ERR_DIM
        assert _call(full_cov=fc, e0=2, ne=2) == ERR_DIM                    # e0 + ne > E = 3
        for j in (-1e-6, float("nan"), float("inf"), -float("inf")):
            assert _call(full_cov=fc, jitter=j) == ERR_DIM, (fc, j)
        assert _call(_gp(D=17), full_cov=fc) == ERR_DIM
        assert _call(_gp(ldk=32), full_cov=fc) == ERR_DIM
        assert _call(_gp(iK=FAKE + 8), full_cov=fc) == ERR_ALIGN
        assert _call(_gp(ldk=65), full_cov=fc) == ERR_ALIGN
        assert _call(full_cov=fc, ws=FAKE + 8) == ERR_ALIGN
        need = WSB(50, 4, 2, 10, 4, fc)
        assert need > 0 and _call(full_cov=fc, wsb=need - 8) == ERR_WS
    assert _call(full_cov=1, T=65535 * 8 + 1) == ERR_DIM                     # pilco_gp_predict's T limits
    assert _call(full_cov=0, T=65535 * 32 + 1) == ERR_DIM
    assert _call(full_cov=1, S=2 ** 30) == ERR_DIM                           # ne S overflows the GEMM leading dimension
    assert _call(full_cov=0, jitter=0.0, wsb=0) == ERR_WS                     # jitter 0 is valid


def test_predict_f_samples_has_gpflow_signature():
    from pilco.models.mgpr import GPRModel
    from pilco.models.smgpr import GPRFITCModel
    for cls in (GPRModel, GPRFITCModel):
        sig = inspect.signature(cls.predict_f_samples)
        assert list(sig.parameters)[:5] == ["self", "Xnew", "num_samples", "full_cov", "full_output_cov"]
        p = sig.parameters
        assert p["num_samples"].default is None and p["full_cov"].default is True and p["full_output_cov"].default is False
        assert p["seed"].kind is inspect.Parameter.KEYWORD_ONLY and p["seed"].default is None


def test_predict_f_samples_fails_loudly_without_gpu(monkeypatch):
    from pilco.models import MGPR, SMGPR
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)
    X, Y, *_ = make_gp_problem(30, 3, 2)
    for m in (MGPR((X, Y)).models[0], SMGPR((X, Y), 5).models[1]):
        for fc in (True, False):
            with pytest.raises(RuntimeError, match="CUDA device"):
                m.predict_f_samples(X[:4], 3, full_cov=fc)
        with pytest.raises(RuntimeError, match="CUDA device"):
            m.predict_f_samples(X[:4])
        for bad in (0, -1, 2.0, 1.5, "3", True, np.float64(4)):
            with pytest.raises(ValueError, match="num_samples"):
                m.predict_f_samples(X[:4], bad)
        with pytest.raises(NotImplementedError):
            m.predict_f_samples(X[:4], 3, full_output_cov=True)
        with pytest.raises(RuntimeError, match="CUDA device"):
            m.predict_f_samples(X[:4], np.int64(3), seed=1)                   # numpy integers are integers


@pytest.mark.skipif(not os.path.exists(CUOBJDUMP), reason="cuobjdump not available")
def test_sample_kernels_sass():
    """The three new kernels exist and touch no local memory (no spills)."""
    funcs = sass(r"gp_sample_")
    names = sorted(re.search(r"gp_sample_\w+?_kernel", k).group(0) for k in funcs)
    assert names == ["gp_sample_diag_kernel", "gp_sample_transpose_kernel", "gp_sample_tril_kernel"], names
    for name, text in funcs.items():
        assert not re.search(r"\b(STL|LDL)\b", text), name
