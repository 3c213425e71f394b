"""CPU tests of GP prediction at deterministic inputs (pilco_gp_predict, GPRModel.predict_f / predict_y /
predict_log_density): the (iK, beta) identity the kernel relies on against GPflow's Cholesky forms, host-side argument
validation of the C entry point, the workspace bound, the GPflow method surface, the no-GPU failure, and the SASS of
the kernel."""
import ctypes as C
import functools
import inspect
import os
import re

import numpy as np
import pytest
import torch

from oracle import python_port as pp
from pilco_b200._lib import lib
import abi_fakes
from abi_fakes import ERR_ALIGN, ERR_DIM, ERR_NULL, ERR_UNSUP, ERR_WS, FAKE
from predict_oracle import fitc_predict_f, gpr_predict_f, ik_beta_predict
from util import CUOBJDUMP, sass, scaled_err


def _recipe(N, seed=0, d=3, k=2):
    """test_predictions.py's data (X = rand(N,d), Y = sin(X) A + noise) with seeded benign hyper-parameters."""
    rng = np.random.RandomState(seed)
    X = rng.rand(N, d)
    A = rng.rand(d, k)
    Y = np.sin(X).dot(A) + 1e-3 * (rng.rand(N, k) - 0.5)
    ell = 1.0 + rng.rand(k, d)
    sf2 = 1.0 + rng.rand(k)
    sn2 = 1e-2 * np.ones(k)
    Xs = rng.rand(40, d) * 1.2 - 0.1
    return X, Y, ell, sf2, sn2, Xs


def test_ik_beta_form_equals_gpflow_gpr():
    X, Y, ell, sf2, sn2, Xs = _recipe(100)
    iK, beta = pp.calculate_factorizations(X, Y, ell, sf2, sn2)
    for e in range(Y.shape[1]):
        m_ref, v_ref = gpr_predict_f(X, Y[:, e], ell[e], sf2[e], sn2[e], Xs)
        m, v = ik_beta_predict(X, ell[e], sf2[e], iK[e], beta[e], Xs)
        assert scaled_err(m, m_ref) <= 1e-10
        assert np.max(np.abs(v - v_ref)) / sf2[e] <= 1e-10
        _, c_ref = gpr_predict_f(X, Y[:, e], ell[e], sf2[e], sn2[e], Xs, full_cov=True)
        assert np.allclose(np.diag(c_ref), v_ref, rtol=0, atol=1e-12 * sf2[e])


def test_ik_beta_form_equals_gpflow_fitc_with_per_output_z():
    X, Y, ell, sf2, sn2, Xs = _recipe(300, seed=1)
    rng = np.random.RandomState(7)
    for e in range(Y.shape[1]):
        Z = rng.rand(50, X.shape[1])                                  # each output its own inducing inputs
        iK, beta = pp.fitc_factorizations(X, Z, Y[:, e:e + 1], ell[e:e + 1], sf2[e:e + 1], sn2[e:e + 1])
        m_ref, v_ref = fitc_predict_f(X, Z, Y[:, e], ell[e], sf2[e], sn2[e], Xs)
        m, v = ik_beta_predict(Z, ell[e], sf2[e], iK[0], beta[0], Xs)
        assert scaled_err(m, m_ref) <= 1e-10
        assert np.max(np.abs(v - v_ref)) / sf2[e] <= 1e-7


_gp = functools.partial(abi_fakes._gp, n=300, D=3, E=2, ldk=320)


def _call(g, e0=0, ne=2, T=10, Xs=FAKE, mean=FAKE, var=FAKE, full_cov=0, ws=FAKE, wsb=1 << 40):
    return lib.pilco_gp_predict(C.byref(g) if g is not None else None, e0, ne, T, Xs, mean, var, full_cov, ws, wsb, None)


def test_predict_argument_validation():
    assert _call(None) == ERR_NULL
    assert _call(_gp(), Xs=None) == ERR_NULL and _call(_gp(), mean=None) == ERR_NULL
    assert _call(_gp(), var=None) == ERR_NULL and _call(_gp(), ws=None) == ERR_NULL
    assert _call(_gp(mode=1)) == ERR_UNSUP
    assert _call(_gp(iK=None)) == ERR_UNSUP
    assert _call(_gp(bs=300 * 3)) == ERR_UNSUP                          # batched (per-restart) model
    assert _call(_gp(), T=0) == ERR_DIM
    assert _call(_gp(), e0=-1) == ERR_DIM
    assert _call(_gp(), e0=1, ne=2) == ERR_DIM                          # e0 + ne > E
    assert _call(_gp(), ne=0) == ERR_DIM
    assert _call(_gp(D=17)) == ERR_DIM                                  # D > PILCO_MAX_D
    assert _call(_gp(E=17), ne=1) == ERR_DIM
    assert _call(_gp(ldk=256)) == ERR_DIM                               # ldk < pilco_pad_n(n)
    assert _call(_gp(iK=FAKE + 8)) == ERR_ALIGN
    assert _call(_gp(ldk=321)) == ERR_ALIGN
    assert _call(_gp(), ws=FAKE + 8) == ERR_ALIGN
    for fc in (0, 1):
        need = lib.pilco_gp_predict_workspace_bytes(300, 3, 2, 10, fc)
        assert need > 0 and _call(_gp(), full_cov=fc, wsb=need - 8) == ERR_WS


def test_predict_workspace_bytes():
    f = lib.pilco_gp_predict_workspace_bytes
    for args in ((0, 3, 2, 10, 0), (300, 0, 2, 10, 0), (300, 17, 2, 10, 0), (300, 3, 0, 10, 0), (300, 3, 17, 10, 0),
                 (300, 3, 2, 0, 0), (300, 3, 2, 0, 1), (300, 3, 2, 65535 * 8 + 1, 1)):
        assert f(*args) == 0, args
    T = 100000
    for n, E in ((300, 10), (2000, 10), (2000, 16), (200, 1)):
        b = f(n, 12, E, T, 0)
        assert 0 < b <= 8 * T * n * E / 50, (n, E, b)                    # no [T, n] intermediate
    assert f(2000, 12, 10, 1000, 1) == 2 * 10 * 1000 * 2048 * 8          # full_cov: K* and K* iK


def test_predict_methods_have_gpflow_signatures():
    from pilco.models.mgpr import GPRModel
    from pilco.models.smgpr import GPRFITCModel
    for cls in (GPRModel, GPRFITCModel):
        for name, first in (("predict_f", "Xnew"), ("predict_y", "Xnew"), ("predict_log_density", "data")):
            sig = inspect.signature(getattr(cls, name))
            assert list(sig.parameters) == ["self", first, "full_cov", "full_output_cov"], (cls, name)
            assert sig.parameters["full_cov"].default is False and sig.parameters["full_output_cov"].default is False


def test_predict_methods_fail_loudly_without_gpu(monkeypatch):
    from pilco.models import MGPR, SMGPR
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)
    X, Y, *_ = _recipe(30)
    for m in (MGPR((X, Y)).models[0], SMGPR((X, Y), 5).models[1]):
        for call in (lambda: m.predict_f(X[:4]), lambda: m.predict_y(X[:4]), lambda: m.predict_log_density((X[:4], Y[:4, :1]))):
            with pytest.raises(RuntimeError, match="CUDA device"):
                call()
    m = MGPR((X, Y)).models[0]
    with pytest.raises(NotImplementedError):
        m.predict_f(X[:4], full_output_cov=True)
    with pytest.raises(NotImplementedError):
        m.predict_y(X[:4], full_cov=True)


@pytest.mark.skipif(not os.path.exists(CUOBJDUMP), reason="cuobjdump not available")
def test_predict_kernel_sass():
    """The quadratic form runs on DMMA.16x8x16 (no 8x8x4), the iK tiles arrive by TMA bulk copy on an mbarrier, and
    nothing touches local memory."""
    funcs = sass(r"gp_predict_kernel")
    assert len(funcs) == 1
    text = next(iter(funcs.values()))
    assert re.search(r"DMMA\.16x8x\d+", text) and "DMMA.8x8x4" not in text
    assert "UBLKCP" in text and "SYNCS.ARRIVE.TRANS64" in text and "TRYWAIT" in text
    assert not re.search(r"\b(STL|LDL)\b", text)
