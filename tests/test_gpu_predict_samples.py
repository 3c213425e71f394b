"""Posterior function samples at deterministic inputs on the device (pilco_gp_predict_samples through
engine.gp_predict_samples and GPRModel.predict_f_samples): parity with the numpy oracle given eps (exact GPs on the
one-CTA and the blocked Cholesky, FITC, both covariance modes), bitwise determinism, the statistics of seeded draws, the
factorisation an MGPR's model samples from, graph replay, and the not-positive-definite return."""
import numpy as np
import pytest
import torch

from oracle import python_port as pp
from pilco_b200 import engine
from predict_samples_oracle import draw, ik_beta_posterior, posterior
from util import make_gp_problem

pytestmark = pytest.mark.gpu


def _inputs(T, D, seed):
    return np.random.RandomState(seed).rand(T, D) * 1.4 - 0.2


def _eps(S, T, ne, seed):
    g = torch.Generator(device=engine.device())
    g.manual_seed(seed)
    return torch.randn((S, T, ne), dtype=engine.F64, device=engine.device(), generator=g)


def _parity(X, Y, ell, sf2, sn2, gp, Xs, e0, ne, S, full_cov, Z=None, bar=1e-10, fact=None):
    """device samples vs the oracle given eps; the bar is ``bar`` of the sample scale, or 4x the oracle's own change
    when its posterior is formed in the (iK, beta) order instead (ill-conditioned covariances), whichever is larger"""
    T = Xs.shape[0]
    eps = _eps(S, T, ne, seed=T + S + ne)
    out, info = engine.gp_predict_samples(gp, Xs, eps, e0=e0, ne=ne, full_cov=full_cov)
    assert out.shape == (S, T, ne) and int(info.abs().max().item()) == 0
    out, eps = out.cpu().numpy(), eps.cpu().numpy()
    iK, beta = fact if fact is not None else pp.calculate_factorizations(X, Y, ell, sf2, sn2)
    C = X if Z is None else Z
    for k, e in enumerate(range(e0, e0 + ne)):
        mean, c = posterior(X, Y[:, e], ell[e], sf2[e], sn2[e], Xs, full_cov=full_cov, Z=Z)
        ref = draw(mean, c, eps[:, :, k], full_cov=full_cov)
        m2, c2 = ik_beta_posterior(C, ell[e], sf2[e], iK[e], beta[e], Xs, full_cov=full_cov)
        own = float(np.max(np.abs(draw(m2, c2, eps[:, :, k], full_cov=full_cov) - ref)))
        scale = float(np.max(np.abs(ref)))
        err = float(np.max(np.abs(out[:, :, k] - ref)))
        print("n=%d T=%d S=%d e=%d full_cov=%d: |device - oracle| %.2e of scale, oracle reordered %.2e"
              % (C.shape[0], T, S, e, full_cov, err / scale, own / scale))
        assert err <= max(bar * scale, 4.0 * own), (err / scale, own / scale)


@pytest.mark.parametrize("n,T", [(300, 64), (300, 1100), (2000, 64), (2000, 1100)])
@pytest.mark.parametrize("full_cov", [True, False])
def test_exact_parity_with_oracle(n, T, full_cov):
    D = 12
    X, Y, ell, sf2, sn2 = make_gp_problem(n, D, 3, seed=n)
    gp = engine.gp_factorize(X, Y, ell, sf2, sn2)
    Xs = _inputs(T, D, seed=T)
    _parity(X, Y, ell, sf2, sn2, gp, Xs, 1, 2, 5, full_cov)                  # ne > 1, from output 1
    _parity(X, Y, ell, sf2, sn2, gp, Xs[:1], 0, 1, 1, full_cov)               # T = 1, S = 1


@pytest.mark.parametrize("full_cov", [True, False])
def test_fitc_parity_with_oracle(full_cov):
    N, M, D = 2000, 200, 3
    X, Y, ell, sf2, sn2 = make_gp_problem(N, D, 1, seed=21)
    Z = np.random.RandomState(22).rand(M, D)
    gp = engine.fitc_factorize(X, Z, Y, ell, sf2, sn2)
    fact = pp.fitc_factorizations(X, Z, Y, ell, sf2, sn2)
    for T in (64, 1100):
        _parity(X, Y, ell, sf2, sn2, gp, _inputs(T, D, seed=23 + T), 0, 1, 4, full_cov, Z=Z, bar=1e-8, fact=fact)


@pytest.mark.parametrize("full_cov", [True, False])
def test_leading_samples_do_not_depend_on_s(full_cov):
    X, Y, ell, sf2, sn2 = make_gp_problem(300, 12, 4, seed=31)
    gp = engine.gp_factorize(X, Y, ell, sf2, sn2)
    Xs = _inputs(600, 12, seed=32)
    eps = _eps(130, 600, 3, seed=33)
    full, _ = engine.gp_predict_samples(gp, Xs, eps, e0=1, ne=3, full_cov=full_cov)
    for s in (1, 7, 64, 65):
        part, _ = engine.gp_predict_samples(gp, Xs, eps[:s].clone(), e0=1, ne=3, full_cov=full_cov)
        assert torch.equal(part, full[:s]), s
    again, _ = engine.gp_predict_samples(gp, Xs, eps, e0=1, ne=3, full_cov=full_cov)
    assert torch.equal(again, full)


def test_diagonal_draw_is_predict_f_bitwise():
    X, Y, ell, sf2, sn2 = make_gp_problem(600, 12, 5, seed=41)
    gp = engine.gp_factorize(X, Y, ell, sf2, sn2)
    Xs = _inputs(3000, 12, seed=42)
    eps = _eps(9, 3000, 3, seed=43)
    out, info = engine.gp_predict_samples(gp, Xs, eps, e0=2, ne=3, full_cov=False)
    mean, var = engine.gp_predict(gp, Xs, e0=2, ne=3)
    assert torch.equal(out, mean[None] + torch.sqrt(var.clamp_min(0.0))[None] * eps)
    assert int(info.abs().max().item()) == 0


def _mgpr(N, seed, sf2=None):
    from pilco.models import MGPR
    rng = np.random.RandomState(seed)
    X = rng.rand(N, 3)
    Y = np.sin(X).dot(rng.rand(3, 2)) + 1e-3 * (rng.rand(N, 2) - 0.5)
    mgpr = MGPR((X, Y))
    for e, m in enumerate(mgpr.models):
        m.kernel.lengthscales.assign(1.0 + rng.rand(3))
        m.kernel.variance.assign(1.0 + rng.rand() if sf2 is None else sf2)
        m.likelihood.variance.assign(1e-2)
    return mgpr, X, Y


def test_seeded_api_statistics():
    mgpr, X, Y = _mgpr(200, seed=51)
    m = mgpr.models[1]
    Xs = _inputs(64, 3, seed=52)
    S = 1 << 16
    smp = np.asarray(m.predict_f_samples(Xs, S, seed=7))
    assert smp.shape == (S, 64, 1)
    assert np.array_equal(smp, np.asarray(m.predict_f_samples(Xs, S, seed=7)))          # same seed, same draw
    assert not np.array_equal(smp[:8], np.asarray(m.predict_f_samples(Xs, 8, seed=8)))
    one = np.asarray(m.predict_f_samples(Xs, seed=7))
    assert one.shape == (64, 1) and np.array_equal(one, smp[0])
    mean, cov = m.predict_f(Xs, full_cov=True)
    target = cov[0] + 1e-6 * np.eye(64)
    z = (smp[:, :, 0].mean(0) - mean[:, 0]) / np.sqrt(np.diag(target) / S)
    print("sample mean: max |z| = %.2f over 64 points" % np.max(np.abs(z)))
    assert np.max(np.abs(z)) < 5.0
    # whitened draws W = L^-1 (samples - mean) with the oracle's L have identity covariance.  Off the diagonal
    # S C_ij^2 ~ chi2_1 each, so their sum over the k = 2016 pairs ~ chi2_k: bound k + 5 sqrt(2k); on the diagonal
    # |C_ii - 1| <= 5 sqrt(2 / S).
    _, c_or = posterior(mgpr.X, mgpr.Y[:, 1], np.asarray(m.kernel.lengthscales), float(m.kernel.variance),
                        float(m.likelihood.variance), Xs)
    L = np.linalg.cholesky(c_or + 1e-6 * np.eye(64))
    W = np.linalg.solve(L, (smp[:, :, 0] - mean[:, 0]).T)
    Cw = W @ W.T / S
    k = 64 * 63 // 2
    chi2 = S * float((Cw[np.triu_indices(64, 1)] ** 2).sum())
    print("whitened: chi2 of the off-diagonal %.0f (k = %d), max |C_ii - 1| %.4f" % (chi2, k, np.max(np.abs(np.diag(Cw) - 1))))
    assert chi2 < k + 5.0 * np.sqrt(2.0 * k)
    assert np.max(np.abs(np.diag(Cw) - 1.0)) < 5.0 * np.sqrt(2.0 / S)
    marg = np.asarray(m.predict_f_samples(Xs, S, full_cov=False, seed=9))[:, :, 0]
    _, var = m.predict_f(Xs)
    assert np.max(np.abs(marg.mean(0) - mean[:, 0]) / np.sqrt(var[:, 0] / S)) < 5.0
    assert np.max(np.abs(marg.var(0) / var[:, 0] - 1.0)) < 5.0 * np.sqrt(2.0 / S)


def test_mgpr_model_samples_from_the_appended_factorisation():
    mgpr, X, Y = _mgpr(400, seed=61)
    mgpr.set_data((X[:300], Y[:300]))
    m = mgpr.models[0]
    Xs = _inputs(50, 3, seed=62)
    before = np.asarray(m.predict_f_samples(Xs, 4, seed=3))
    mgpr.set_data((X, Y))
    after = np.asarray(m.predict_f_samples(Xs, 4, seed=3))
    assert mgpr.last_update == "append"
    mean, cov = m.predict_f(Xs, full_cov=True)
    eps = _eps(4, 50, 1, seed=3).cpu().numpy()[:, :, 0]                      # the API's draw for seed 3
    ref = draw(mean[:, 0], cov[0], eps)
    scale = float(np.max(np.abs(ref)))
    err = float(np.max(np.abs(after[:, :, 0] - ref))) / scale
    print("appended model vs predict_f's covariance: %.2e of scale; change from the old model %.2e"
          % (err, float(np.max(np.abs(after - before))) / scale))
    assert err <= 1e-8
    assert float(np.max(np.abs(after - before))) / scale > 1e-6


def test_graph_capture_replays_bitwise():
    X, Y, ell, sf2, sn2 = make_gp_problem(300, 12, 2, seed=71)
    gp = engine.gp_factorize(X, Y, ell, sf2, sn2)
    Xs = engine.dev(_inputs(700, 12, seed=72))
    eps = _eps(16, 700, 2, seed=73)
    ref = [engine.gp_predict_samples(gp, Xs, eps, full_cov=fc)[0] for fc in (True, False)]
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        outs = [engine.gp_predict_samples(gp, Xs, eps, full_cov=fc)[0] for fc in (True, False)]
    g.replay()
    torch.cuda.synchronize()
    for a, b in zip(outs, ref):
        assert torch.equal(a, b)


def test_workspace_limit_is_a_value_error():
    X, Y, ell, sf2, sn2 = make_gp_problem(300, 12, 1, seed=81)
    gp = engine.gp_factorize(X, Y, ell, sf2, sn2)
    Xs = _inputs(1000, 12, seed=82)
    need = engine.predict_samples_workspace_bytes(gp, 1000, 2)
    with pytest.raises(ValueError, match=r"need %d workspace bytes.*T=\d+ would fit" % need):
        engine.gp_predict_samples(gp, Xs, _eps(2, 1000, 1, seed=1), max_ws_bytes=need // 4)


def test_not_positive_definite_is_reported(monkeypatch):
    """Two equal input rows far from the data: the covariance is exactly sf2 11' there (sf2 = 1), singular without
    jitter.  The engine returns info != 0 (an ordinary return code); the API raises."""
    mgpr, X, Y = _mgpr(100, seed=91, sf2=1.0)
    Xs = np.array([[50.0, 50.0, 50.0], [50.0, 50.0, 50.0], [60.0, 50.0, 50.0]])
    gp = mgpr.device_gp()
    _, info = engine.gp_predict_samples(gp, Xs, _eps(2, 3, 2, seed=1), full_cov=True, jitter=0.0)
    assert info.cpu().numpy().tolist()[0] != 0 and info.cpu().numpy().tolist()[1] != 0
    _, info = engine.gp_predict_samples(gp, Xs, _eps(2, 3, 2, seed=1), full_cov=True)        # default jitter: fine
    assert int(info.abs().max().item()) == 0
    real = engine.gp_predict_samples
    monkeypatch.setattr(engine, "gp_predict_samples", lambda *a, **k: real(*a, **dict(k, jitter=0.0)))
    with pytest.raises(RuntimeError, match="Cholesky decomposition was not successful"):
        mgpr.models[0].predict_f_samples(Xs, 2, seed=0)
