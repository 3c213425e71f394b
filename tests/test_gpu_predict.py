"""GP prediction at deterministic inputs on the device (pilco_gp_predict through engine.gp_predict and the GPflow
methods GPRModel.predict_f / predict_y / predict_log_density): kernel arithmetic against a numpy contraction of the
same device factors, end-to-end agreement with GPflow's Cholesky forms (tests/predict_oracle.py), bitwise independence
of a point's result from its batch, the full covariance, the factorisation each model predicts from, and CUDA-graph
replay."""
import numpy as np
import pytest
import scipy.stats
import torch

from pilco_b200 import engine
from predict_oracle import fitc_predict_f, gpr_predict_f, se_ard
from util import make_gp_problem, scaled_err

pytestmark = pytest.mark.gpu


def _inputs(T, D, seed):
    return np.random.RandomState(seed).rand(T, D) * 1.4 - 0.2


def _host_contraction(gp, Xs, e0, ne):
    """mean, var and the error scales sum|k beta|, sum|k_i iK_ij k_j| from the device factors, in numpy"""
    n = gp.n
    C, ell, sf2 = gp.X.cpu().numpy(), gp.ell.cpu().numpy(), gp.sf2.cpu().numpy()
    iK, beta = gp.iK[:, :n, :n].cpu().numpy(), gp.beta.cpu().numpy()
    out = []
    for e in range(e0, e0 + ne):
        K = se_ard(Xs, C, ell[e], sf2[e])
        W = K @ iK[e]
        out.append((K @ beta[e], sf2[e] - (W * K).sum(1), np.abs(K) @ np.abs(beta[e]),
                    ((np.abs(K) @ np.abs(iK[e])) * np.abs(K)).sum(1)))
    return [np.stack(v, 1) for v in zip(*out)]


@pytest.mark.parametrize("n,D,E,T,e0,ne", [
    (1, 1, 1, 1, 0, 1), (37, 3, 2, 30, 0, 2), (37, 16, 3, 4099, 1, 2), (300, 12, 10, 1000, 0, 10),
    (300, 1, 16, 30, 5, 7), (600, 16, 16, 4099, 0, 16), (2000, 12, 4, 1000, 2, 1), (2000, 3, 2, 4099, 0, 2)])
def test_kernel_arithmetic_against_device_factors(n, D, E, T, e0, ne):
    X, Y, ell, sf2, sn2 = make_gp_problem(n, D, E, seed=n + D)
    gp = engine.gp_factorize(X, Y, ell, sf2, sn2)
    Xs = _inputs(T, D, seed=T)
    mean, var = engine.gp_predict(gp, Xs, e0=e0, ne=ne)
    assert mean.shape == (T, ne) and var.shape == (T, ne)
    m_ref, v_ref, m_sc, v_sc = _host_contraction(gp, Xs, e0, ne)
    em = float(np.max(np.abs(mean.cpu().numpy() - m_ref) / m_sc))
    ev = float(np.max(np.abs(var.cpu().numpy() - v_ref) / v_sc))
    print("kernel vs device factors n=%d D=%d E=%d T=%d: mean %.2e, var %.2e (relative to sum |k iK k|)" % (n, D, E, T, em, ev))
    assert em <= 1e-12 and ev <= 1e-12


def _set_hypers(models, ell, sf2, sn2):
    for e, m in enumerate(models):
        m.kernel.lengthscales.assign(ell[e])
        m.kernel.variance.assign(sf2[e])
        m.likelihood.variance.assign(sn2[e])


def _recipe(N, seed=0, d=3, k=2):
    """test_predictions.py's data with seeded benign hyper-parameters (sn2 = 1e-2)"""
    rng = np.random.RandomState(seed)
    X = rng.rand(N, d)
    A = rng.rand(d, k)
    Y = np.sin(X).dot(A) + 1e-3 * (rng.rand(N, k) - 0.5)
    return X, Y, 1.0 + rng.rand(k, d), 1.0 + rng.rand(k), 1e-2 * np.ones(k)


@pytest.mark.parametrize("N", [100, 600])
def test_mgpr_models_match_gpflow_gpr(N):
    from pilco.models import MGPR
    X, Y, ell, sf2, sn2 = _recipe(N)
    mgpr = MGPR((X, Y))
    _set_hypers(mgpr.models, ell, sf2, sn2)
    Xs = _inputs(500, 3, seed=5)
    for e, m in enumerate(mgpr.models):
        mean, var = m.predict_f(Xs)
        assert mean.shape == (500, 1) and var.shape == (500, 1)
        m_ref, v_ref = gpr_predict_f(X, Y[:, e], ell[e], sf2[e], sn2[e], Xs)
        em, ev = scaled_err(mean[:, 0], m_ref), float(np.max(np.abs(var[:, 0] - v_ref))) / sf2[e]
        print("GPR N=%d output %d vs GPflow form: mean %.2e of scale, var %.2e of sf2" % (N, e, em, ev))
        assert em <= 1e-9 and ev <= 1e-8
        mean_c, cov = m.predict_f(Xs[:200], full_cov=True)
        assert cov.shape == (1, 200, 200)
        _, c_ref = gpr_predict_f(X, Y[:, e], ell[e], sf2[e], sn2[e], Xs[:200], full_cov=True)
        assert float(np.max(np.abs(cov[0] - c_ref))) / sf2[e] <= 1e-8
        _, _, m_sc, v_sc = _host_contraction(mgpr.device_gp(), Xs[:200], e, 1)
        assert np.max(np.abs(mean_c - mean[:200]) / m_sc) <= 1e-12
        assert np.max(np.abs(np.diag(cov[0]) - var[:200, 0]) / v_sc[:, 0]) <= 1e-12
        assert float(np.max(np.abs(cov[0] - cov[0].T))) / float(v_sc.max()) <= 1e-12


@pytest.mark.parametrize("N,M", [(300, 50), (2000, 200)])
def test_gprfitc_models_match_gpflow_fitc_with_their_own_z(N, M):
    from pilco.models import SMGPR
    X, Y, ell, sf2, sn2 = _recipe(N, seed=1)
    smgpr = SMGPR((X, Y), M)
    _set_hypers(smgpr.models, ell, sf2, sn2)
    rng = np.random.RandomState(11)
    for m in smgpr.models:                                             # per-output inducing inputs
        m.inducing_variable.Z.assign(rng.rand(M, 3))
    assert not np.array_equal(np.asarray(smgpr.models[1].inducing_variable.Z), np.asarray(smgpr.Z))
    Xs = _inputs(1000, 3, seed=6)
    bar = 1e-9 if N <= 300 else 1e-6
    vbar = 1e-7 if N <= 300 else 1e-6
    for e, m in enumerate(smgpr.models):
        mean, var = m.predict_f(Xs)
        m_ref, v_ref = fitc_predict_f(X, np.asarray(m.inducing_variable.Z), Y[:, e], ell[e], sf2[e], sn2[e], Xs)
        em, ev = scaled_err(mean[:, 0], m_ref), float(np.max(np.abs(var[:, 0] - v_ref))) / sf2[e]
        print("FITC N=%d M=%d output %d vs GPflow form: mean %.2e of scale, var %.2e of sf2" % (N, M, e, em, ev))
        assert em <= bar and ev <= vbar


def test_batch_position_and_output_subset_are_bitwise_independent():
    X, Y, ell, sf2, sn2 = make_gp_problem(300, 12, 10, seed=2)
    gp = engine.gp_factorize(X, Y, ell, sf2, sn2)
    Xs = _inputs(4099, 12, seed=3)
    mean, var = engine.gp_predict(gp, Xs)
    for a, b in ((0, 1), (17, 50), (31, 33), (1000, 4099), (4098, 4099)):
        m2, v2 = engine.gp_predict(gp, Xs[a:b])
        assert torch.equal(m2, mean[a:b]) and torch.equal(v2, var[a:b]), (a, b)
    perm = np.random.RandomState(0).permutation(4099)
    mp, vp = engine.gp_predict(gp, Xs[perm])
    assert torch.equal(mp, mean[perm]) and torch.equal(vp, var[perm])
    for e0, ne in ((0, 1), (3, 1), (9, 1), (2, 5)):
        m1, v1 = engine.gp_predict(gp, Xs, e0=e0, ne=ne)
        assert torch.equal(m1, mean[:, e0:e0 + ne]) and torch.equal(v1, var[:, e0:e0 + ne]), (e0, ne)


def test_predict_y_and_log_density_match_scipy():
    from pilco.models import MGPR
    X, Y, ell, sf2, sn2 = _recipe(200, seed=4)
    mgpr = MGPR((X, Y))
    _set_hypers(mgpr.models, ell, sf2, sn2)
    Xs = _inputs(300, 3, seed=8)
    Ys = np.sin(Xs).dot(np.random.RandomState(4).rand(3, 2))
    for e, m in enumerate(mgpr.models):
        mean, var = m.predict_f(Xs)
        my, vy = m.predict_y(Xs)
        assert np.array_equal(my, mean) and np.allclose(vy, var + sn2[e], rtol=0, atol=1e-15)
        ld = m.predict_log_density((Xs, Ys[:, e:e + 1]))
        assert ld.shape == (300,)
        ref = scipy.stats.norm.logpdf(Ys[:, e], loc=mean[:, 0], scale=np.sqrt(var[:, 0] + sn2[e]))
        assert np.max(np.abs(ld - ref)) <= 1e-10 * np.max(np.abs(ref))
        assert type(ld).__name__ == "HostArray" and type(my).__name__ == "HostArray"


def test_factorisation_follows_the_model():
    from pilco.models import MGPR
    X, Y, ell, sf2, sn2 = _recipe(400, seed=9)
    mgpr = MGPR((X[:300], Y[:300]))
    _set_hypers(mgpr.models, ell, sf2, sn2)
    Xs = _inputs(200, 3, seed=10)

    def check(Xd, Yd, what, bar=1e-9):
        for e, m in enumerate(mgpr.models):
            mean, var = m.predict_f(Xs)
            m_ref, v_ref = gpr_predict_f(Xd, Yd[:, e], np.asarray(m.kernel.lengthscales), float(m.kernel.variance),
                                         float(m.likelihood.variance), Xs)
            assert scaled_err(mean[:, 0], m_ref) <= bar, what
            assert float(np.max(np.abs(var[:, 0] - v_ref))) / float(m.kernel.variance) <= 10 * bar, what

    check(X[:300], Y[:300], "initial")
    gp0 = mgpr.device_gp()
    mgpr.set_data((X, Y))                                              # appended rows: the owner's O(n^2 k) update
    check(X, Y, "append")
    assert mgpr.last_update == "append" and mgpr.device_gp() is not gp0
    mgpr.set_data((X[::-1].copy(), Y[::-1].copy()))                    # not an append: refactorisation
    check(X[::-1], Y[::-1], "refactorise")
    assert mgpr.last_update == "factorize"
    ell0 = mgpr.lengthscales.copy()
    mgpr.optimize(maxiter=20)                                          # new hyper-parameters (trained noise can be
    assert not np.array_equal(mgpr.lengthscales, ell0)                 # small: iK less well conditioned)
    check(X[::-1], Y[::-1], "optimize", bar=1e-6)
    m0 = mgpr.models[0]                                                # own data set directly: own factorisation
    m0.data = (X[:100], Y[:100, :1])
    mean, _ = m0.predict_f(Xs)
    m_ref, _ = gpr_predict_f(X[:100], Y[:100, 0], np.asarray(m0.kernel.lengthscales), float(m0.kernel.variance),
                             float(m0.likelihood.variance), Xs)
    assert scaled_err(mean[:, 0], m_ref) <= 1e-9


def test_notebook_validation_loop_runs_on_mgpr_and_smgpr():
    """examples/Hyperparameter setting and troubleshooting tips.ipynb, cell 6: predict_y of every output model."""
    from pilco.models import MGPR, SMGPR
    X, Y, ell, sf2, sn2 = _recipe(300, seed=12)
    X_new = _inputs(50, 3, seed=13)
    for model in (MGPR((X, Y)), SMGPR((X, Y), 30)):
        _set_hypers(model.models, ell, sf2, sn2)
        for i, m in enumerate(model.models):
            y_pred_test, var_pred_test = m.predict_y(X_new)
            assert y_pred_test.shape == (50, 1) and var_pred_test.shape == (50, 1)
            assert np.all(np.isfinite(y_pred_test)) and np.all(var_pred_test > 0)


def test_graph_capture_replays_bitwise():
    X, Y, ell, sf2, sn2 = make_gp_problem(600, 12, 8, seed=14)
    gp = engine.gp_factorize(X, Y, ell, sf2, sn2)
    Xs = engine.dev(_inputs(1000, 12, seed=15))
    mean, var = engine.gp_predict(gp, Xs)
    mc, cc = engine.gp_predict(gp, Xs[:64], full_cov=True)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        gm, gv = engine.gp_predict(gp, Xs)
        gmc, gcc = engine.gp_predict(gp, Xs[:64], full_cov=True)
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(gm, mean) and torch.equal(gv, var)
    assert torch.equal(gmc, mc) and torch.equal(gcc, cc)
