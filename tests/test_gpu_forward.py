"""GPU parity tests of the forward path through the C ABI (``-m gpu``): every device entry point against
the numpy oracle on seeded inputs.  fp64 tolerances are written beside each assertion."""
import numpy as np
import pytest

from util import relerr, scaled_err, make_gp_problem, make_input, hyp_of

pytestmark = pytest.mark.gpu

RTOL = 1e-9        # fp64 path; the reference's own bar is 1e-4 (tests/test_predictions.py:61-63)


def _engine():
    from pilco_b200 import engine
    return engine


@pytest.mark.parametrize("n,D,E", [(100, 3, 2), (37, 1, 1), (64, 4, 3), (130, 5, 4), (300, 12, 10),
                                   (257, 7, 6), (65, 13, 2), (500, 10, 8), (600, 3, 2),
                                   (1000, 4, 2)])        # n >= 512: multi-CTA Cholesky + DMMA GEMM path
def test_gp_factorize_matches_oracle(n, D, E):
    from oracle import python_port as pp
    eng = _engine()
    X, Y, ell, sf2, sn2 = make_gp_problem(n, D, E, seed=n)
    gp = eng.gp_factorize(X, Y, ell, sf2, sn2)
    iK_ref, beta_ref = pp.calculate_factorizations(X, Y, ell, sf2, sn2)
    assert int(gp.info.max().item()) == 0
    iK = gp.iK.cpu().numpy()
    assert scaled_err(gp.beta.cpu().numpy(), beta_ref) < 1e-8
    assert scaled_err(iK[:, :n, :n], iK_ref) < 1e-8
    assert np.all(iK[:, n:, :] == 0) and np.all(iK[:, :, n:] == 0)        # zero padding is part of the ABI


@pytest.mark.parametrize("n,D,E,R", [(100, 3, 2, 1), (37, 1, 1, 2), (64, 4, 3, 3), (130, 5, 4, 2),
                                     (300, 12, 10, 2), (257, 7, 6, 1), (65, 13, 2, 2), (70, 16, 3, 1),
                                     (500, 10, 8, 1), (600, 3, 2, 2)])
def test_mm_forward_matches_oracle(n, D, E, R):
    """the moment match of the device-factorised model against the extended-precision oracle given the SAME factors
    (tests/mm_oracle.py; the factorisation has its own test above): every entry of M, S, V within 2.5e3 eps64 of its
    condition scale, the bar of test_gpu_mm_regimes.py (5.6e-13 of the sum of |terms|; it replaces 1e-7 and, for S,
    1e-6 of the largest entry)"""
    import mm_oracle as mo
    if not mo.HAVE_EXTENDED:
        pytest.skip(mo.NEED_EXTENDED)
    eng = _engine()
    X, Y, ell, sf2, sn2 = make_gp_problem(n, D, E, seed=n + 1)
    gp = eng.gp_factorize(X, Y, ell, sf2, sn2)
    ms = [make_input(D, seed=10 + r, scale=0.3 + 0.4 * r) for r in range(R)]
    m = np.concatenate([a for a, _ in ms])
    s = np.stack([b for _, b in ms])
    M, S, V, info = eng.mm_forward(gp, m, s)
    assert int(info.max().item()) == 0
    beta, iK = gp.beta.cpu().numpy(), gp.iK.cpu().numpy()[:, :n, :n]
    for r in range(R):
        ref = mo.moment_match(X, ell, sf2, beta, iK, m[r], s[r])
        for name, got in (("M", M), ("S", S), ("V", V)):
            err = np.abs(got[r].cpu().numpy().astype(mo.LD) - ref[name])
            assert float(np.max(err / (mo.EPS64 * ref["c" + name]))) <= 2.5e3, (name, r)


def test_mm_forward_zero_covariance():
    """s = 0 (PILCO.compute_action, pilco.py:115-116) must reduce to the plain GP mean."""
    from oracle import python_port as pp
    eng = _engine()
    X, Y, ell, sf2, sn2 = make_gp_problem(80, 4, 2, seed=5)
    gp = eng.gp_factorize(X, Y, ell, sf2, sn2)
    m = np.random.RandomState(0).rand(1, 4)
    M, S, V, info = eng.mm_forward(gp, m, np.zeros((1, 4, 4)))
    iK, beta = pp.calculate_factorizations(X, Y, ell, sf2, sn2)
    k = pp.se_ard_K(m, X, ell, sf2)[:, 0, :]
    assert scaled_err(M[0].cpu().numpy(), (k * beta).sum(1)) < 1e-10


# ---- the reference's own test recipes (tests/test_*.py), oracle = MATLAB transcription -------------
def test_recipe_predictions():
    """tests/test_predictions.py:13-63 (gp0.m), incl. the set_data cache-invalidation step."""
    from oracle import matlab_port as mp
    from pilco.models import MGPR
    np.random.seed(0)
    d, k = 3, 2
    X0 = np.random.rand(100, d)
    A = np.random.rand(d, k)
    Y0 = np.sin(X0).dot(A) + 1e-3 * (np.random.rand(100, k) - 0.5)
    mgpr = MGPR((X0, Y0))
    mgpr.optimize()
    m = np.random.rand(1, d)
    s = np.random.rand(d, d)
    s = s.dot(s.T)
    M, S, V = mgpr.predict_on_noisy_inputs(m, s)
    X0 = 5 * np.random.rand(100, d)
    mgpr.set_data((X0, Y0))
    M, S, V = mgpr.predict_on_noisy_inputs(m, s)
    ell = np.stack([mod.kernel.lengthscales for mod in mgpr.models])
    sf2 = np.stack([mod.kernel.variance for mod in mgpr.models])
    sn2 = np.stack([mod.likelihood.variance for mod in mgpr.models])
    Mm, Sm, Vm = mp.gp0(dict(hyp=hyp_of(ell, sf2, sn2), inputs=X0, targets=Y0), m.T, s)
    assert M.shape == Mm.T.shape and S.shape == Sm.shape and V.shape == Vm.shape
    np.testing.assert_allclose(M, Mm.T, rtol=1e-4)
    np.testing.assert_allclose(S, Sm, rtol=1e-4)
    np.testing.assert_allclose(V, Vm, rtol=1e-4)


def test_recipe_sparse_predictions():
    """tests/test_sparse_predictions.py:12-57 (gp1.m)."""
    from oracle import matlab_port as mp
    from pilco.models import SMGPR
    np.random.seed(0)
    d, k = 3, 2
    X0 = np.random.rand(100, d)
    A = np.random.rand(d, k)
    Y0 = np.sin(X0).dot(A) + 1e-3 * (np.random.rand(100, k) - 0.5)
    smgpr = SMGPR((X0, Y0), num_induced_points=30)
    smgpr.optimize()
    m = np.random.rand(1, d)
    s = np.random.rand(d, d)
    s = s.dot(s.T)
    M, S, V = smgpr.predict_on_noisy_inputs(m, s)
    ell = np.stack([mod.kernel.lengthscales for mod in smgpr.models])
    sf2 = np.stack([mod.kernel.variance for mod in smgpr.models])
    sn2 = np.stack([mod.likelihood.variance for mod in smgpr.models])
    gm = dict(hyp=hyp_of(ell, sf2, sn2), inputs=X0, targets=Y0, induce=smgpr.Z.numpy())
    Mm, Sm, Vm = mp.gp1(gm, m.T, s)
    np.testing.assert_allclose(M, Mm.T, rtol=1e-4)
    np.testing.assert_allclose(S, Sm, rtol=1e-4)
    np.testing.assert_allclose(V, Vm, rtol=1e-4)


def test_recipe_rbf_controller():
    """tests/test_controllers.py:13-57 (gp2.m)."""
    from oracle import matlab_port as mp
    from pilco.controllers import RbfController
    np.random.seed(0)
    d, k, b = 3, 2, 100
    X0 = np.random.rand(100, d)
    A = np.random.rand(d, k)
    Y0 = np.sin(X0).dot(A) + 1e-3 * (np.random.rand(100, k) - 0.5)
    rbf = RbfController(3, 2, b)
    rbf.set_data((X0, Y0))
    m = np.random.rand(1, d)
    s = np.random.rand(d, d)
    s = s.dot(s.T)
    M, S, V = rbf.compute_action(m, s, squash=False)
    ell = np.stack([mod.kernel.lengthscales.numpy() for mod in rbf.models])
    sf2 = np.stack([mod.kernel.variance.numpy() for mod in rbf.models])
    sn2 = np.stack([mod.likelihood.variance.numpy() for mod in rbf.models])
    Mm, Sm, Vm = mp.gp2(dict(hyp=hyp_of(ell, sf2, sn2), inputs=X0, targets=Y0), m.T, s)
    assert M.shape == Mm.T.shape and S.shape == Sm.shape and V.shape == Vm.shape
    np.testing.assert_allclose(M, Mm.T, rtol=1e-4)
    np.testing.assert_allclose(S, Sm, rtol=1e-4)
    np.testing.assert_allclose(V, Vm, rtol=1e-4)


def test_recipe_linear_controller_and_squash():
    """tests/test_controllers.py:59-113 (conlin.m, gSin.m)."""
    from oracle import matlab_port as mp
    from pilco.controllers import LinearController, squash_sin
    np.random.seed(0)
    d, k = 3, 2
    m = np.random.rand(1, d)
    s = np.random.rand(d, d)
    s = s.dot(s.T)
    W = np.random.rand(k, d)
    b = np.random.rand(1, k)
    lin = LinearController(d, k)
    lin.W.assign(W)
    lin.b.assign(b)
    M, S, V = lin.compute_action(m, s, squash=False)
    Mm, Sm, Vm = mp.conlin(dict(p=dict(w=W, b=b.T)), m.T, s)
    np.testing.assert_allclose(M, Mm.T, rtol=1e-12)
    np.testing.assert_allclose(S, Sm, rtol=1e-10)
    np.testing.assert_allclose(V, Vm, rtol=1e-12)
    M, S, C = squash_sin(m, s, 7.0)
    Mm, Sm, Cm = mp.gSin(m.T, s, 7.0)
    np.testing.assert_allclose(M, Mm.T, rtol=1e-10)
    np.testing.assert_allclose(S, Sm, rtol=1e-9)
    np.testing.assert_allclose(C, Cm, rtol=1e-10, atol=1e-300)


def test_recipe_reward():
    """tests/test_rewards.py:13-31 (reward.m), default rtol 1e-7."""
    from oracle import matlab_port as mp
    from pilco.rewards import ExponentialReward
    rng = np.random.RandomState(3)
    for k in (2, 5, 10):
        m = rng.rand(1, k)
        s = rng.rand(k, k)
        s = s.dot(s.T)
        reward = ExponentialReward(k)
        M, S = reward.compute_reward(m, s)
        muR, _, _, sR = mp.reward(m.T, s, reward.t.numpy().T, reward.W.numpy())
        np.testing.assert_allclose(M, muR, rtol=1e-7)
        np.testing.assert_allclose(S, sR, rtol=1e-7, atol=1e-15)


def test_recipe_cascade_forward():
    """tests/test_cascade.py:17-78 (pred.m/propagate.m) -- forward cascade with random linear policy
    (the policy-optimisation part of the recipe is covered in test_gpu_policy.py)."""
    from oracle import matlab_port as mp
    from pilco.models.pilco import PILCO
    np.random.seed(0)
    d, k, horizon = 2, 1, 10
    e = np.array([[10.0]])
    X0 = np.random.rand(100, d + k)
    A = np.random.rand(d + k, d)
    Y0 = np.sin(X0).dot(A) + 1e-3 * (np.random.rand(100, d) - 0.5)
    pilco = PILCO((X0, Y0))
    pilco.controller.max_action = e
    pilco.optimize_models(restarts=2)
    m = np.random.rand(1, d)
    s = np.random.rand(d, d)
    s = s.dot(s.T)
    M, S, reward = pilco.predict(m, s, horizon)
    policy = dict(p=dict(w=pilco.controller.W.numpy(), b=pilco.controller.b.numpy().T), maxU=e)
    ell = np.stack([mod.kernel.lengthscales.numpy() for mod in pilco.mgpr.models])
    sf2 = np.stack([mod.kernel.variance.numpy() for mod in pilco.mgpr.models])
    sn2 = np.stack([mod.likelihood.variance.numpy() for mod in pilco.mgpr.models])
    dynmodel = dict(hyp=hyp_of(ell, sf2, sn2), inputs=X0, targets=Y0)
    plant = dict(angi=np.zeros(0), poli=np.arange(d) + 1, dyni=np.arange(d) + 1, difi=np.arange(d) + 1)
    Mm, Sm = mp.pred(policy, plant, dynmodel, m.T, s, horizon)
    np.testing.assert_allclose(M[0], Mm[:, -1], rtol=2e-4)
    np.testing.assert_allclose(S, Sm[:, :, -1], rtol=2e-4)
    assert reward.shape == (1, 1) and np.isfinite(reward).all()


@pytest.mark.parametrize("kind,R", [("linear", 1), ("linear", 3), ("rbf", 1), ("rbf", 2)])
def test_rollout_matches_python_port(kind, R):
    """H-step cascade, batched over R restarts, vs the vectorised port of pilco.py:118-153."""
    from oracle import python_port as pp
    from pilco_b200 import engine, _lib
    Ds, U, n, H, bf = 4, 2, 90, 6, 20
    D = Ds + U
    X, Y, ell, sf2, sn2 = make_gp_problem(n, D, Ds, seed=7)
    Y = 0.1 * Y
    gp = engine.gp_factorize(X, Y, ell, sf2, sn2)
    rng = np.random.RandomState(11)
    maxa = np.array([1.5, 0.7])
    Wr, tr = np.diag(rng.rand(Ds) + 0.5), 0.1 * rng.rand(Ds)
    m0, S0 = X[0, :Ds], 0.05 * np.eye(Ds)
    if kind == "linear":
        W = rng.randn(R, U, Ds)
        b = rng.randn(R, U)
        spec = dict(kind=_lib.POLICY_LINEAR, Ds=Ds, U=U, squash=True, max_action=maxa,
                    W=W if R > 1 else W[0], b=b if R > 1 else b[0])
        acts = [lambda m, s, r=r: pp.linear_action(W[r], b[r][None], m, s, True, maxa[None]) for r in range(R)]
    else:
        Xc, Yc = rng.randn(R, bf, Ds), 0.1 * rng.randn(R, bf, U)
        lc = 1.0 + 0.1 * rng.randn(R, U, Ds)
        pgp = engine.gp_factorize(Xc if R > 1 else Xc[0], Yc if R > 1 else Yc[0], lc if R > 1 else lc[0],
                                  np.ones((R, U)) if R > 1 else np.ones(U),
                                  1e-4 * np.ones((R, U)) if R > 1 else 1e-4 * np.ones(U), need_iK=False, mode=1)
        spec = dict(kind=_lib.POLICY_RBF, Ds=Ds, U=U, squash=True, max_action=maxa, gp=pgp)
        acts = [lambda m, s, r=r: pp.rbf_action(Xc[r], Yc[r], lc[r], m, s, True, maxa[None]) for r in range(R)]
    plan = engine.RolloutPlan(gp, spec, [dict(kind=_lib.REWARD_EXP, coef=1.0, W=Wr, t=tr)], m0, S0, H, R=R)
    tm, tS, rew = plan.forward()
    assert int(plan.info.max().item()) == 0
    iK_ref, beta_ref = pp.calculate_factorizations(X, Y, ell, sf2, sn2)
    dyn = lambda m, s: pp.predict_given_factorizations(X, ell, sf2, m, s, iK_ref, beta_ref)
    rfn = lambda m, s: pp.exponential_reward(m, s, Wr, tr[None])
    for r in range(R):
        Mr, Sr, Rr = pp.predict(m0[None], S0, H, acts[r], dyn, rfn)
        assert scaled_err(tm[r, -1].cpu().numpy(), Mr[0]) < 1e-8
        assert scaled_err(tS[r, -1].cpu().numpy(), Sr) < 1e-7
        assert abs(float(rew[r]) - Rr.item()) < 1e-8 * max(1.0, abs(Rr.item()))


def test_gp_append_matches_refactorisation():
    """Incremental set_data (SURVEY section 8f-2; mgpr.py:38-45 with the rows of a new episode appended,
    inv_double_pendulum.py:102-103): the O(n^2 k) block-inverse update of the resident model (pilco_gp_append) against
    a full refactorisation of the grown data set -- factors and moment-match outputs, two appends in a row."""
    from pilco_b200 import engine
    n0, D, E = 200, 5, 3
    X, Y, ell, sf2, sn2 = make_gp_problem(n0 + 70, D, E, seed=11)
    gp = engine.gp_factorize(X[:n0], Y[:n0], ell, sf2, sn2)
    m, s = make_input(D, seed=3, scale=0.3)
    for n1 in (n0 + 40, n0 + 70):                      # 200 -> 240 -> 270 (crosses a multiple of 64: ldk 256 -> 320)
        gp = engine.gp_append(gp, X[:n1], Y[:n1])
        ref = engine.gp_factorize(X[:n1], Y[:n1], ell, sf2, sn2)
        assert int(gp.info.max().item()) == 0 and gp.n == n1 and gp.ldk == engine.pad_n(n1)
        iK, iKr = gp.iK.cpu().numpy(), ref.iK.cpu().numpy()
        assert np.all(iK[:, n1:, :] == 0) and np.all(iK[:, :, n1:] == 0)
        assert scaled_err(iK, iKr) < 1e-9
        assert scaled_err(gp.beta.cpu().numpy(), ref.beta.cpu().numpy()) < 1e-9
        out, outr = engine.mm_forward(gp, m, s[None]), engine.mm_forward(ref, m, s[None])
        for a, b in zip(out[:3], outr[:3]):
            assert scaled_err(a.cpu().numpy(), b.cpu().numpy()) < 1e-9
    assert gp.appends == 2


def test_mgpr_set_data_appends_incrementally():
    """The class-level policy: appended rows + unchanged hyper-parameters -> resident model updated ('append');
    anything else (changed hypers, changed old rows, shrinking) -> full refactorisation; same predictions either way."""
    from pilco.models import MGPR
    n0, D, E = 120, 4, 2
    X, Y, ell, sf2, sn2 = make_gp_problem(n0 + 50, D, E, seed=5)
    m, s = make_input(D, seed=2, scale=0.3)

    def fixed(mg):
        for i, mod in enumerate(mg.models):
            mod.kernel.lengthscales.assign(ell[i]); mod.kernel.variance.assign(sf2[i]); mod.likelihood.variance.assign(sn2[i])
    mg = MGPR((X[:n0], Y[:n0])); fixed(mg)
    mg.predict_on_noisy_inputs(m, s)
    assert mg.last_update == "factorize"
    mg.set_data((X[:n0 + 30], Y[:n0 + 30]))
    M1, S1, V1 = mg.predict_on_noisy_inputs(m, s)
    assert mg.last_update == "append"
    ref = MGPR((X[:n0 + 30], Y[:n0 + 30])); fixed(ref)
    Mr, Sr, Vr = ref.predict_on_noisy_inputs(m, s)
    for a, b in ((M1, Mr), (S1, Sr), (V1, Vr)):
        assert scaled_err(a, b) < 1e-9
    mg.models[0].kernel.lengthscales.assign(ell[0] * 1.1)          # hyper-parameters changed -> refactorise
    mg.set_data((X[:n0 + 50], Y[:n0 + 50]))
    mg.predict_on_noisy_inputs(m, s)
    assert mg.last_update == "factorize"
    X2 = X[:n0 + 50].copy(); X2[0, 0] += 0.5                       # an OLD row changed -> not an append
    mg.set_data((np.vstack([X2, X[:5] + 0.1]), np.vstack([Y[:n0 + 50], Y[:5]])))
    mg.predict_on_noisy_inputs(m, s)
    assert mg.last_update == "factorize"
