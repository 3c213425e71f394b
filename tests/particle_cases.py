"""Seeded particle problems shared by the particle tests: dynamics models, policies (as the engine's spec and as the
oracles' dicts), reward terms, initial states and normals, and small PILCO / SafePILCO objects.  Importing this module
touches no device: the builders that factorise on the GPU do so when called."""
import numpy as np
import torch

from pilco_b200 import engine, _lib
import particle_grad_oracle as pgo
from util import make_gp_problem, make_rollout_problem

BOX2 = np.array([2, 1, 1.0, 0, 0.2, 0.9, 1, 0.1, 0.8])             # dims 0, 1 inside (low, high)
BOX1C = np.array([1, 0, 1.0, 2, -np.inf, 0.6])                    # dim 2 not below 0.6


# ---- host problems: numpy factors of a small exact GP -----------------------------------------------------------------
def _problem(seed, n=25, Ds=3, U=1):
    rng = np.random.RandomState(seed)
    D = Ds + U
    C_ = rng.rand(n, D)
    Y = 0.3 * np.sin(3.0 * C_).dot(rng.rand(D, Ds))
    ell, sf2 = 0.5 + 0.4 * rng.rand(Ds, D), 0.05 * (1.0 + rng.rand(Ds))
    iK, beta = [], []
    for e in range(Ds):
        d = (C_[:, None] - C_[None]) / ell[e]
        K = sf2[e] * np.exp(-0.5 * (d * d).sum(-1)) + 1e-3 * np.eye(n)
        iK.append(np.linalg.inv(K)); beta.append(iK[-1] @ Y[:, e])
    return dict(C=C_, ell=ell, sf2=sf2, iK=np.stack(iK), beta=np.stack(beta)), rng


def _terms(Ds):
    return [dict(kind=_lib.REWARD_EXP, coef=1.0, W=np.diag(np.arange(1.0, Ds + 1)) + 0.2, t=0.4 * np.ones(Ds)),
            dict(kind=_lib.REWARD_LINEAR, coef=0.3, W=np.linspace(-1, 1, Ds), t=None),
            dict(kind=_lib.REWARD_EXP, coef=0.2, channel=_lib.CHANNEL_MULT, W=2.0 * np.eye(Ds), t=np.zeros(Ds)),
            dict(kind=_lib.REWARD_LINEAR, coef=0.05, channel=_lib.CHANNEL_MULT, W=np.ones(Ds), t=None)]


def _linear_pilco(**kw):
    from pilco.models import PILCO
    from pilco.controllers import LinearController
    X = np.random.RandomState(0).rand(20, 3); Y = 0.1 * X[:, :2]
    return PILCO((X, Y), controller=LinearController(2, 1), horizon=4, **kw), X


def _safe_pilco():
    from safe_pilco_extension.safe_pilco import SafePILCO
    from safe_pilco_extension.rewards_safe import RiskOfCollision
    from pilco.controllers import LinearController
    from pilco.rewards import LinearReward
    X = np.random.RandomState(1).rand(30, 5); Y = 0.1 * X[:, :4]
    return SafePILCO((X, Y), controller=LinearController(4, 1), horizon=4, reward_add=LinearReward(4, np.ones(4)),
                     reward_mult=RiskOfCollision(4, [0.0, 0.1], [0.6, 0.9]), mu=-4.0)


def _host_problem(E, A, U, seed, n=30):
    """numpy factors of a small exact GP on [phi(x), u] (D = E + A + U inputs, E outputs)"""
    rng = np.random.RandomState(seed)
    D = E + A + U
    Cx = rng.rand(n, D) * 2.0 - 1.0
    Y = 0.1 * np.sin(2.0 * Cx).dot(rng.rand(D, E))
    ell, sf2 = 0.7 + 0.5 * rng.rand(E, D), 0.02 * (1.0 + rng.rand(E))
    iK, beta = [], []
    for e in range(E):
        d = (Cx[:, None] - Cx[None]) / ell[e]
        K = sf2[e] * np.exp(-0.5 * (d * d).sum(-1)) + 1e-3 * np.eye(n)
        iK.append(np.linalg.inv(K)); beta.append(iK[-1] @ Y[:, e])
    return dict(C=Cx, ell=ell, sf2=sf2, iK=np.stack(iK), beta=np.stack(beta)), rng


def _joint_terms(E, A, U, other):
    """an EXP_SA term on the first angle's (sin, cos) and a state EXP term on the raw dimension ``other``"""
    Dh = E + A
    W = np.zeros((Dh + U, Dh + U)); W[E - A, E - A] = W[E - A + 1, E - A + 1] = 1.0; W[Dh, Dh] = 0.1
    t = np.zeros(Dh + U); t[E - A + 1] = -1.0
    Ws = np.zeros((E, E)); Ws[other, other] = 2.0
    return [dict(kind=_lib.REWARD_EXP_SA, coef=1.0, W=W, t=t),
            dict(kind=_lib.REWARD_EXP, coef=0.5, W=Ws, t=0.3 * np.ones(E)),
            dict(kind=_lib.REWARD_LINEAR, coef=0.2, channel=_lib.CHANNEL_MULT, W=np.eye(E)[other], t=None)]


def _policy(kind, rng, U, Dh, squash=True):
    if kind == "linear":
        return dict(kind=_lib.POLICY_LINEAR, squash=squash, maxa=0.8 + rng.rand(U), W=0.5 * rng.randn(U, Dh),
                    b=rng.randn(U))
    bf = 8
    return _rbf_point(dict(kind=_lib.POLICY_RBF, squash=squash, maxa=0.8 + rng.rand(U), Xc=rng.randn(bf, Dh),
                           Yc=0.3 * rng.randn(bf, U), ell=1.0 + 0.2 * rng.rand(U, Dh), sf2=np.ones(U),
                           sn2=1e-2 * np.ones(U)))


def _rbf_point(pol):
    """the numpy oracle's RBF policy (C, ell, sf2, beta) of pgo's parametrisation (Xc, Yc, ell, sf2, sn2)"""
    beta = pgo.rbf_beta(pgo.T(pol["Xc"]), pgo.T(pol["Yc"]), pgo.T(pol["ell"]), pol["sf2"], pol["sn2"])
    return dict(pol, C=pol["Xc"], beta=beta.detach().numpy())


# ---- device problems --------------------------------------------------------------------------------------------------
def _dyn_np(gp):
    return dict(C=gp.X.cpu().numpy(), ell=gp.ell.cpu().numpy(), sf2=gp.sf2.cpu().numpy(),
                iK=gp.iK.cpu().numpy(), beta=gp.beta.cpu().numpy())


def _rbf(Xc, Yc, lc, maxa):
    U = Yc.shape[1]
    pgp = engine.gp_factorize(Xc, Yc, lc, np.ones(U), 1e-4 * np.ones(U), need_iK=False, mode=1)
    spec = dict(kind=_lib.POLICY_RBF, Ds=Xc.shape[1], U=U, squash=True, max_action=maxa, gp=pgp)
    pol = dict(kind=_lib.POLICY_RBF, squash=True, maxa=maxa, C=Xc, ell=lc, sf2=np.ones(U), beta=pgp.beta.cpu().numpy())
    return spec, pol


def _linear(W, b, maxa, squash):
    U, Ds = W.shape
    return (dict(kind=_lib.POLICY_LINEAR, Ds=Ds, U=U, squash=squash, max_action=maxa, W=W, b=b),
            dict(kind=_lib.POLICY_LINEAR, squash=squash, maxa=maxa, W=W, b=b))


def _oracle_pol(spec, pol):
    """the autograd oracles' policy dict of a policy spec (the RBF policy by its data, not its factors)"""
    if spec["kind"] == _lib.POLICY_LINEAR:
        return pol
    g = spec["gp"]
    return dict(kind=_lib.POLICY_RBF, squash=pol["squash"], maxa=pol["maxa"], Xc=g.X.cpu().numpy(), Yc=g.Y.cpu().numpy(),
                ell=g.ell.cpu().numpy(), sf2=g.sf2.cpu().numpy(), sn2=g.sn2.cpu().numpy())


def _controller_np(ctrl):
    U = ctrl.num_outputs
    return dict(kind=_lib.POLICY_RBF, squash=True, maxa=np.broadcast_to(np.asarray(ctrl.max_action, dtype=np.float64), (U,)),
                C=np.asarray(ctrl.models[0].X), ell=np.asarray(ctrl.lengthscales), sf2=np.asarray(ctrl.variance).reshape(U),
                beta=ctrl.device_gp().beta.cpu().numpy())


def _all_terms(Ds):
    """exp, linear and box terms on both channels"""
    rng = np.random.RandomState(Ds)
    Wl = rng.randn(Ds)
    return [dict(kind=_lib.REWARD_EXP, coef=1.0, W=np.eye(Ds), t=0.5 * np.ones(Ds)),
            dict(kind=_lib.REWARD_LINEAR, coef=0.3, W=Wl, t=None),
            dict(kind=_lib.REWARD_BOX, coef=-2.0, W=BOX2, t=None),
            dict(kind=_lib.REWARD_EXP, coef=0.1, channel=_lib.CHANNEL_MULT, W=2.0 * np.eye(Ds), t=np.zeros(Ds)),
            dict(kind=_lib.REWARD_LINEAR, coef=0.01, channel=_lib.CHANNEL_MULT, W=Wl, t=None),
            dict(kind=_lib.REWARD_BOX, coef=0.2, channel=_lib.CHANNEL_MULT, W=BOX1C, t=None)]


def _case(name):
    """-> dyn (DeviceGP), policy spec, oracle policy, reward terms, m0, S0, H, P, mult_mu"""
    if name == "metric_rbf":
        pb = make_rollout_problem(300, 10, 2, 50, 1, seed=5)
        gp = engine.gp_factorize(pb["X"], pb["Y"], pb["ell"], pb["sf2"], pb["sn2"])
        spec, pol = _rbf(pb["Xc"][0], pb["Yc"][0], pb["lc"][0], pb["maxa"])
        return gp, spec, pol, _all_terms(10), pb["m0"], pb["S0"], 10, 1000, 1.5
    if name in ("linear_squash", "linear_nosquash"):
        X, Y, ell, sf2, sn2 = make_gp_problem(100, 5, 4, seed=6)
        gp = engine.gp_factorize(X, 0.1 * Y, ell, 0.1 * sf2, 1e-3 * np.ones(4))
        rng = np.random.RandomState(7)
        spec, pol = _linear(0.5 * rng.randn(1, 4), rng.randn(1), np.array([1.3]), name == "linear_squash")
        return gp, spec, pol, _all_terms(4), X[0, :4], 0.05 * np.eye(4), 8, 777, -3.0
    if name == "fitc":
        pb = make_rollout_problem(2000, 4, 1, 20, 1, seed=8)
        Z = np.random.RandomState(9).rand(200, 5)
        gp = engine.fitc_factorize(pb["X"], Z, pb["Y"], pb["ell"], pb["sf2"], pb["sn2"])
        spec, pol = _rbf(pb["Xc"][0], pb["Yc"][0], pb["lc"][0], pb["maxa"])
        return gp, spec, pol, _all_terms(4)[:3], pb["m0"], pb["S0"], 6, 300, 0.0
    assert name == "n1_d16_h0"
    X, Y, ell, sf2, sn2 = make_gp_problem(1, 16, 15, seed=10)
    gp = engine.gp_factorize(X, 0.1 * Y, ell, sf2, sn2)
    spec, pol = _linear(np.random.RandomState(11).randn(1, 15), np.zeros(1), np.ones(1), True)
    return gp, spec, pol, _all_terms(15)[:1], X[0, :15], 0.1 * np.eye(15), 0, 50, 0.0


def _draw(m0, S0, P, H, seed):
    rng = np.random.RandomState(seed)
    Ds = m0.shape[0]
    return m0[None] + rng.randn(P, Ds) @ np.linalg.cholesky(S0).T, rng.randn(P, H, Ds)


def _batch_case(kind, R):
    """-> dyn, batched policy spec, per-restart unbatched specs, reward terms, m0, S0, H, P, mult_mu"""
    if kind in ("rbf", "fitc"):
        Ds, U = (6, 2) if kind == "rbf" else (4, 1)
        pb = make_rollout_problem(300 if kind == "rbf" else 1500, Ds, U, 20, R, seed=30 + R)
        if kind == "rbf":
            gp = engine.gp_factorize(pb["X"], pb["Y"], pb["ell"], pb["sf2"], pb["sn2"])
        else:
            Z = np.random.RandomState(31).rand(150, Ds + U)
            gp = engine.fitc_factorize(pb["X"], Z, pb["Y"], pb["ell"], pb["sf2"], pb["sn2"])
        pgp = engine.gp_factorize(pb["Xc"], pb["Yc"], pb["lc"], np.ones((R, U)), 1e-4 * np.ones((R, U)),
                                  need_iK=False, mode=1)
        maxa = 0.8 + 0.4 * np.arange(U)
        spec = dict(kind=_lib.POLICY_RBF, Ds=Ds, U=U, squash=True, max_action=maxa, gp=pgp)
        ldw = engine.pad_n(pgp.n)
        singles = []
        for r in range(R):                      # restart r's arrays, as an unbatched policy
            one = engine.DeviceGP(pgp.X[r], pgp.ell[r], pgp.sf2[r], pgp.beta[r], mode=1)
            one.fact_ws = pgp.fact_ws[r * U * ldw * ldw:(r + 1) * U * ldw * ldw]
            singles.append(dict(spec, gp=one))
        return gp, spec, singles, _all_terms(Ds), pb["m0"], pb["S0"], 5, 300, 1.5
    X, Y, ell, sf2, sn2 = make_gp_problem(100, 5, 4, seed=32)
    gp = engine.gp_factorize(X, 0.1 * Y, ell, 0.1 * sf2, 1e-3 * np.ones(4))
    rng = np.random.RandomState(33)
    W, b = 0.5 * rng.randn(R, 1, 4), rng.randn(R, 1)
    spec = dict(kind=_lib.POLICY_LINEAR, Ds=4, U=1, squash=True, max_action=np.array([1.3]), W=W, b=b)
    singles = [dict(spec, W=W[r], b=b[r]) for r in range(R)]
    return gp, spec, singles, _all_terms(4), X[0, :4], 0.05 * np.eye(4), 7, 777, -3.0


def _revisit_problem(H, P, seed):
    """state lengthscales 1e12 (the model ignores the state) and a squashed constant action of 5, outside the data's
    action range [0, 1): every step of a particle has the same input, where var is close to sf2"""
    Ds, U = 3, 1
    X, Y, ell, sf2, sn2 = make_gp_problem(60, Ds + U, Ds, seed=seed)
    ell[:, :Ds] = 1e12
    gp = engine.gp_factorize(X, 0.1 * Y, ell, sf2, sn2)
    spec, _ = _linear(np.zeros((U, Ds)), np.array([np.pi / 2]), np.array([5.0]), True)
    terms = [dict(kind=_lib.REWARD_LINEAR, coef=1.0, W=np.ones(Ds), t=None)]
    rng = np.random.RandomState(seed)
    return gp, spec, terms, 0.5 + 0.1 * rng.randn(P, Ds), rng.randn(P, H, Ds)


def _pilco_data(seed, n=80, Ds=3, U=1):
    rng = np.random.RandomState(seed)
    X = rng.rand(n, Ds + U)
    return X, 0.1 * np.sin(X).dot(rng.rand(Ds + U, Ds))


def _pilco(kind, seed, **kw):
    from pilco.models import PILCO
    from pilco.controllers import RbfController, LinearController
    np.random.seed(seed)
    X, Y = _pilco_data(seed)
    ctrl = RbfController(3, 1, 10, max_action=1.2) if kind == "rbf" else LinearController(3, 1, max_action=1.0)
    pilco = PILCO((X[:60], Y[:60]), controller=ctrl, horizon=6, m_init=X[0:1, :3], S_init=0.05 * np.eye(3), **kw)
    return pilco, X, Y


def _angle_terms(E, A, U, joint):
    """state terms on the raw state (exp, linear, MULT box on dimension 0); with ``joint`` an EXP_SA term on the first
    angle's (sin, cos) = (0, -1) and a LINEAR_SA term on the action"""
    Dh, D = E + A, E + A + U
    rng = np.random.RandomState(E + A)
    terms = [dict(kind=_lib.REWARD_EXP, coef=1.0, W=0.5 * np.eye(E), t=0.2 * np.ones(E)),
             dict(kind=_lib.REWARD_LINEAR, coef=0.3, W=rng.randn(E), t=None),
             dict(kind=_lib.REWARD_BOX, coef=0.2, channel=_lib.CHANNEL_MULT, W=np.array([1, 1, 1.0, 0, -0.5, 0.8]),
                  t=None)]
    if joint:
        W = np.zeros((D, D)); k = E - A if A else 0                   # A = 0: on state dimensions 0, 1
        W[k, k] = W[k + 1, k + 1] = 1.0; W[Dh, Dh] = 0.1
        t = np.zeros(D); t[k + 1] = -1.0
        terms += [dict(kind=_lib.REWARD_EXP_SA, coef=0.8, W=W, t=t),
                  dict(kind=_lib.REWARD_LINEAR_SA, coef=-0.05, W=np.r_[np.zeros(Dh), np.ones(U)], t=None)]
    return terms


def _angle_case(E, dims, U=1, kind="linear", fitc=False, joint=False, n=150, R=1, seed=0):
    """-> gp, spec (a leading R when R > 1), oracle policy dicts per restart, terms, A"""
    A = len(dims)
    Dh, D = E + A, E + A + U
    X, Y, ell, sf2, sn2 = make_gp_problem(n, D, E, seed=seed + D)
    X = 2.0 * X - 1.0
    if fitc:
        Z = np.random.RandomState(seed).rand(60, D) * 2.0 - 1.0
        gp = engine.fitc_factorize(X, Z, 0.05 * Y, ell, 0.05 * sf2, 1e-3 * np.ones(E))
    else:
        gp = engine.gp_factorize(X, 0.05 * Y, ell, 0.05 * sf2, 1e-3 * np.ones(E))
    rng = np.random.RandomState(seed + 7)
    maxa = 0.8 + 0.4 * np.arange(U)
    if kind == "linear":
        W, b = 0.5 * rng.randn(R, U, Dh), rng.randn(R, U)
        if R == 1:
            spec, pol = _linear(W[0], b[0], maxa, True)
            pols = [pol]
        else:
            spec = dict(kind=_lib.POLICY_LINEAR, Ds=Dh, U=U, squash=True, max_action=maxa, W=W, b=b)
            pols = [_linear(W[r], b[r], maxa, True)[1] for r in range(R)]
    else:
        assert R == 1
        spec, pol = _rbf(rng.rand(12, Dh) * 2.0 - 1.0, 0.3 * rng.randn(12, U), 1.0 + 0.2 * rng.rand(U, Dh), maxa)
        pols = [pol]
    return gp, spec, pols, _angle_terms(E, A, U, joint)


def _box_case():
    """SafePILCO-like: a linear policy, a linear additive reward and one box as the only MULT term"""
    X, Y, ell, sf2, sn2 = make_gp_problem(100, 5, 4, seed=6)
    gp = engine.gp_factorize(X, 0.1 * Y, ell, 0.1 * sf2, 1e-3 * np.ones(4))
    rng = np.random.RandomState(48)
    W, b = 0.5 * rng.randn(1, 4), rng.randn(1)
    spec = dict(kind=_lib.POLICY_LINEAR, Ds=4, U=1, squash=True, max_action=np.array([1.3]), W=W, b=b)
    terms = [dict(kind=_lib.REWARD_LINEAR, coef=0.3, W=rng.randn(4), t=None),
             dict(kind=_lib.REWARD_BOX, coef=1.0, channel=_lib.CHANNEL_MULT, W=BOX2, t=None)]
    return gp, spec, terms, X[0, :4], 0.05 * np.eye(4), 6, -4.0


def _seeded(P, H, Ds, m0, S0, seed):
    d = engine.device()
    gen = torch.Generator(device=d)
    gen.manual_seed(seed)
    F = engine.dev(np.linalg.cholesky(S0))
    x0 = engine.dev(m0)[None] + torch.randn((P, Ds), dtype=engine.F64, device=d, generator=gen) @ F.T
    return x0, torch.randn((P, H, Ds), dtype=engine.F64, device=d, generator=gen)
