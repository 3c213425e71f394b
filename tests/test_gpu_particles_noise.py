"""Particle rollouts with measurement noise at the policy's input on the device (pilco_particles_noisy_* through
engine.ParticlePlan, ConsistentGradPlan and particles_rollout with ``measurement_noise``, DESIGN.md section 23): forward
parity of both samplers with the numpy oracle (tests/particle_oracle.py) given the same x0, eps and nu, the
pathwise, consistent and score gradients against torch autograd on the oracle, the pathwise gradient against central
differences of the device forward, nz = NULL against the angle calls, v = 0 against the calls without noise, the
structural and bitwise properties, and the one-step moments against the noisy moment-matching rollout."""
import ctypes as C

import numpy as np
import pytest
import torch

from pilco_b200 import engine, _lib
from pilco_b200._lib import lib
from particle_cases import _angle_case, _dyn_np, _linear, _oracle_pol
from particle_grad_oracle import consistent_value_and_grad, score_grad, value_and_grad
from particle_oracle import consistent_rollout, moment_check, particle_rollout
from util import _rel, make_rollout_problem, scaled_err

pytestmark = pytest.mark.gpu


def _draw(E, P, H, seed):
    rng = np.random.RandomState(seed)
    return 0.8 * rng.randn(P, E), rng.randn(P, H, E), rng.randn(P, H, E)


def _var(E, seed=0):
    return 0.01 + 0.03 * np.random.RandomState(seed + 100).rand(E)


SHAPES = {                                                      # E, dims, U, policy, FITC, joint terms
    "linear": (4, [], 1, "linear", False, False),
    "rbf": (4, [], 1, "rbf", False, True),
    "cartpole": (4, [1], 1, "rbf", False, False),
    "double_pendulum": (6, [1, 2], 1, "linear", False, True),
    "joint_terms": (4, [], 2, "linear", False, True),
    "fitc": (4, [1], 1, "rbf", True, False),
}


@pytest.mark.parametrize("name", sorted(SHAPES))
@pytest.mark.parametrize("consistent", [False, True])
def test_forward_parity_with_oracle(name, consistent):
    E, dims, U, kind, fitc, joint = SHAPES[name]
    gp, spec, pols, terms = _angle_case(E, dims, U, kind, fitc, joint)
    P, H, mu = (300 if consistent else 1000), 6, 1.5
    x0, eps, nu = _draw(E, P, H, seed=P + H)
    v = _var(E)
    out = [t.cpu().numpy() for t in engine.particles_rollout(gp, spec, terms, x0, eps, mult_mu=mu, consistent=consistent,
                                                             angles=dims, measurement_noise=v, nu=nu)]
    f = consistent_rollout if consistent else particle_rollout
    kw = dict(angle_dims=dims, nu=nu, v=v)
    ref = f(_dyn_np(gp), pols[0], terms, x0, eps, mu, **kw)
    own = scaled_err(f(_dyn_np(gp), pols[0], terms, x0, eps, mu, swap=True, **kw)[0], ref[0]) if consistent else 0.0
    errs = []
    for o, r in zip(out, ref):
        errs.append(scaled_err(o, r) if r.size and np.abs(r).max() > 0 else float(np.abs(o).max(initial=0.0)))
    print("noisy particles %s consistent=%s vs oracle: traj %.1e act %.1e reward %.1e risk %.1e ret %.1e (own %.1e)"
          % ((name, consistent) + tuple(errs) + (own,)))
    assert max(errs) <= max(1e-9, 10.0 * own)
    assert np.array_equal(out[0][:, 0], x0)


def _grad_plan(gp, spec, terms, x0, eps, nu, v, mu, dims, R=1, estimator="pathwise", consistent=False):
    if consistent:
        plan = engine.ConsistentGradPlan(gp, spec, terms, x0.shape[0], eps.shape[1], mult_mu=mu, R=R, angles=dims,
                                         measurement_noise=v)
    else:
        plan = engine.ParticlePlan(gp, spec, terms, x0.shape[0], eps.shape[1], mult_mu=mu, grad=True, R=R,
                                   estimator=estimator, angles=dims, measurement_noise=v)
    plan.set_inputs(x0, eps, nu)
    g = plan.launch_grad()
    return plan, {k: t.cpu().numpy() for k, t in g.items()}


@pytest.mark.parametrize("name", sorted(SHAPES))
@pytest.mark.parametrize("estimator", ["pathwise", "consistent", "score"])
def test_gradients_match_autograd_oracle(name, estimator):
    E, dims, U, kind, fitc, joint = SHAPES[name]
    gp, spec, pols, terms = _angle_case(E, dims, U, kind, fitc, joint)
    P, H, mu = 200, 5, 1.5
    x0, eps, nu = _draw(E, P, H, seed=P + H + 1)
    v = _var(E, 1)
    plan, g = _grad_plan(gp, spec, terms, x0, eps, nu, v, mu, dims,
                         estimator="score" if estimator == "score" else "pathwise", consistent=estimator == "consistent")
    args = (_dyn_np(gp), _oracle_pol(spec, pols[0]), terms)
    own = 0.0
    if estimator == "pathwise":
        val, ref = value_and_grad(*args, x0, eps, mu, angle_dims=dims, nu=nu, v=v)
    elif estimator == "consistent":
        val, ref, _ = consistent_value_and_grad(*args, x0, eps, mu, angle_dims=dims, nu=nu, v=v)
        own = _rel(consistent_value_and_grad(*args, x0, eps, mu, swap=True, angle_dims=dims, nu=nu, v=v)[1], ref)
    else:
        traj = plan.outputs()[0].cpu().numpy()
        ref = score_grad(*args, traj, eps, mu, angle_dims=dims, nu=nu, v=v)
        val = float(plan.outputs()[4].mean())
    err, verr = _rel(g, ref), abs(float(g["value"][0]) - val) / max(abs(val), 1e-300)
    print("noisy gradient %s %s vs autograd oracle: %.1e of scale, value %.1e (own %.1e)" % (name, estimator, err, verr,
                                                                                           own))
    bar = 1e-6 if fitc else 1e-8
    assert err <= max(bar, 10.0 * own) and verr <= max(1e-9, 10.0 * own)


def test_pathwise_gradient_matches_central_differences_of_device_forward():
    E, dims, U = 6, [1, 2], 1
    gp, spec, _, terms = _angle_case(E, dims, U, "linear", joint=True)
    x0, eps, nu = _draw(E, 500, 6, seed=9)
    v = _var(E, 2)
    _, g = _grad_plan(gp, spec, terms, x0, eps, nu, v, 1.5, dims)
    val = lambda W, b: float(engine.particles_rollout(gp, dict(spec, W=W, b=b), terms, x0, eps, mult_mu=1.5, angles=dims,
                                                      measurement_noise=v, nu=nu)[4].mean())
    rng = np.random.RandomState(3)
    dW, db = rng.randn(*spec["W"].shape), rng.randn(*spec["b"].shape)
    h = 1e-5
    fd = (val(spec["W"] + h * dW, spec["b"] + h * db) - val(spec["W"] - h * dW, spec["b"] - h * db)) / (2 * h)
    gd = float((g["W"] * dW).sum() + (g["b"] * db).sum())
    print("directional derivative: central difference %.12e, pathwise %.12e" % (fd, gd))
    assert abs(fd - gd) <= 1e-6 * abs(gd)


_FWD = [lib.pilco_particles_noisy_rollout, lib.pilco_particles_noisy_consistent_rollout]
_GRAD = {("pathwise", False): lib.pilco_particles_noisy_batch_grad_rollout,
         ("score", False): lib.pilco_particles_noisy_score_grad_rollout,
         ("pathwise", True): lib.pilco_particles_noisy_consistent_grad_rollout}


def test_null_noise_is_bitwise_the_angle_call():
    """nz = NULL writes bitwise what the angle calls write, and with ang = NULL what the calls without angles write"""
    for E, dims in ((4, [1]), (4, [])):
        gp, spec, _, terms = _angle_case(E, dims, 1, "linear", joint=True)
        x0, eps, _ = _draw(E, 300, 5, seed=2)
        ang = engine.angles_struct(dims, E)
        for consistent, f in zip((False, True), _FWD):
            plan = engine.ParticlePlan(gp, spec, terms, 300, 5, mult_mu=0.5, consistent=consistent, angles=dims)
            plan.set_inputs(x0, eps)
            plan.launch()
            ref = [t.clone() for t in plan.outputs()]
            for t in plan.outputs():
                t.zero_()
            assert f(C.byref(plan.pr), C.byref(ang) if ang is not None else None, None, engine.stream_ptr()) == 0
            assert all(torch.equal(a, b) for a, b in zip(plan.outputs(), ref))
        for (estimator, consistent), fn in _GRAD.items():
            if consistent:
                plan = engine.ConsistentGradPlan(gp, spec, terms, 300, 5, mult_mu=0.5, angles=dims)
            else:
                plan = engine.ParticlePlan(gp, spec, terms, 300, 5, mult_mu=0.5, grad=True, estimator=estimator,
                                           angles=dims)
            plan.set_inputs(x0, eps)
            g = {k: t.cpu().numpy() for k, t in plan.launch_grad().items()}
            ref = [t.clone() for t in plan.outputs()]
            for t in list(plan.gbuf.values()) + list(plan.outputs()):
                t.zero_()
            assert fn(C.byref(plan.pr), C.byref(ang) if ang is not None else None, None, 1, C.byref(plan.grad),
                      engine.stream_ptr()) == 0
            assert all(torch.equal(a, b) for a, b in zip(plan.outputs(), ref))
            assert all(np.array_equal(plan.gbuf[k].cpu().numpy(), g[k]) for k in g), (estimator, consistent)


@pytest.mark.parametrize("dims", [[], [1]])
def test_zero_noise_is_the_noiseless_call(dims):
    """v = 0 with any nu: forward outputs bitwise, gradients within 1e-12 of scale (J' phi_bar is split in two sums)"""
    E = 4
    gp, spec, _, terms = _angle_case(E, dims, 1, "rbf", joint=True)
    x0, eps, nu = _draw(E, 300, 5, seed=3)
    for consistent in (False, True):
        a = engine.particles_rollout(gp, spec, terms, x0, eps, mult_mu=0.5, consistent=consistent, angles=dims)
        b = engine.particles_rollout(gp, spec, terms, x0, eps, mult_mu=0.5, consistent=consistent, angles=dims,
                                     measurement_noise=np.zeros(E), nu=nu)
        assert all(torch.equal(u, w) for u, w in zip(a, b))
    for estimator, consistent in _GRAD:
        est = dict(estimator=estimator, consistent=consistent)
        pa, ga = _grad_plan(gp, spec, terms, x0, eps, None, None, 0.5, dims, **est)
        pb, gb = _grad_plan(gp, spec, terms, x0, eps, nu, np.zeros(E), 0.5, dims, **est)
        assert all(torch.equal(u, w) for u, w in zip(pa.outputs(), pb.outputs()))
        err = _rel(gb, {k: ga[k] for k in ga if k != "value"})
        print("v = 0 %s consistent=%s: gradient %.1e of scale" % (estimator, consistent, err))
        assert err <= 1e-12 and np.array_equal(ga["value"], gb["value"])


def test_structural_properties():
    """a linear policy with W = 0 ignores v and nu bitwise; nu in a dimension with v_i = 0 changes no bit"""
    E, dims = 4, [1]
    gp, spec, _, terms = _angle_case(E, dims, 1, "linear", joint=True)
    x0, eps, nu = _draw(E, 300, 5, seed=4)
    zero = dict(spec, W=np.zeros_like(spec["W"]))
    v = _var(E)
    for estimator, consistent in _GRAD:
        est = dict(estimator=estimator, consistent=consistent)
        pa, ga = _grad_plan(gp, zero, terms, x0, eps, None, None, 0.5, dims, **est)
        pb, gb = _grad_plan(gp, zero, terms, x0, eps, nu, v, 0.5, dims, **est)
        assert all(torch.equal(u, w) for u, w in zip(pa.outputs(), pb.outputs()))
        assert all(np.array_equal(ga[k], gb[k]) for k in ga if k != "W"), (estimator, consistent)
        v2 = v.copy(); v2[2] = 0.0
        nu2 = nu.copy(); nu2[:, :, 2] += 1.0
        pc, gc = _grad_plan(gp, spec, terms, x0, eps, nu, v2, 0.5, dims, **est)
        pd, gd = _grad_plan(gp, spec, terms, x0, eps, nu2, v2, 0.5, dims, **est)
        assert all(torch.equal(u, w) for u, w in zip(pc.outputs(), pd.outputs()))
        assert all(np.array_equal(gc[k], gd[k]) for k in gc), (estimator, consistent)


def test_restarts_rows_and_graph_replay_are_bitwise():
    """R = 3 restarts each the R = 1 call with its policy; a particle independent of P and its row; graph replay"""
    E, dims, U = 4, [1], 1
    gp, spec, _, terms = _angle_case(E, dims, U, "linear", joint=True, R=3)
    x0, eps, nu = _draw(E, 150, 5, seed=5)
    v = _var(E)
    for estimator, consistent in _GRAD:
        est = dict(estimator=estimator, consistent=consistent)
        plan, g = _grad_plan(gp, spec, terms, x0, eps, nu, v, 0.5, dims, R=3, **est)
        for r in range(3):
            p1, g1 = _grad_plan(gp, dict(spec, W=spec["W"][r], b=spec["b"][r]), terms, x0, eps, nu, v, 0.5, dims, **est)
            assert all(torch.equal(a[r], b) for a, b in zip(plan.outputs(), p1.outputs()))
            assert all(np.array_equal(g[k][r], g1[k].reshape(g[k][r].shape)) for k in g1), (estimator, consistent, r)
    one = dict(spec, W=spec["W"][0], b=spec["b"][0])
    perm = np.random.RandomState(1).permutation(150)
    for consistent in (False, True):
        run = lambda a, b, c: engine.particles_rollout(gp, one, terms, a, b, mult_mu=0.5, consistent=consistent,
                                                       angles=dims, measurement_noise=v, nu=c)
        full, part, pm = run(x0, eps, nu), run(x0[:60], eps[:60], nu[:60]), run(x0[perm], eps[perm], nu[perm])
        for a, b, c in zip(full, part, pm):
            assert torch.equal(a[:60], b) and torch.equal(a[torch.as_tensor(perm, device=a.device)], c)
    for estimator in ("pathwise", "score"):
        plan = engine.ParticlePlan(gp, one, terms, 150, 5, mult_mu=0.5, grad=True, estimator=estimator, angles=dims,
                                   measurement_noise=v)
        plan.set_inputs(x0, eps, nu)
        fwd = engine.ParticlePlan(gp, one, terms, 150, 5, mult_mu=0.5, angles=dims, measurement_noise=v)
        fwd.set_inputs(x0, eps, nu)
        plan.launch_grad(); fwd.launch()
        ref = [t.clone() for t in list(plan.outputs()) + list(plan.gbuf.values()) + list(fwd.outputs())]
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            plan.launch_grad()
            fwd.launch()
        got = list(plan.outputs()) + list(plan.gbuf.values()) + list(fwd.outputs())
        for t in got:
            t.zero_()
        graph.replay()
        torch.cuda.synchronize()
        assert all(torch.equal(a, b) for a, b in zip(got, ref))


def test_one_step_moments_match_noisy_moment_matching():
    """H = 1, no angles, a linear unsquashed policy: [x, W (x + nu) + b] is Gaussian, so RolloutPlan(measurement_noise=v)
    gives the exact moments of x_1 that 2^20 particles sample; the noiseless RolloutPlan's moments fail the check"""
    E, U = 10, 2
    pb = make_rollout_problem(300, E, U, 50, 1, seed=13)
    gp = engine.gp_factorize(pb["X"], pb["Y"], pb["ell"], pb["sf2"], pb["sn2"])
    rng = np.random.RandomState(14)
    spec, _ = _linear(0.5 * rng.randn(U, E), rng.randn(U), np.ones(U), False)
    terms = [dict(kind=_lib.REWARD_EXP, coef=1.0, W=np.eye(E), t=pb["m0"] + 0.3)]
    m0, S0 = pb["m0"], 0.1 * np.eye(E)
    v = 0.2 + 0.3 * rng.rand(E)
    moments = []
    for nz in (v, None):
        tm, tS, _ = engine.RolloutPlan(gp, spec, terms, m0, S0, 1, R=1, measurement_noise=nz).forward()
        moments.append((tm[0, 1].cpu().numpy(), tS[0, 1].cpu().numpy()))
    P = 1 << 20
    g = torch.Generator(device=engine.device())
    g.manual_seed(15)
    d = engine.device()
    x0 = engine.dev(m0)[None] + torch.randn((P, E), dtype=engine.F64, device=d, generator=g) @ \
        engine.dev(np.linalg.cholesky(S0)).T
    eps = torch.randn((P, 1, E), dtype=engine.F64, device=d, generator=g)
    nu = torch.randn((P, 1, E), dtype=engine.F64, device=d, generator=g)
    traj = engine.particles_rollout(gp, spec, terms, x0, eps, measurement_noise=v, nu=nu)[0][:, 1].cpu().numpy()
    worst, bare = moment_check(traj, *moments[0]), moment_check(traj, *moments[1])
    print("one-step moments at P=2^20: %.2f standard errors against the noisy moments, %.2f against the noiseless"
          % (worst, bare))
    assert worst <= 5.0 and bare > 5.0
