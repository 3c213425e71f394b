"""Particle rollouts with angular state dimensions on the device (pilco_particles_angles_* through engine.ParticlePlan,
ConsistentGradPlan and particles_rollout with ``angles``, DESIGN.md section 20): forward parity of both samplers with
the numpy oracle (tests/particle_oracle.py) given the same x0 and eps, the pathwise, consistent and score gradients
against torch autograd on the oracle, the pathwise gradient against central differences of the device forward, A = 0 /
NULL against the calls without angles, periodicity in the angles, and the bitwise properties of the particle kernels."""
import ctypes as C

import numpy as np
import pytest
import torch

from pilco_b200 import engine, _lib
from pilco_b200._lib import lib
from particle_cases import _angle_case, _angle_terms, _dyn_np, _oracle_pol
from particle_grad_oracle import consistent_value_and_grad, score_grad, value_and_grad
from particle_oracle import consistent_rollout, particle_rollout
from util import _rel, scaled_err

pytestmark = pytest.mark.gpu


def _draw_raw(E, P, H, seed):
    rng = np.random.RandomState(seed)
    return 0.8 * rng.randn(P, E), rng.randn(P, H, E)


SHAPES = {                                                      # E, dims, U, policy, FITC, joint terms
    "cartpole_linear": (4, [1], 1, "linear", False, False),
    "cartpole_rbf": (4, [1], 1, "rbf", False, True),
    "double_pendulum": (6, [1, 2], 1, "rbf", False, False),
    "all_angles": (2, [0, 1], 1, "linear", False, True),
    "d16": (10, [0, 2, 4, 6, 8], 1, "linear", False, False),
    "joint_terms": (4, [3], 2, "linear", False, True),
    "fitc": (4, [1], 1, "rbf", True, False),
}


@pytest.mark.parametrize("name", sorted(SHAPES))
@pytest.mark.parametrize("consistent", [False, True])
def test_forward_parity_with_oracle(name, consistent):
    E, dims, U, kind, fitc, joint = SHAPES[name]
    gp, spec, pols, terms = _angle_case(E, dims, U, kind, fitc, joint)
    P, H, mu = (300 if consistent else 1000), 6, 1.5
    x0, eps = _draw_raw(E, P, H, seed=P + H)
    out = [t.cpu().numpy() for t in engine.particles_rollout(gp, spec, terms, x0, eps, mult_mu=mu,
                                                             consistent=consistent, angles=dims)]
    f = consistent_rollout if consistent else particle_rollout
    ref = f(_dyn_np(gp), pols[0], terms, x0, eps, mult_mu=mu, angle_dims=dims)
    own = scaled_err(f(_dyn_np(gp), pols[0], terms, x0, eps, mult_mu=mu, swap=True, angle_dims=dims)[0],
                     ref[0]) if consistent else 0.0
    shapes = [(P, H + 1, E), (P, H, U), (P, H), (P, H), (P,)]
    errs = []
    for what, o, r, shp in zip(("traj", "act", "reward", "risk", "ret"), out, ref, shapes):
        assert o.shape == shp, what
        errs.append(scaled_err(o, r) if r.size and np.abs(r).max() > 0 else float(np.abs(o).max(initial=0.0)))
    print("angle particles %s consistent=%s vs oracle: traj %.1e act %.1e reward %.1e risk %.1e ret %.1e (own %.1e)"
          % ((name, consistent) + tuple(errs) + (own,)))
    assert max(errs) <= max(1e-9, 10.0 * own)
    assert np.array_equal(out[0][:, 0], x0)


def _grad_plan(gp, spec, terms, x0, eps, mu, dims, R=1, estimator="pathwise", consistent=False):
    if consistent:
        plan = engine.ConsistentGradPlan(gp, spec, terms, x0.shape[0], eps.shape[1], mult_mu=mu, R=R, angles=dims)
    else:
        plan = engine.ParticlePlan(gp, spec, terms, x0.shape[0], eps.shape[1], mult_mu=mu, grad=True, R=R,
                                   estimator=estimator, angles=dims)
    plan.set_inputs(x0, eps)
    g = plan.launch_grad()
    return plan, {k: v.cpu().numpy() for k, v in g.items()}


@pytest.mark.parametrize("name", ["cartpole_linear", "cartpole_rbf", "double_pendulum", "all_angles", "joint_terms",
                                  "fitc"])
@pytest.mark.parametrize("estimator", ["pathwise", "consistent", "score"])
def test_gradients_match_autograd_oracle(name, estimator):
    E, dims, U, kind, fitc, joint = SHAPES[name]
    gp, spec, pols, terms = _angle_case(E, dims, U, kind, fitc, joint)
    P, H, mu = 200, 5, 1.5
    x0, eps = _draw_raw(E, P, H, seed=P + H + 1)
    plan, g = _grad_plan(gp, spec, terms, x0, eps, mu, dims, estimator="score" if estimator == "score" else "pathwise",
                         consistent=estimator == "consistent")
    args = (_dyn_np(gp), _oracle_pol(spec, pols[0]), terms)
    own = 0.0
    if estimator == "pathwise":
        v, ref = value_and_grad(*args, x0, eps, mu, angle_dims=dims)
    elif estimator == "consistent":
        v, ref, _ = consistent_value_and_grad(*args, x0, eps, mu, angle_dims=dims)
        own = _rel(consistent_value_and_grad(*args, x0, eps, mu, swap=True, angle_dims=dims)[1], ref)
    else:
        traj = plan.outputs()[0].cpu().numpy()
        ref = score_grad(*args, traj, eps, mu, angle_dims=dims)
        v = float(plan.outputs()[4].mean())
    err, verr = _rel(g, ref), abs(float(g["value"][0]) - v) / max(abs(v), 1e-300)
    print("angle gradient %s %s vs autograd oracle: %.1e of scale, value %.1e (own %.1e)" % (name, estimator, err, verr,
                                                                                           own))
    bar = 1e-6 if fitc else 1e-8
    assert err <= max(bar, 10.0 * own) and verr <= max(1e-9, 10.0 * own)


def test_batched_gradient_restarts_match_single_policy_calls():
    """R = 3 linear policies: restart r bitwise the R = 1 call with policy r, and each against the autograd oracle"""
    E, dims, U = 4, [1], 1
    gp, spec, pols, terms = _angle_case(E, dims, U, "linear", joint=True, R=3)
    x0, eps = _draw_raw(E, 150, 5, seed=5)
    plan, g = _grad_plan(gp, spec, terms, x0, eps, 0.5, dims, R=3)
    for r in range(3):
        one = dict(spec, W=spec["W"][r], b=spec["b"][r])
        p1, g1 = _grad_plan(gp, one, terms, x0, eps, 0.5, dims)
        for a, b in zip(plan.outputs(), p1.outputs()):
            assert torch.equal(a[r], b)
        for k in g1:
            assert np.array_equal(g[k][r], g1[k].reshape(g[k][r].shape)), k
        _, ref = value_and_grad(_dyn_np(gp), pols[r], terms, x0, eps, 0.5, angle_dims=dims)
        assert _rel({k: g[k][r] for k in ref}, ref) <= 1e-8


def test_pathwise_gradient_matches_central_differences_of_device_forward():
    E, dims, U = 6, [1, 2], 1
    gp, spec, pols, terms = _angle_case(E, dims, U, "linear", joint=True)
    x0, eps = _draw_raw(E, 500, 6, seed=9)
    _, g = _grad_plan(gp, spec, terms, x0, eps, 1.5, dims)
    val = lambda W, b: float(engine.particles_rollout(gp, dict(spec, W=W, b=b), terms, x0, eps, mult_mu=1.5,
                                                      angles=dims)[4].mean())
    rng = np.random.RandomState(3)
    dW, db = rng.randn(*spec["W"].shape), rng.randn(*spec["b"].shape)
    h = 1e-5
    fd = (val(spec["W"] + h * dW, spec["b"] + h * db) - val(spec["W"] - h * dW, spec["b"] - h * db)) / (2 * h)
    gd = float((g["W"] * dW).sum() + (g["b"] * db).sum())
    print("directional derivative: central difference %.12e, pathwise %.12e" % (fd, gd))
    assert abs(fd - gd) <= 1e-6 * abs(gd)


def test_no_angles_is_bitwise_the_call_without_angles():
    """the angle entry points with ang = NULL and A = 0 write bitwise what the calls without angles write"""
    E, U = 4, 1
    gp, spec, pols, terms = _angle_case(E, [], U, "linear", joint=True)
    x0, eps = _draw_raw(E, 300, 5, seed=2)
    for consistent in (False, True):
        plan = engine.ParticlePlan(gp, spec, terms, 300, 5, mult_mu=0.5, consistent=consistent)
        plan.set_inputs(x0, eps)
        plan.launch()
        ref = [t.clone() for t in plan.outputs()]
        f = lib.pilco_particles_angles_consistent_rollout if consistent else lib.pilco_particles_angles_rollout
        for ang in (None, _lib.Angles()):
            for t in plan.outputs():
                t.zero_()
            assert f(C.byref(plan.pr), C.byref(ang) if ang is not None else None, engine.stream_ptr()) == 0
            assert all(torch.equal(a, b) for a, b in zip(plan.outputs(), ref))
    for estimator, consistent, fn in (("pathwise", False, lib.pilco_particles_angles_batch_grad_rollout),
                                      ("score", False, lib.pilco_particles_angles_score_grad_rollout),
                                      ("pathwise", True, lib.pilco_particles_angles_consistent_grad_rollout)):
        plan, g = _grad_plan(gp, spec, terms, x0, eps, 0.5, None, estimator=estimator, consistent=consistent)
        ref = [t.clone() for t in plan.outputs()]
        for ang in (None, _lib.Angles()):
            for v in plan.gbuf.values():
                v.zero_()
            assert fn(C.byref(plan.pr), C.byref(ang) if ang is not None else None, 1, C.byref(plan.grad),
                      engine.stream_ptr()) == 0
            assert all(torch.equal(a, b) for a, b in zip(plan.outputs(), ref))
            assert all(np.array_equal(plan.gbuf[k].cpu().numpy(), g[k]) for k in g), (estimator, consistent)


@pytest.mark.parametrize("estimator", ["pathwise", "consistent", "score"])
def test_periodic_in_the_angles(estimator):
    """x0 + 2 pi e_a: the same actions, step rewards, returns and gradients (the state terms do not read dimension a),
    the trajectory shifted by 2 pi in dimension a only"""
    E, dims, U = 4, [1, 3], 1
    gp, spec, pols, _ = _angle_case(E, dims, U, "rbf", joint=True)
    terms = _angle_terms(E, len(dims), U, True)[2:]                  # the box on dimension 0 and the joint terms
    x0, eps = _draw_raw(E, 200, 4, seed=4)
    run = lambda x: _grad_plan(gp, spec, terms, x, eps, 0.5, dims, estimator="score" if estimator == "score" else
                               "pathwise", consistent=estimator == "consistent")
    pa, ga = run(x0)
    for k, a in enumerate(dims):
        x1 = x0.copy(); x1[:, a] += 2.0 * np.pi * (k + 1)
        pb, gb = run(x1)
        ta, tb = pa.outputs()[0].cpu().numpy(), pb.outputs()[0].cpu().numpy()
        shift = np.zeros(E); shift[a] = 2.0 * np.pi * (k + 1)
        assert np.max(np.abs(tb - ta - shift)) <= 1e-10
        for u, v in zip(pa.outputs()[1:], pb.outputs()[1:]):
            assert np.max(np.abs(u.cpu().numpy() - v.cpu().numpy()), initial=0.0) <= 1e-10
        assert _rel(gb, ga) <= 1e-9


def test_particle_is_independent_of_batch_and_row():
    E, dims, U = 6, [1, 2], 1
    gp, spec, _, terms = _angle_case(E, dims, U, "rbf", joint=True)
    x0, eps = _draw_raw(E, 400, 5, seed=6)
    for consistent in (False, True):
        full = engine.particles_rollout(gp, spec, terms, x0, eps, mult_mu=0.5, consistent=consistent, angles=dims)
        part = engine.particles_rollout(gp, spec, terms, x0[:150], eps[:150], mult_mu=0.5, consistent=consistent,
                                        angles=dims)
        perm = np.random.RandomState(1).permutation(400)
        pm = engine.particles_rollout(gp, spec, terms, x0[perm], eps[perm], mult_mu=0.5, consistent=consistent,
                                      angles=dims)
        for a, b, c in zip(full, part, pm):
            assert torch.equal(a[:150], b) and torch.equal(a[torch.as_tensor(perm, device=a.device)], c)


def test_graph_replay_is_bitwise_equal_to_eager():
    E, dims, U = 4, [1], 1
    gp, spec, _, terms = _angle_case(E, dims, U, "rbf", joint=True)
    x0, eps = _draw_raw(E, 300, 5, seed=7)
    for estimator in ("pathwise", "score"):
        plan = engine.ParticlePlan(gp, spec, terms, 300, 5, mult_mu=0.5, grad=True, estimator=estimator, angles=dims)
        plan.set_inputs(x0, eps)
        fwd = engine.ParticlePlan(gp, spec, terms, 300, 5, mult_mu=0.5, angles=dims)
        fwd.set_inputs(x0, eps)
        plan.launch_grad(); fwd.launch()
        ref = [t.clone() for t in plan.outputs()] + [v.clone() for v in plan.gbuf.values()]
        fref = [t.clone() for t in fwd.outputs()]
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            plan.launch_grad()
            fwd.launch()
        for t in list(plan.outputs()) + list(plan.gbuf.values()) + list(fwd.outputs()):
            t.zero_()
        graph.replay()
        torch.cuda.synchronize()
        got = list(plan.outputs()) + list(plan.gbuf.values())
        assert all(torch.equal(a, b) for a, b in zip(got, ref))
        assert all(torch.equal(a, b) for a, b in zip(fwd.outputs(), fref))


def test_pendulum_model_from_pilco():
    """the engine calls on a model trained on [phi(x), u] by PILCO(angle_dims=[0]) (examples/pendulum_angles_numpy.py)"""
    import os
    import sys
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "examples"))
    from pendulum_angles_numpy import make_pilco
    _, pilco, X, Y = make_pilco(T=10, bf=6, episodes=2)
    gp, spec = pilco.mgpr.device_gp(), pilco.policy_spec()
    terms = [dict(kind=_lib.REWARD_EXP_SA, coef=1.0, W=np.diag([0.05, 1.0, 1.0, 0.0]), t=np.array([0.0, 0.0, -1.0, 0.0]))]
    P, H = 256, 10
    rng = np.random.RandomState(0)
    x0, eps = 0.1 * rng.randn(P, 2), rng.randn(P, H, 2)
    plan = engine.ParticlePlan(gp, spec, terms, P, H, grad=True, estimator="score", angles=[0])
    plan.set_inputs(x0, eps)
    g = plan.launch_grad()
    assert all(np.all(np.isfinite(v.cpu().numpy())) for v in g.values())
    out = engine.particles_rollout(gp, spec, terms, x0, eps, consistent=True, angles=[0])
    assert out[0].shape == (P, H + 1, 2) and bool(torch.isfinite(out[0]).all())
    pol = dict(kind=_lib.POLICY_RBF, squash=True, maxa=np.atleast_1d(spec["max_action"]).astype(float),
               C=spec["gp"].X.cpu().numpy(), ell=spec["gp"].ell.cpu().numpy(), sf2=spec["gp"].sf2.cpu().numpy(),
               beta=spec["gp"].beta.cpu().numpy())
    ref = consistent_rollout(_dyn_np(gp), pol, terms, x0, eps, angle_dims=[0])
    own = scaled_err(consistent_rollout(_dyn_np(gp), pol, terms, x0, eps, swap=True, angle_dims=[0])[0], ref[0])
    err = scaled_err(out[0].cpu().numpy(), ref[0])
    print("pendulum consistent particles vs oracle: %.1e (the oracle with its sums reordered: %.1e)" % (err, own))
    assert err <= max(1e-9, 10.0 * own)                         # the bar of the consistent sampler's own tests
