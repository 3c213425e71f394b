"""GPU tests of the stochastic policy optimiser (pilco_normals, pilco_adam_update, policy_opt.StochasticEvaluator,
PILCO.optimize_policy_sampled(optimizer="adam"); DESIGN.md section 32): the normals against the oracle, across call
lengths, eager against graph replay and their statistics; one iteration against the draws, the existing plan's gradient
and the oracle's Adam step, bit for bit, on every sampler and policy class; graph replays against eager iterations,
restarts against single runs, a frozen NaN restart and reruns; and the behaviour of a trained policy out of sample."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import sgd_oracle as so
from particle_cases import _pilco
from pilco_b200 import controllers, engine, policy_opt
from pilco_b200.models.pilco import PILCO, _sqrt_factor
from util import ROOT

pytestmark = pytest.mark.gpu

F64 = torch.float64


def _it(k=0):
    return torch.full((1,), k, dtype=torch.int64, device="cuda")


def _normals(n, seed, stream, k):
    return engine.normals(torch.empty(n, dtype=F64, device="cuda"), seed, stream, _it(k))


# ---- the normals -------------------------------------------------------------------------------------------------------
def test_normals_match_the_oracle_and_their_prefixes():
    for seed, stream, k, n in ((0, 0, 0, 1), (7, 3, 2, 1001), (2 ** 64 - 1, 2 ** 32 - 1, 2 ** 31, 70001)):
        got = _normals(n, seed, stream, k).cpu().numpy()
        ref = so.normals(seed, stream, k, n)
        u1, _ = so.pair_uniforms(seed, stream, k, (n + 1) // 2)
        r = np.repeat(np.sqrt(-2.0 * np.log(u1)), 2)[:n]
        assert np.all(np.abs(got - ref) <= 1e-15 * r), (seed, stream, k)
        for m in (1, n // 2, n - 1):
            if m >= 1:
                assert torch.equal(_normals(m, seed, stream, k), torch.as_tensor(got[:m], device="cuda"))
    big = _normals(1 << 22, 5, 1, 0)                                   # a grid-stride launch: the same bits
    assert torch.equal(big[:70001], _normals(70001, 5, 1, 0))


def test_normals_graph_replay_reads_the_counter_at_run_time():
    it = _it(0)
    out = torch.empty(4097, dtype=F64, device="cuda")
    engine.normals(out, 11, 2, it)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        engine.normals(out, 11, 2, it)
    for k in (0, 5, 123456):
        it.fill_(k)
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(out, _normals(4097, 11, 2, k)), k


def test_normals_statistics():
    N = 1 << 24
    a, b, c = _normals(N, 2024, 0, 0), _normals(N, 2024, 1, 0), _normals(N, 2024, 0, 1)
    se = 1.0 / np.sqrt(N)
    for x in (a, b, c):
        assert abs(float(x.mean())) < 5 * se
        assert abs(float(x.var()) - 1.0) < 5 * np.sqrt(2.0) * se
        assert abs(float((x * x * x * x).mean()) - 3.0) < 5 * np.sqrt(96.0) * se
    for x, y in ((a, b), (a, c), (b, c)):                               # streams and iterations uncorrelated
        assert abs(float((x * y).mean())) < 5 * se
    assert abs(float((a[0::2] * a[1::2]).mean())) < 5 * np.sqrt(2.0) * se    # the two elements of a pair


# ---- one iteration against the plan and the oracle --------------------------------------------------------------------
def _mlp_pilco(seed=0):
    np.random.seed(seed)
    p, X, Y = _pilco("linear", seed)
    return PILCO((X[:60], Y[:60]), controller=controllers.MlpController(3, 1, hidden=(8, 8), max_action=1.0),
                 horizon=6, m_init=X[0:1, :3], S_init=0.05 * np.eye(3))


def _problem(policy, seed=0):
    if policy == "mlp":
        return _mlp_pilco(seed)
    return _pilco(policy, seed)[0]


def _flats(pilco, R, seed=1):
    np.random.seed(seed)
    return policy_opt.initial_flats(pilco.controller, R)


SAMPLERS = {"stepwise": {}, "consistent": dict(consistent=True), "features": dict(consistent=True, num_features=32),
            "resample": dict(resample=True)}


def _evaluator(pilco, flats, P, seed, lr=1e-2, **kw):
    m0 = np.asarray(pilco.m_init, dtype=np.float64).reshape(-1)
    return policy_opt.StochasticEvaluator(pilco, flats.shape[0], flats, P, seed, m0, _sqrt_factor(pilco.S_init),
                                          lr=lr, trace_rows=8, **kw)


def _reference_step(pilco, flats, P, seed, lr, consistent=False, resample=False, num_features=None, exploration=None):
    """the draws of iteration 0 through engine.normals, ParticleEvaluator's loss and gradient on them, the oracle's
    Adam step -> theta"""
    Ds, H = pilco.state_dim, int(pilco.horizon)
    m0 = engine.dev(np.asarray(pilco.m_init, dtype=np.float64).reshape(-1))
    Ft = engine.dev(_sqrt_factor(pilco.S_init)).T
    x0 = m0[None] + _normals(P * Ds, seed, 0, 0).reshape(P, Ds) @ Ft
    eps, xi, draws = None, None, None
    if num_features is not None:
        dyn = pilco.mgpr.device_gp()
        zeta = _normals(dyn.E * num_features * dyn.D, seed, 4, 0).reshape(dyn.E, num_features, dyn.D)
        w = _normals(P * dyn.E * 2 * num_features, seed, 5, 0).reshape(P, dyn.E, 2 * num_features)
        eps_y = _normals(P * dyn.E * dyn.n, seed, 6, 0).reshape(P, dyn.E, dyn.n)
        draws = engine.feature_draws(dyn, P, num_features, zeta, w, eps_y)
    else:
        eps = _normals(P * H * Ds, seed, 1, 0).reshape(P, H, Ds)
    if resample:
        xi = _normals(P * H * Ds, seed, 3, 0).reshape(P, H, Ds)
    pe = policy_opt.ParticleEvaluator(pilco, flats.shape[0], x0, eps, consistent=consistent, exploration=exploration,
                                      resample=resample, xi=xi, features=draws)
    pe.use_graph = False
    loss, grad = pe(flats)
    R, n = flats.shape
    packed = np.hstack([loss[:, None], np.zeros((R, 1)), grad])
    z = np.zeros((R, n))
    return so.adam(flats, packed, z, z, np.zeros(R, dtype=np.int64), np.ones(R), np.ones(R), 0, np.full((8, R), np.nan),
                   np.zeros((8, R), dtype=np.int32), lr, 0.9, 0.999, 1e-8, 0.0)


CASES = [("linear", "stepwise", None), ("linear", "consistent", None), ("linear", "features", None),
         ("linear", "resample", None), ("rbf", "stepwise", None), ("rbf", "consistent", None),
         ("mlp", "stepwise", None), ("mlp", "features", None), ("mlp", "resample", None),
         ("linear", "stepwise", 0.7), ("mlp", "consistent", 0.7)]


@pytest.mark.parametrize("policy,sampler,b", CASES)
def test_one_iteration_is_the_draws_the_plan_and_the_oracle_step(policy, sampler, b):
    pilco = _problem(policy)
    flats, P, seed, lr = _flats(pilco, 3), 48, 99, 1e-2
    kw = dict(SAMPLERS[sampler], exploration=b)
    ev = _evaluator(pilco, flats, P, seed, lr=lr, **kw)
    ev.iteration()
    ref = _reference_step(pilco, flats, P, seed, lr, **kw)
    assert np.array_equal(ev.theta.cpu().numpy(), ref["theta"]), (policy, sampler, b)
    assert np.array_equal(ev.adam.trace.cpu().numpy()[0], ref["trace"][0])
    assert ev.adam.ok.cpu().numpy()[0].all() and int(ev.adam.iter.item()) == 1
    assert not np.array_equal(ref["theta"], flats)


# ---- determinism -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("policy,sampler", [("linear", "stepwise"), ("rbf", "consistent"), ("mlp", "features")])
def test_graph_replays_are_eager_iterations(policy, sampler):
    pilco = _problem(policy)
    flats, N = _flats(pilco, 2), 6
    a, b = _evaluator(pilco, flats, 32, 5, **SAMPLERS[sampler]), _evaluator(pilco, flats, 32, 5, **SAMPLERS[sampler])
    a.capture()
    for _ in range(N):
        a.replay()
        b.iteration()
    torch.cuda.synchronize()
    assert torch.equal(a.theta, b.theta) and torch.equal(a.adam.m, b.adam.m) and torch.equal(a.adam.v, b.adam.v)
    assert torch.equal(a.adam.trace.nan_to_num(7.0), b.adam.trace.nan_to_num(7.0))
    assert int(a.adam.iter.item()) == N and (a.adam.t == N).all()
    assert not torch.equal(a.adam.trace[0], a.adam.trace[1])           # fresh particles at every iteration


@pytest.mark.parametrize("policy", ["linear", "mlp"])
def test_a_restart_is_its_single_run_and_a_nan_restart_freezes(policy):
    pilco = _problem(policy)
    flats, N = _flats(pilco, 3), 4
    many = _evaluator(pilco, flats, 40, 8)
    one = _evaluator(pilco, flats[1:2], 40, 8)
    bad = flats.copy()
    bad[0] = np.nan
    frozen = _evaluator(pilco, bad, 40, 8)
    for _ in range(N):
        for ev in (many, one, frozen):
            ev.iteration()
    assert torch.equal(many.theta[1:2], one.theta)
    assert torch.equal(frozen.theta[1:], many.theta[1:]) and torch.equal(frozen.adam.m[1:], many.adam.m[1:])
    assert torch.isnan(frozen.theta[0]).all() and int(frozen.adam.t[0]) == 0
    assert not frozen.adam.ok[:N, 0].any() and frozen.adam.ok[:N, 1:].all()
    assert torch.equal(frozen.adam.m[0], torch.zeros_like(frozen.adam.m[0]))


def test_two_runs_with_one_seed_are_equal_and_the_value_is_the_held_out_one():
    pilco = _problem("linear")
    start = pilco.controller.get_flat().copy()
    out = []
    for _ in range(2):
        pilco.controller.set_flat(start)
        np.random.seed(3)
        v = pilco.optimize_policy_sampled(optimizer="adam", maxiter=20, restarts=3, num_samples=64, seed=17,
                                          learning_rate=1e-2)
        out.append((v, pilco.controller.get_flat().copy(), np.asarray(pilco.adam_trace.value).copy()))
    assert out[0][0] == out[1][0] and np.array_equal(out[0][1], out[1][1])
    assert np.array_equal(out[0][2], out[1][2]) and out[0][2].shape == (20, 3)
    assert pilco.adam_trace.ok.all()
    ev = _evaluator(pilco, out[0][1][None], 64, 17)
    assert float(ev.held_out().item()) == out[0][0]                    # the winner re-evaluated on the held-out draws


# ---- behaviour ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("policy", ["linear", "mlp"])
def test_adam_raises_the_out_of_sample_return(policy):
    pilco = _problem(policy)
    H, S = pilco.horizon, 1 << 14
    before = pilco.sample_policy_gradient(pilco.m_init, pilco.S_init, H, num_samples=S, seed=12345).returns
    best = pilco.optimize_policy_sampled(optimizer="adam", maxiter=300, restarts=2, num_samples=128, seed=1,
                                         learning_rate=1e-2)
    after = pilco.sample_policy_gradient(pilco.m_init, pilco.S_init, H, num_samples=S, seed=12345).returns
    d = np.asarray(after) - np.asarray(before)                         # the same particles: paired differences
    se = d.std(ddof=1) / np.sqrt(S)
    print("Adam %s: out-of-sample mean return %.5f -> %.5f (+%.1f standard errors), held-out value %.5f"
          % (policy, np.mean(before), np.mean(after), d.mean() / se, best))
    assert d.mean() > 5 * se
    assert np.isfinite(best) and np.all(np.isfinite(np.asarray(pilco.adam_trace.value)))


def test_example_runs_shortened():
    env = dict(os.environ, PYTHONPATH=ROOT)
    code = ("import sys; sys.path.insert(0, %r); import pendulum_sgd_numpy as ex; "
            "r, s = ex.run(episodes=1, T=10, horizon=10, random_episodes=2, maxiter=20, num_samples=32); "
            "assert len(s) == 1" % os.path.join(ROOT, "examples"))
    res = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, env=env, timeout=900)
    assert res.returncode == 0, res.stdout[-2000:] + res.stderr[-2000:]
    assert "Adam episode 0" in res.stdout
