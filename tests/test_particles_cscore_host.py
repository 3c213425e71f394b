"""CPU tests of the score-function gradient over consistent function samples (pilco_particles_consistent_score_grad_*,
engine.ConsistentGradPlan(estimator="score"), DESIGN.md section 25): the torch oracle (tests/particle_grad_oracle.py's
score_grad(consistent=True))
against autograd of the joint Gaussian log-density of each particle's path, against section 16's score gradient at
H = 2 and, in expectation, against the consistent pathwise gradient; the status codes, their order and the workspace
sizes of the C entry points on fake descriptors; the new kernel's registers and SASS; and the engine's checks before
any allocation."""
import os
import re
import subprocess

import numpy as np
import pytest
import torch

from pilco_b200 import _lib, engine
from pilco_b200._lib import lib
from abi_fakes import (ERR_DIM, ERR_NULL, ERR_UNSUP, ERR_WS, FAKE, PT_MAX_P, _angle_particles, _angles, _batched, _grad,
                       _noise, _particles, _score_grad_cases)
from particle_cases import _problem, _terms
import particle_grad_oracle as pgo
import particle_oracle as po
from util import CUOBJDUMP, ROOT, _ref, _rel, sass_named

F64 = torch.float64


# ---- the oracle -------------------------------------------------------------------------------------------------------
def _linear(rng, Ds, squash=True):
    return dict(kind=_lib.POLICY_LINEAR, squash=squash, maxa=np.array([1.2]), W=0.6 * rng.randn(1, Ds),
                b=0.2 * rng.randn(1))


def _joint_logdensity_grad(dyn, pol, traj):
    """d/dtheta (1/P) sum_p sum_e log N(f_pe; mu_e(X~_p), K_post,e(X~_p, X~_p)) over the steps t < H-1, X~_p the
    particle's inputs [x_t, pi(x_t)] and f the increments, via torch.distributions.MultivariateNormal"""
    prm, act = pgo.policy(pol)
    P, H1, Ds = traj.shape
    Hm = H1 - 2
    C_, ell, sf2, iK = (pgo.T(dyn[k]) for k in ("C", "ell", "sf2", "iK"))
    n = C_.shape[0]
    tot = torch.zeros((), dtype=F64)
    for p in range(P):
        x = pgo.T(traj[p, :Hm])
        X = torch.cat([x, act(x)], 1)                              # [Hm, D]
        mu = pgo.gp_latent(dyn, X)[0]
        f = pgo.T(traj[p, 1:Hm + 1] - traj[p, :Hm])
        for e in range(ell.shape[0]):
            Ks = pgo._se(X, C_, ell[e], sf2[e])
            K = pgo._se(X, X, ell[e], sf2[e]) - Ks @ iK[e][:n, :n] @ Ks.T
            K = 0.5 * (K + K.T)
            tot = tot + torch.distributions.MultivariateNormal(mu[:, e], covariance_matrix=K).log_prob(f[:, e])
    return pgo._grads(tot / P, prm)


def test_whitening_identity():
    """w = 1, no degenerate pivot: the surrogate is the log-density of the particle's whole path under its draw"""
    dyn, rng = _problem(51)
    pol = _linear(rng, 3)
    terms = [dict(kind=_lib.REWARD_LINEAR, coef=1.0, W=np.ones(3), t=None)]
    P, H = 12, 5
    x0, eps = 0.5 + 0.2 * rng.randn(P, 3), rng.randn(P, H, 3)
    traj = po.consistent_rollout(dyn, pol, terms, x0, eps)[0]
    g, ratio = pgo.score_grad(dyn, pol, terms, traj, eps, w=np.ones((P, H - 1)), direct=False, consistent=True)
    ref = _joint_logdensity_grad(dyn, pol, traj)
    err = _rel(g, ref)
    print("whitening identity: %.1e of the gradient's scale, smallest pivot d2 / (tau sf2) %.1e" % (err, ratio))
    assert ratio > 1e3 and err <= 1e-10


@pytest.mark.parametrize("squash", [True, False])
def test_two_steps_is_the_step_wise_score_gradient(squash):
    """H = 2: step 0 is the same transition in both samplers, so the oracle is section 16's"""
    dyn, rng = _problem(52)
    pol = _linear(rng, 3, squash)
    joint = dict(kind=_lib.REWARD_EXP_SA, coef=0.7, W=np.eye(4) + 0.1, t=0.2 * np.ones(4))
    terms = _terms(3) + [joint]
    P = 200
    x0, eps = 0.5 + 0.2 * rng.randn(P, 3), rng.randn(P, 2, 3)
    traj = po.consistent_rollout(dyn, pol, terms, x0, eps, mult_mu=1.5)[0]
    g, ratio = pgo.score_grad(dyn, pol, terms, traj, eps, 1.5, consistent=True)
    ref = pgo.score_grad(dyn, pol, terms, traj, eps, 1.5)
    err = _rel(g, ref)
    print("H = 2 against the step-wise score gradient: %.1e of the gradient's scale" % err)
    assert ratio > 1.0 and err <= 1e-12


def test_expected_gradient_is_the_consistent_pathwise_gradient():
    """smooth terms on both channels: the oracle's mean and the consistent pathwise oracle's mean over the same
    particles agree (paired, 16 x 1000 particles)"""
    dyn, rng = _problem(53)
    pol = _linear(rng, 3)
    terms = _terms(3)
    P, H, K = 1000, 4, 16
    score, path, ratio = {"W": [], "b": []}, {"W": [], "b": []}, np.inf
    for k in range(K):
        r = np.random.RandomState(2000 + k)
        x0, eps = 0.5 + 0.2 * r.randn(P, 3), r.randn(P, H, 3)
        traj = po.consistent_rollout(dyn, pol, terms, x0, eps, mult_mu=1.5)[0]
        g, rt = pgo.score_grad(dyn, pol, terms, traj, eps, 1.5, consistent=True)
        gp = pgo.consistent_value_and_grad(dyn, pol, terms, x0, eps, 1.5)[1]
        ratio = min(ratio, rt)
        for key in score:
            score[key].append(g[key]); path[key].append(gp[key])
    worst = 0.0
    for key in score:
        d = np.stack(score[key]) - np.stack(path[key])
        worst = max(worst, float(np.max(np.abs(d.mean(0)) / (d.std(0, ddof=1) / np.sqrt(K)))))
    print("consistent score vs pathwise oracle, paired over %d x %d particles: worst %.2f standard errors, smallest "
          "pivot d2 / (tau sf2) %.1e" % (K, P, worst, ratio))
    assert ratio > 1e3 and worst <= 5.0


def test_degenerate_steps_are_dropped():
    """a revisited input makes every later pivot degenerate: those steps carry no term, so with w = 1 only step 0's
    log-density is left"""
    dyn, rng = _problem(54)
    pol = dict(kind=_lib.POLICY_LINEAR, squash=False, maxa=np.ones(1), W=np.zeros((1, 3)), b=np.array([0.3]))
    ell = np.concatenate([1e12 * np.ones((3, 3)), dyn["ell"][:, 3:]], 1)              # the state is ignored
    iK = []
    for e in range(3):
        d = (dyn["C"][:, None] - dyn["C"][None]) / ell[e]
        iK.append(np.linalg.inv(dyn["sf2"][e] * np.exp(-0.5 * (d * d).sum(-1)) + 1e-3 * np.eye(dyn["C"].shape[0])))
    iK = np.stack(iK)
    dyn = dict(dyn, ell=ell, iK=iK, beta=np.einsum("enm,me->en", iK, np.sin(3.0 * dyn["C"][:, :3])))
    terms = [dict(kind=_lib.REWARD_LINEAR, coef=1.0, W=np.ones(3), t=None)]
    P, H = 30, 4
    x0, eps = 0.5 + 0.1 * rng.randn(P, 3), rng.randn(P, H, 3)
    traj = po.consistent_rollout(dyn, pol, terms, x0, eps)[0]
    g = pgo.score_grad(dyn, pol, terms, traj, eps, w=np.ones((P, H - 1)), direct=False, consistent=True)[0]
    one = pgo.score_grad(dyn, pol, terms, traj[:, :3], eps[:, :2], w=np.ones((P, 1)), direct=False, consistent=True)[0]
    assert all(np.all(np.isfinite(g[k])) for k in g) and np.abs(one["b"]).max() > 0.0
    np.testing.assert_allclose(g["b"], one["b"], rtol=1e-12, atol=0.0)


# ---- the C entry points on fake descriptors ---------------------------------------------------------------------------
def _call(pr, ang, nz, R, g):
    return lib.pilco_particles_consistent_score_grad_rollout(_ref(pr), _ref(ang), _ref(nz), R, _ref(g), None)


def _path_call(pr, ang, nz, R, g):
    return lib.pilco_particles_noisy_consistent_grad_rollout(_ref(pr), _ref(ang), _ref(nz), R, _ref(g), None)


def _ws(pr, ang, nz, R):
    return lib.pilco_particles_consistent_score_grad_workspace_bytes(_ref(pr), _ref(ang), _ref(nz), R)


def _path_ws(pr, ang, nz, R):
    return lib.pilco_particles_noisy_consistent_grad_workspace_bytes(_ref(pr), _ref(ang), _ref(nz), R)


def _all_cases():
    """(pr, ang, nz, R, g) rejected by the consistent pathwise call: section 16's plain cases, angles, noise and
    both, with bad variances, a missing nu and bad angle maps"""
    out = [(pr, None, None, R, g) for pr, R, g, _ in _score_grad_cases()]
    for A in (1, 2):
        for kind in (_lib.POLICY_LINEAR, _lib.POLICY_RBF):
            out.append((_angle_particles(kind, A=A), _angles(*range(A)), None, 1, _grad()))
            out.append((_angle_particles(kind, A=A, batched=True), _angles(*range(A)), _noise(), 3, _grad()))
    out.append((_angle_particles(A=1), _angles(3), None, 1, _grad()))                # out-of-range dimension
    out.append((_angle_particles(A=2), _angles(1, 1), _noise(), 1, _grad()))         # repeated dimension
    out.append((_angle_particles(A=1), _angles(0), _noise([float("nan")] * 3), 1, _grad()))
    for nz in (_noise(), _noise([0.0] * 3), _noise([-1.0, 0.1, 0.1]), _noise([0.1, float("inf"), 0.1]),
               _noise(nu=None)):
        out.append((_particles(), None, nz, 1, _grad()))
        out.append((_batched(), _angles(), nz, 3, _grad()))                          # A = 0: no angles
        out.append((_particles(H=0), None, nz, 1, _grad()))                          # H = 0 reads no nu
    pr = _particles(); pr.x0 = None
    out.append((pr, None, _noise([float("nan")] * 3, nu=None), 1, _grad()))          # the description first
    g = _grad(); g.value = None
    out.append((_particles(), None, _noise([-1.0] * 3), 1, g))
    out.append((_particles(), None, _noise([-1.0] * 3), 0, _grad()))
    out.append((None, None, _noise(), 1, _grad()))
    out.append((None, _angles(1), None, 1, _grad()))
    return out


def test_status_codes_are_the_consistent_pathwise_calls():
    """every code, in the same order: the same status on every case the consistent pathwise call rejects, and a
    workspace query that is 0 exactly where that call's is"""
    seen = set()
    for i, (pr, ang, nz, R, g) in enumerate(_all_cases()):
        want = _path_call(pr, ang, nz, R, g)
        assert want != 0, i
        assert _call(pr, ang, nz, R, g) == want, i
        assert (_ws(pr, ang, nz, R) == 0) == (_path_ws(pr, ang, nz, R) == 0), i
        seen.add(want)
    assert seen >= {ERR_NULL, ERR_DIM, ERR_WS, ERR_UNSUP}


def test_workspace_short_of_the_score_layout_and_overflow():
    for pr, ang, nz in ((_batched(), None, None), (_batched(_lib.POLICY_RBF), None, None),
                        (_angle_particles(A=2, batched=True), _angles(0, 2), None),
                        (_angle_particles(A=1, batched=True), _angles(1), _noise())):
        need = _ws(pr, ang, nz, 3)
        g = _grad(); g.ws_bytes = need - 8
        assert need > _path_ws(pr, ang, nz, 3) > 0 and _call(pr, ang, nz, 3, g) == ERR_WS
        g.ws = FAKE + 8; g.ws_bytes = need
        assert _call(pr, ang, nz, 3, g) == _path_call(pr, ang, nz, 3, g) != 0
    pr = _particles(P=PT_MAX_P, H=(1 << 31) - 1)                     # size_t overflow and 2^31 - 1 CTAs
    g = _grad(); g.ws_bytes = (1 << 64) - 1
    assert _ws(pr, None, None, 1) == 0 and _call(pr, None, None, 1, g) == ERR_DIM
    assert _ws(_batched(P=1000), None, None, PT_MAX_P // 1000 + 1) == 0


def _even(k):
    return k + (k & 1)


@pytest.mark.parametrize("kind", [_lib.POLICY_LINEAR, _lib.POLICY_RBF])
def test_workspace_bytes_are_the_stated_layout(kind):
    """the consistent pathwise gradient's layout, then G [H-1,T], the sums [R,H], m_bar and v_bar [H-1,T,E] and the
    x~_bar history [H,T,D]"""
    for P, H, R, A, noisy in ((1000, 5, 1, 0, False), (1000, 5, 2, 1, False), (777, 12, 3, 2, True),
                              (1, 0, 1, 0, False), (1, 1, 1, 0, True), (64, 2, 4, 1, True)):
        pr = _angle_particles(kind, A=A, P=P, H=H, batched=R > 1) if A else (_batched if R > 1 else _particles)(
            kind, P=P, H=H)
        ang = _angles(*range(A)) if A else None
        nz = _noise() if noisy else None
        T, E, D, Hm = R * P, 3, 3 + A + 1, max(H - 1, 0)
        extra = 8 * (_even(Hm * T) + _even(R * H) + 2 * _even(Hm * T * E) + _even(H * T * D))
        assert _ws(pr, ang, nz, R) == _path_ws(pr, ang, nz, R) + extra > extra, (P, H, R, A, noisy)


def test_symbols_are_exported():
    for f in ("pilco_particles_consistent_score_grad_workspace_bytes", "pilco_particles_consistent_score_grad_rollout"):
        assert hasattr(lib, f) and f in _lib.SIGNATURES
    header = open(os.path.join(ROOT, "include", "pilco_b200.h")).read()
    assert "pilco_particles_consistent_score_grad_rollout(" in header


def test_new_kernel_does_not_spill():
    """ptxas of particles_cscore.cu: pc_white_kernel has no stack frame and no spills; it holds no per-step or
    per-dimension array, so this one compile covers every D <= 16 and every H"""
    nvcc = "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not installed")
    res = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas", "-v",
                          "-cubin", "-o", os.devnull, os.path.join(ROOT, "pilco_b200", "csrc", "particles_cscore.cu")],
                         capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    props = dict(re.findall(r"Function properties for (\S+)\n\s*(.*)", res.stderr))
    pc = {k: v for k, v in props.items() if re.match(r"_Z\d+pc_", k)}
    assert len(pc) == 1, sorted(props)
    for name, p in pc.items():
        assert "0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads" in p, (name, p)


@pytest.mark.skipif(not os.path.exists(CUOBJDUMP), reason="cuobjdump not available")
def test_new_kernel_has_no_local_memory():
    sass = sass_named(["pc_white_kernel"])
    assert set(sass) == {"pc_white_kernel"}
    assert not re.search(r"\b(STL|LDL)\b", sass["pc_white_kernel"])


# ---- the engine -------------------------------------------------------------------------------------------------------
def test_engine_checks_before_any_allocation(monkeypatch):
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)
    with pytest.raises(ValueError, match="exploration"):
        engine.ConsistentGradPlan(None, None, None, 10, 3, estimator="score", exploration=0.5)
    with pytest.raises(ValueError, match="exploration"):
        engine.ConsistentGradPlan(None, None, None, 10, 3, estimator="score", exploration=0.0)
    for bad in ("reinforce", None, "Score"):
        with pytest.raises(ValueError, match="estimator"):
            engine.ConsistentGradPlan(None, None, None, 10, 3, estimator=bad)
    with pytest.raises(ValueError, match="ConsistentGradPlan"):          # the other spelling stays refused
        engine.ParticlePlan(None, None, None, 10, 3, consistent=True, estimator="score")
