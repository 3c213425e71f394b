"""CPU tests of the particle rollout (pilco_particles_rollout, PILCO.sample_trajectories): argument validation of the C
entry points (rejecting calls only: a call that passed validation would launch kernels), the pilco_particles layout
against its ctypes mirror, the host build of the box-indicator formula, the kernel's SASS, the failure without a GPU,
and the numpy particle oracle (tests/particle_oracle.py) against the moment-matching oracle where moment matching is
exact."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest
import torch

from oracle import python_port as pp
from pilco_b200 import _lib
from pilco_b200._lib import lib
from abi_fakes import ERR_ALIGN, ERR_DIM, ERR_NULL, ERR_UNSUP, ERR_WS, FAKE, _particles
from particle_oracle import moment_check, particle_rollout
from util import CUOBJDUMP, ROOT, sass


def _run(pr):
    return lib.pilco_particles_rollout(C.byref(pr) if pr is not None else None, None)


def test_particles_argument_validation():
    assert _run(None) == ERR_NULL
    assert _run(_particles()) == ERR_WS                                     # valid description, no workspace
    for kind in (_lib.POLICY_LINEAR, _lib.POLICY_RBF):
        for rk in (_lib.REWARD_EXP, _lib.REWARD_LINEAR, _lib.REWARD_BOX):
            for ch in (_lib.CHANNEL_ADD, _lib.CHANNEL_MULT):
                assert _run(_particles(kind, rk, ch)) == ERR_WS, (kind, rk, ch)
    assert _run(_particles(H=0)) == ERR_WS
    for P, H in ((0, 5), (65535 * 32 + 1, 5), (10, -1)):
        assert _run(_particles(P=P, H=H)) == ERR_DIM, (P, H)
    for field in ("x0", "eps", "traj", "act", "step_reward", "step_risk", "ret", "ws"):
        pr = _particles(); setattr(pr, field, None)
        assert _run(pr) == ERR_NULL, field
    pr = _particles(); pr.dyn.beta = None
    assert _run(pr) == ERR_NULL
    pr = _particles(); pr.pol.W = None
    assert _run(pr) == ERR_NULL
    pr = _particles(); pr.pol.max_action = None
    assert _run(pr) == ERR_NULL
    pr = _particles(); pr.rewards[0].t = None                               # the exp reward needs its target
    assert _run(pr) == ERR_NULL
    pr = _particles(); pr.rewards[0].W = None
    assert _run(pr) == ERR_NULL
    pr = _particles(); pr.dyn.mode = 1
    assert _run(pr) == ERR_UNSUP
    pr = _particles(); pr.dyn.iK = None
    assert _run(pr) == ERR_UNSUP
    pr = _particles(); pr.dyn.X_bs = 50 * 4                                 # batched dynamics
    assert _run(pr) == ERR_UNSUP
    pr = _particles(); pr.pol.W_bs = 3                                      # batched linear policy
    assert _run(pr) == ERR_UNSUP
    pr = _particles(_lib.POLICY_RBF); pr.pol.rbf.beta_bs = 20              # batched RBF policy
    assert _run(pr) == ERR_UNSUP
    pr = _particles(_lib.POLICY_RBF); pr.pol.rbf.mode = 0
    assert _run(pr) == ERR_UNSUP
    assert _run(_particles(kind=7)) == ERR_UNSUP
    assert _run(_particles(reward_kind=9)) == ERR_UNSUP
    assert _run(_particles(channel=5)) == ERR_UNSUP
    pr = _particles(); pr.pol.U = 2                                         # Ds + U != dyn.D
    assert _run(pr) == ERR_DIM
    pr = _particles(); pr.dyn.E = 4                                         # E != Ds
    assert _run(pr) == ERR_DIM
    pr = _particles(); pr.dyn.D = 17; pr.pol.U = 14
    assert _run(pr) == ERR_DIM
    pr = _particles(); pr.dyn.ldk = 32                                      # ldk < pilco_pad_n(n)
    assert _run(pr) == ERR_DIM
    pr = _particles(_lib.POLICY_RBF); pr.pol.rbf.E = 2                      # RBF outputs != U
    assert _run(pr) == ERR_DIM
    for nr in (0, 9):
        pr = _particles(); pr.n_rewards = nr
        assert _run(pr) == ERR_DIM
    pr = _particles(); pr.dyn.iK = FAKE + 8
    assert _run(pr) == ERR_ALIGN
    pr = _particles(); pr.dyn.ldk = 65
    assert _run(pr) == ERR_ALIGN
    pr = _particles(); pr.ws = FAKE + 8; pr.ws_bytes = 1 << 40
    assert _run(pr) == ERR_ALIGN
    pr = _particles()
    need = lib.pilco_particles_workspace_bytes(C.byref(pr))
    pr.ws_bytes = need - 8
    assert need > 0 and _run(pr) == ERR_WS


def test_particles_workspace_bytes():
    f = lambda pr: lib.pilco_particles_workspace_bytes(C.byref(pr) if pr is not None else None)
    assert f(None) == 0
    for P, H in ((0, 5), (65535 * 32 + 1, 5), (10, -1)):
        assert f(_particles(P=P, H=H)) == 0
    pr = _particles(P=1000, H=5)
    pred = lib.pilco_gp_predict_workspace_bytes(50, 4, 3, 1000, 0)
    assert f(pr) >= 8 * 1000 * (4 + 3 + 3) + pred                          # x~ [P,D], mean and var [P,Ds], predict's
    assert f(pr) == f(_particles(P=1000, H=40))                            # nothing scales with H
    assert f(_particles(P=100000)) < 8 * 100000 * 64                       # O(P), no [P, n] intermediate


def test_particles_struct_layout_matches_mirror(tmp_path):
    """pilco_particles as the C compiler lays it out (include/pilco_b200.h) against the ctypes mirror."""
    fields = ["P", "H", "dyn", "pol", "n_rewards", "rewards", "mult_mu", "x0", "eps", "traj", "act", "step_reward",
              "step_risk", "ret", "ws", "ws_bytes"]
    src = tmp_path / "particles_layout.c"
    src.write_text("#include <stdio.h>\n#include <stddef.h>\n#include \"%s\"\nint main(void) {\n"
                   "    printf(\"sizeof %%zu\\n\", sizeof(pilco_particles));\n%s    return 0;\n}\n"
                   % (os.path.join(ROOT, "include", "pilco_b200.h"),
                      "".join("    printf(\"%s %%zu\\n\", offsetof(pilco_particles, %s));\n" % (f, f) for f in fields)))
    exe = str(tmp_path / "particles_layout")
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Werror", "-o", exe, str(src)])
    got = dict(line.split() for line in subprocess.check_output([exe], text=True).splitlines())
    assert C.sizeof(_lib.Particles) == int(got.pop("sizeof"))
    assert set(got) == set(fields)
    for f, off in got.items():
        assert getattr(_lib.Particles, f).offset == int(off), f


def test_box_point_formula_on_host(tmp_path):
    """risk_box_point (pilco_b200/csrc/risk_math.cuh, the formula the particle kernel executes) compiled for the host:
    the indicator of the open box, complemented when inside = 0, and the limit of risk_box_eval as s -> 0."""
    src = tmp_path / "box_point.cpp"
    src.write_text('#include "%s"\nextern "C" double box_point(const double* prm, const double* x) '
                   '{ return risk_box_point(prm, x); }\n'
                   'extern "C" double box_eval(int Ds, const double* prm, const double* m, const double* s) '
                   '{ return risk_box_eval(Ds, prm, m, s, nullptr, nullptr); }\n'
                   % os.path.join(ROOT, "pilco_b200", "csrc", "risk_math.cuh"))
    so = str(tmp_path / "box_point.so")
    subprocess.check_call(["g++", "-O1", "-shared", "-fPIC", "-o", so, str(src)])
    h = C.CDLL(so)
    dp = C.POINTER(C.c_double)
    h.box_point.restype = h.box_eval.restype = C.c_double
    h.box_point.argtypes = [dp, dp]
    h.box_eval.argtypes = [C.c_int, dp, dp, dp]
    c = lambda a: np.ascontiguousarray(a, dtype=np.float64).ctypes.data_as(dp)
    inf = float("inf")
    rng = np.random.RandomState(0)
    Ds = 4
    for dims, lows, highs, inside in [((0, 2), (-0.3, -1.0), (0.4, 0.2), 1.0), ((1,), (-0.2,), (inf,), 1.0),
                                      ((3,), (-inf,), (0.7,), 1.0), ((2,), (-0.5,), (0.6,), 0.0)]:
        prm = np.array([len(dims), inside, 1.0] + [v for k in range(len(dims)) for v in (dims[k], lows[k], highs[k])])
        for _ in range(200):
            x = rng.randn(Ds)
            ins = all(lo < x[d] < hi for d, lo, hi in zip(dims, lows, highs))
            assert h.box_point(c(prm), c(x)) == float(ins == bool(inside))
            if min(min(abs(x[d] - lo), abs(x[d] - hi)) for d, lo, hi in zip(dims, lows, highs)) > 1e-3:
                lim = h.box_eval(Ds, c(prm), c(x), c(1e-12 * np.eye(Ds)))
                assert abs(lim - h.box_point(c(prm), c(x))) < 1e-12
        x = np.zeros(Ds)
        x[dims[0]] = lows[0] if np.isfinite(lows[0]) else highs[0]          # on the boundary: outside (open box)
        assert h.box_point(c(prm), c(x)) == float(not bool(inside))


@pytest.mark.skipif(not os.path.exists(CUOBJDUMP), reason="cuobjdump not available")
def test_particle_step_kernel_has_no_local_memory():
    funcs = sass(r"pt_step_kernel")
    assert len(funcs) == 1
    text = next(iter(funcs.values()))
    assert not re.search(r"\b(STL|LDL)\b", text)


def test_sample_trajectories_fails_loudly_without_gpu(monkeypatch):
    from pilco.models import PILCO
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)
    X = np.random.RandomState(0).rand(20, 3); Y = 0.1 * X[:, :2]
    pilco = PILCO((X, Y))
    with pytest.raises(RuntimeError, match="CUDA device"):
        pilco.sample_trajectories(X[0, :2], 0.1 * np.eye(2), 3, num_samples=10, seed=0)


def test_oracle_one_step_moments_match_moment_matching():
    """From a Gaussian x0 under a linear unsquashed policy the joint input is Gaussian and moment matching gives the
    exact mean and covariance of x1 and the exact expected step-0 reward: the particle oracle must agree with the
    moment-matching oracle within 5 standard errors at 1e5 particles."""
    rng = np.random.RandomState(4)
    Ds, U, n, P = 3, 1, 60, 100000
    D = Ds + U
    X = rng.rand(n, D)
    Y = 0.3 * np.sin(3.0 * X).dot(rng.rand(D, Ds))
    ell, sf2, sn2 = 0.6 + 0.4 * rng.rand(Ds, D), 0.05 * (1.0 + rng.rand(Ds)), 1e-3 * np.ones(Ds)
    iK, beta = pp.calculate_factorizations(X, Y, ell, sf2, sn2)
    W, b = rng.randn(U, Ds), rng.randn(U)
    m0, S0 = X[0, :Ds], 0.08 * np.eye(Ds) + 0.02
    Wr, tr = np.diag([1.0, 2.0, 0.5]), 0.3 * np.ones(Ds)
    M1, S1 = pp.propagate(m0[None], S0, lambda m, s: pp.linear_action(W, b, m, s, False),
                          lambda m, s: pp.predict_given_factorizations(X, ell, sf2, m, s, iK, beta))
    r0 = pp.exponential_reward(m0[None], S0, Wr, tr[None])[0][0, 0]
    x0 = m0[None] + rng.randn(P, Ds) @ np.linalg.cholesky(S0).T
    eps = rng.randn(P, 1, Ds)
    dyn = dict(C=X, ell=ell, sf2=sf2, iK=iK, beta=beta)
    pol = dict(kind=_lib.POLICY_LINEAR, W=W, b=b, squash=False)
    traj, act, rew, risk, ret = particle_rollout(dyn, pol, [dict(kind=_lib.REWARD_EXP, W=Wr, t=tr)], x0, eps)
    worst = moment_check(traj[:, 1], M1[0], S1)
    z = (rew[:, 0].mean() - r0) / (rew[:, 0].std() / np.sqrt(P))
    print("one-step moments, oracle particles vs moment matching: worst %.2f standard errors, reward %.2f" % (worst, z))
    assert worst <= 5.0 and abs(z) <= 5.0
    assert np.array_equal(ret, rew[:, 0]) and not risk.any()
    assert np.max(np.abs(act[:, 0] - (x0 @ W.T + b))) < 1e-14
