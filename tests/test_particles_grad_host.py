"""CPU tests of the particle rollout's pathwise gradient (pilco_particles_rollout_grad, pilco_gp_predict_vjp,
PILCO.sample_policy_gradient, PILCO.policy_gradient): the torch autograd oracle (tests/particle_grad_oracle.py) against
central finite differences of the numpy particle oracle, the closed-form predict VJP against autograd, the
pilco_particles_grad layout against its ctypes mirror, argument validation of the new entry points (rejecting calls
only), the kernels' SASS and the failure without a GPU."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest
import torch

from pilco_b200 import _lib
from pilco_b200._lib import lib
from abi_fakes import ERR_ALIGN, ERR_DIM, ERR_NULL, ERR_UNSUP, ERR_WS, FAKE, _gp, _grad, _particles
from particle_cases import _problem, _terms
from particle_oracle import particle_rollout
from particle_grad_oracle import predict_vjp, rbf_pol_np, value_and_grad
from util import CUOBJDUMP, ROOT, sass_named


def _fd_check(dyn, pol, key_map, terms, x0, eps, mu, h=1e-6):
    """autograd gradient against central differences of the numpy oracle's mean return, every parameter"""
    v, g = value_and_grad(dyn, pol, terms, x0, eps, mu)
    worst, scale = 0.0, max(np.abs(gv).max() for gv in g.values())
    for k, (src, rebuild) in key_map.items():
        base = np.asarray(pol[src], dtype=np.float64)
        for idx in np.ndindex(base.shape):
            vals = []
            for s in (1.0, -1.0):
                p = base.copy(); p[idx] += s * h
                vals.append(particle_rollout(dyn, rebuild(src, p), terms, x0, eps, mu)[4].mean())
            fd = (vals[0] - vals[1]) / (2 * h)
            worst = max(worst, abs(fd - g[k][idx]) / scale)
    ref_v = particle_rollout(dyn, rebuild(src, base), terms, x0, eps, mu)[4].mean()
    return worst, abs(v - ref_v)


def test_autograd_oracle_matches_finite_differences_linear():
    dyn, rng = _problem(1)
    Ds, U, P, H = 3, 1, 40, 4
    W, b, maxa = 0.7 * rng.randn(U, Ds), rng.randn(U), np.array([1.2])
    x0, eps = 0.5 + 0.2 * rng.randn(P, Ds), rng.randn(P, H, Ds)
    for squash in (True, False):
        pol = dict(kind=_lib.POLICY_LINEAR, squash=squash, maxa=maxa, W=W, b=b)

        def rebuild(src, p):
            q = dict(pol); q[src] = p
            return q
        worst, dv = _fd_check(dyn, pol, {"W": ("W", rebuild), "b": ("b", rebuild)}, _terms(Ds), x0, eps, -2.0)
        print("linear (squash=%s): autograd vs central differences %.1e of scale, value %.1e" % (squash, worst, dv))
        assert worst < 1e-6 and dv < 1e-13


def test_autograd_oracle_matches_finite_differences_rbf():
    dyn, rng = _problem(2)
    Ds, U, bf, P, H = 3, 1, 6, 30, 3
    Xc, Yc, lc, maxa = rng.rand(bf, Ds), 0.5 * rng.randn(bf, U), 0.6 + 0.3 * rng.rand(U, Ds), np.array([0.9])
    x0, eps = 0.5 + 0.2 * rng.randn(P, Ds), rng.randn(P, H, Ds)
    prm = dict(Xc=Xc, Yc=Yc, ell=lc)

    def rebuild(src, p):
        q = dict(prm); q[src] = p
        return rbf_pol_np(q["Xc"], q["Yc"], q["ell"], maxa)
    pol = dict(kind=_lib.POLICY_RBF, squash=True, maxa=maxa, Xc=Xc, Yc=Yc, ell=lc, sf2=np.ones(U), sn2=1e-4 * np.ones(U))
    worst, dv = _fd_check(dyn, pol, {"X": ("Xc", rebuild), "Y": ("Yc", rebuild), "ell": ("ell", rebuild)},
                          _terms(Ds), x0, eps, 1.5)
    print("rbf: autograd vs central differences %.1e of scale, value %.1e" % (worst, dv))
    assert worst < 1e-6 and dv < 1e-13


def test_predict_vjp_closed_form_matches_autograd():
    dyn, rng = _problem(3, n=30, Ds=3, U=2)
    T = 17
    Xs, gm, gv = rng.rand(T, 5), rng.randn(T, 3), rng.randn(T, 3)
    g, scale = predict_vjp(dyn, Xs, gm, gv)
    x = torch.tensor(Xs, requires_grad=True)
    C_, ell, sf2, iK, beta = (torch.as_tensor(dyn[k]) for k in ("C", "ell", "sf2", "iK", "beta"))
    tot = 0.0
    for e in range(3):
        d = (x[:, None] - C_[None]) / ell[e]
        K = sf2[e] * torch.exp(-0.5 * (d * d).sum(-1))
        tot = tot + (torch.as_tensor(gm[:, e]) * (K @ beta[e])).sum() \
            + (torch.as_tensor(gv[:, e]) * (sf2[e] - ((K @ iK[e]) * K).sum(1))).sum()
    ga = torch.autograd.grad(tot, x)[0].numpy()
    err = np.max(np.abs(ga - g) / scale)
    print("closed-form predict VJP vs autograd: %.1e of sum |terms|" % err)
    assert err < 1e-13


def test_particles_grad_struct_layout_matches_mirror(tmp_path):
    fields = ["gW", "gb", "gXc", "gYc", "gell", "pol_L", "value", "ws", "ws_bytes"]
    src = tmp_path / "grad_layout.c"
    src.write_text("#include <stdio.h>\n#include <stddef.h>\n#include \"%s\"\nint main(void) {\n"
                   "    printf(\"sizeof %%zu\\n\", sizeof(pilco_particles_grad));\n%s    return 0;\n}\n"
                   % (os.path.join(ROOT, "include", "pilco_b200.h"),
                      "".join("    printf(\"%s %%zu\\n\", offsetof(pilco_particles_grad, %s));\n" % (f, f) for f in fields)))
    exe = str(tmp_path / "grad_layout")
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Werror", "-o", exe, str(src)])
    got = dict(line.split() for line in subprocess.check_output([exe], text=True).splitlines())
    assert C.sizeof(_lib.ParticlesGrad) == int(got.pop("sizeof"))
    assert set(got) == set(fields)
    for f, off in got.items():
        assert getattr(_lib.ParticlesGrad, f).offset == int(off), f


def _run(pr, g):
    return lib.pilco_particles_rollout_grad(C.byref(pr) if pr is not None else None,
                                            C.byref(g) if g is not None else None, None)


def test_particles_grad_argument_validation():
    assert _run(None, _grad()) == ERR_NULL
    assert _run(_particles(), None) == ERR_NULL
    assert _run(_particles(), _grad()) == ERR_WS                            # valid description, no workspace
    for kind in (_lib.POLICY_LINEAR, _lib.POLICY_RBF):
        for rk in (_lib.REWARD_EXP, _lib.REWARD_LINEAR, _lib.REWARD_BOX):
            for ch in (_lib.CHANNEL_ADD, _lib.CHANNEL_MULT):
                assert _run(_particles(kind, rk, ch), _grad()) == ERR_WS, (kind, rk, ch)
    pr = _particles(); pr.ws = None                                         # the forward's workspace is not used
    assert _run(pr, _grad()) == ERR_WS
    assert _run(_particles(H=0), _grad()) == ERR_WS
    for P, H in ((0, 5), (65535 * 32 + 1, 5), (10, -1)):
        assert _run(_particles(P=P, H=H), _grad()) == ERR_DIM, (P, H)
    for field in ("x0", "eps", "traj", "act", "step_reward", "step_risk", "ret"):    # the forward's arguments
        pr = _particles(); setattr(pr, field, None)
        assert _run(pr, _grad()) == ERR_NULL, field
    pr = _particles(); pr.dyn.iK = None
    assert _run(pr, _grad()) == ERR_UNSUP
    pr = _particles(); pr.dyn.mode = 1
    assert _run(pr, _grad()) == ERR_UNSUP
    pr = _particles(_lib.POLICY_RBF); pr.pol.rbf.beta_bs = 20
    assert _run(pr, _grad()) == ERR_UNSUP
    assert _run(_particles(kind=7), _grad()) == ERR_UNSUP
    assert _run(_particles(reward_kind=9), _grad()) == ERR_UNSUP
    assert _run(_particles(channel=5), _grad()) == ERR_UNSUP
    pr = _particles(); pr.dyn.E = 4
    assert _run(pr, _grad()) == ERR_DIM
    pr = _particles(); pr.dyn.iK = FAKE + 8
    assert _run(pr, _grad()) == ERR_ALIGN
    for field in ("value", "ws", "gW", "gb"):
        g = _grad(); setattr(g, field, None)
        assert _run(_particles(), g) == ERR_NULL, field
    for field in ("gXc", "gYc", "gell", "pol_L"):                           # pol_L: the RBF policy's Cholesky factors
        g = _grad(); setattr(g, field, None)
        assert _run(_particles(_lib.POLICY_RBF), g) == ERR_NULL, field
        assert _run(_particles(), g) == ERR_WS, field                       # not needed by the linear policy
    g = _grad(); g.gW = g.gb = None
    assert _run(_particles(_lib.POLICY_RBF), g) == ERR_WS
    g = _grad(); g.ws = FAKE + 8; g.ws_bytes = 1 << 40
    assert _run(_particles(), g) == ERR_ALIGN
    for kind in (_lib.POLICY_LINEAR, _lib.POLICY_RBF):
        pr = _particles(kind)
        need = lib.pilco_particles_grad_workspace_bytes(C.byref(pr))
        g = _grad(); g.ws_bytes = need - 8
        assert need > 0 and _run(pr, g) == ERR_WS


def test_particles_grad_workspace_bytes():
    f = lambda pr: lib.pilco_particles_grad_workspace_bytes(C.byref(pr) if pr is not None else None)
    assert f(None) == 0
    for P, H in ((0, 5), (65535 * 32 + 1, 5), (10, -1)):
        assert f(_particles(P=P, H=H)) == 0
    P, H, Ds, U, D, n = 1000, 5, 3, 1, 4, 50
    pred = lib.pilco_gp_predict_workspace_bytes(n, D, Ds, P, 0)
    vjp = lib.pilco_gp_predict_vjp_workspace_bytes(n, D, Ds, P)
    assert f(_particles(P=P, H=H)) >= 8 * P * H * (D + Ds + U) + max(pred, vjp)
    big = _particles(P=100000, H=40)
    assert f(big) < 8 * 100000 * (40 * (D + Ds + U) + 64)                  # O(P H (Ds+U)), no [P, n] intermediate


def test_predict_vjp_argument_validation():
    def run(gp=None, T=100, ptrs=(FAKE,) * 5, ws_bytes=1 << 40):
        gp = _gp() if gp is None else gp
        return lib.pilco_gp_predict_vjp(C.byref(gp), T, *ptrs[:4], ptrs[4], ws_bytes, None)
    assert lib.pilco_gp_predict_vjp(None, 10, FAKE, FAKE, FAKE, FAKE, FAKE, 1 << 40, None) == ERR_NULL
    for k in range(5):
        p = [FAKE] * 5; p[k] = None
        assert run(ptrs=p) == ERR_NULL, k
    for field in ("X", "ell", "sf2", "beta"):
        gp = _gp(); setattr(gp, field, None)
        assert run(gp) == ERR_NULL, field
    assert run(_gp(mode=1)) == ERR_UNSUP
    assert run(_gp(iK=None)) == ERR_UNSUP
    gp = _gp(); gp.X_bs = 200
    assert run(gp) == ERR_UNSUP
    for T in (0, 65535 * 32 + 1):
        assert run(T=T) == ERR_DIM, T
    assert run(_gp(D=17)) == ERR_DIM
    assert run(_gp(E=17)) == ERR_DIM
    assert run(_gp(ldk=32)) == ERR_DIM
    assert run(_gp(iK=FAKE + 8)) == ERR_ALIGN
    assert run(_gp(ldk=65)) == ERR_ALIGN
    assert run(ptrs=(FAKE,) * 4 + (FAKE + 8,)) == ERR_ALIGN
    need = lib.pilco_gp_predict_vjp_workspace_bytes(50, 4, 3, 100)
    assert need > 0 and run(ws_bytes=need - 8) == ERR_WS
    assert lib.pilco_gp_predict_vjp_workspace_bytes(50, 4, 3, 65535 * 32 + 1) == 0
    assert lib.pilco_gp_predict_vjp_workspace_bytes(50, 17, 3, 10) == 0


@pytest.mark.skipif(not os.path.exists(CUOBJDUMP), reason="cuobjdump not available")
def test_gradient_kernels_sass():
    names = ["gp_predict_vjp_kernel", "pg_step_kernel", "pg_param_kernel", "pg_rbf_finish_kernel"]
    sass = sass_named(names)
    assert set(sass) == set(names)
    for k, text in sass.items():
        assert not re.search(r"\b(STL|LDL)\b", text), k
    assert "DMMA.16x8x16" in sass["gp_predict_vjp_kernel"] and "UBLKCP" in sass["gp_predict_vjp_kernel"]


def test_gradient_methods_fail_loudly_without_gpu(monkeypatch):
    from pilco.models import PILCO
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)
    X = np.random.RandomState(0).rand(20, 3); Y = 0.1 * X[:, :2]
    pilco = PILCO((X, Y))
    with pytest.raises(RuntimeError, match="CUDA device"):
        pilco.sample_policy_gradient(X[0, :2], 0.1 * np.eye(2), 3, num_samples=10, seed=0)
    with pytest.raises(RuntimeError, match="CUDA device"):
        pilco.policy_gradient()
