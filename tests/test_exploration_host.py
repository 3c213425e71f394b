"""CPU tests of the exploration objective (DESIGN.md section 21): the numpy variance VJP against the golden fixture of
reward.m's six outputs, the per-term variance against Monte Carlo, the torch statement of the objective against its
autograd gradient and central differences (both signs of b, angles and joint terms), and the library side that needs no
GPU: exported symbols, the pilco_exploration layout, spill-free new kernels and validation before any device work."""
import ctypes
import os
import re
import subprocess

import numpy as np
import pytest
import torch

from pilco_b200 import _lib
from abi_fakes import ERR_DIM, ERR_NULL, ERR_UNSUP, ERR_WS, FAKE, _rollout
import action_reward_oracle as aro
import exploration_oracle as eo
from oracle import torch_port as tp
from particle_grad_oracle import T
from util import CUOBJDUMP, ROOT, make_gp_problem, sass

GOLDEN = os.path.join(ROOT, "tests", "golden", "reward_var.npz")


@pytest.mark.parametrize("kdim", [2, 5])
def test_variance_vjp_matches_reward_m(kdim):
    g = np.load(GOLDEN)
    m, s, W, t = (g["%s_%d" % (k, kdim)] for k in ("m", "s", "W", "t"))
    m, t = m.reshape(-1), t.reshape(-1)
    r1, dm1, dS1 = eo.exp_moment_vjp(m, s, W, t, 1.0)
    var, dm, dS = eo.exp_var_vjp(m, s, W, t)
    for got, ref in ((r1, g["muR_%d" % kdim]), (dm1, g["dmuRdm_%d" % kdim]), (dS1, g["dmuRdS_%d" % kdim]),
                     (var, g["sR_%d" % kdim]), (dm, g["dsRdm_%d" % kdim]), (dS, g["dsRdS_%d" % kdim])):
        ref = np.asarray(ref).reshape(np.shape(got))
        assert np.max(np.abs(got - ref)) <= 1e-12 * max(1.0, np.max(np.abs(ref)))
    assert g["sR_%d" % kdim].item() > aro.VAR_FLOOR                  # reward.m's clamp is not in play


def _torch_vjp(fn, m, s):
    mt, st = T(m).requires_grad_(), T(s).requires_grad_()
    gm, gs = torch.autograd.grad(fn(mt[None], st), (mt, st), allow_unused=True)
    gm = torch.zeros_like(mt) if gm is None else gm                 # a linear term's variance does not depend on m
    return gm.numpy(), 0.5 * (gs + gs.T).numpy()


def test_variance_vjp_matches_autograd():
    """the f-generalised exponential form and the linear form against autograd of the torch per-term variance"""
    rng = np.random.RandomState(3)
    for D in (1, 3, 7):
        B = rng.randn(D, D)
        s = 0.3 * B @ B.T
        C = rng.randn(D, D)
        W, t, m = C @ C.T / D + 0.1 * np.eye(D), rng.randn(D), rng.randn(D)
        term = dict(kind=_lib.REWARD_EXP, W=W, t=t)
        var, dm, dS = eo.exp_var_vjp(m, s, W, t)
        rm, rS = _torch_vjp(lambda a, b: aro.term_var(term, a, b), m, s)
        assert abs(var - float(aro.term_var(term, T(m)[None], T(s)))) < 1e-14
        assert np.max(np.abs(dm - rm)) < 1e-12 * max(1.0, np.max(np.abs(rm)))
        assert np.max(np.abs(dS - rS)) < 1e-12 * max(1.0, np.max(np.abs(rS)))
        for f in (1.0, 2.0, 0.5):                                   # r_f is r_1 with f W
            rf, dmf, dSf = eo.exp_moment_vjp(m, s, W, t, f)
            assert abs(rf - eo.exp_moment_vjp(m, s, f * W, t, 1.0)[0]) < 1e-14
            rm, rS = _torch_vjp(lambda a, b: tp.exponential_reward(a, b, T(f * W), T(t)[None])[0, 0], m, s)
            assert np.max(np.abs(dmf - rm)) < 1e-12 * max(1.0, np.max(np.abs(rm)))
            assert np.max(np.abs(dSf - rS)) < 1e-12 * max(1.0, np.max(np.abs(rS)))
        Wl = rng.randn(D)
        lterm = dict(kind=_lib.REWARD_LINEAR, W=Wl)
        var, dm, dS = eo.linear_var_vjp(m, s, Wl)
        rm, rS = _torch_vjp(lambda a, b: aro.term_var(lterm, a, b), m, s)
        assert abs(var - float(aro.term_var(lterm, T(m)[None], T(s)))) < 1e-13
        assert np.max(np.abs(dm - rm)) == 0.0 and np.max(np.abs(dS - rS)) < 1e-13


@pytest.mark.parametrize("kind", ["exp", "linear", "exp_sa"])
def test_term_variance_matches_monte_carlo(kind):
    from pilco_b200 import _lib
    rng = np.random.RandomState({"exp": 1, "linear": 2, "exp_sa": 3}[kind])
    D = 5 if kind == "exp_sa" else 3
    B = rng.randn(D, D)
    s, m = 0.2 * B @ B.T, 0.3 * rng.randn(D)
    if kind == "linear":
        W = rng.randn(D)
        term = dict(kind=_lib.REWARD_LINEAR, W=W)
        f = lambda x: x @ W
    else:
        C = rng.randn(D, D)
        W, t = C @ C.T / D, 0.2 * rng.randn(D)
        term = dict(kind=_lib.REWARD_EXP_SA if kind == "exp_sa" else _lib.REWARD_EXP, W=W, t=t)
        f = lambda x: np.exp(-0.5 * np.einsum("ni,ij,nj->n", x - t, W, x - t))
    x = rng.multivariate_normal(m, s, size=10 ** 6)
    r = f(x)
    mc = r.var()
    se = np.sqrt(np.mean((r - r.mean()) ** 4) / len(r))              # standard error of the variance estimate
    got = float(aro.term_var(term, T(m)[None], T(s)))
    assert abs(got - mc) < 5 * se + 1e-12, (got, mc, se)


def _objective_case(angle_dims, kind, b, seed=0):
    """a small cascade with state and joint terms on both channels (the MULT ones must not enter sigma)"""
    from pilco_b200 import _lib
    Ds, U = 3, 1
    A = len(angle_dims)
    Dh = Ds + A
    D = Dh + U
    X, Y, ell, sf2, sn2 = make_gp_problem(40, D, Ds, seed=seed)
    rng = np.random.RandomState(seed + 1)
    maxa = 1.2 * np.ones(U)
    Bj = rng.randn(D, D)
    terms = [dict(kind=_lib.REWARD_EXP, coef=1.0, W=np.diag(0.5 + rng.rand(Ds)), t=0.3 * rng.randn(Ds)),
             dict(kind=_lib.REWARD_LINEAR, coef=0.4, W=rng.randn(Ds), t=None),
             dict(kind=_lib.REWARD_EXP_SA, coef=-0.5, W=0.2 * Bj @ Bj.T, t=0.2 * rng.randn(D)),
             dict(kind=_lib.REWARD_LINEAR_SA, coef=0.3, W=rng.randn(D), t=None),
             dict(kind=_lib.REWARD_EXP, coef=0.2, channel=_lib.CHANNEL_MULT, W=np.eye(Ds), t=np.zeros(Ds))]
    if kind == "linear":
        params = [T(0.3 * rng.randn(U, Dh)), T(0.1 * rng.randn(U))]
    else:
        params = [T(0.5 * rng.randn(6, Dh)), T(0.3 * rng.randn(6, U)), T(1.0 + 0.1 * rng.rand(U, Dh))]
    Bs = rng.randn(Ds, Ds)
    m0, S0 = T(0.5 * rng.rand(Ds)), T(0.05 * Bs @ Bs.T)
    fn = lambda prm, m, S: aro.problem_rollout(kind, prm, X, 0.05 * Y, ell, sf2, sn2, maxa, terms, m, S, 4, mult_mu=2.0,
                                               angle_dims=angle_dims, b=b)
    return fn, params, m0, S0, terms


@pytest.mark.parametrize("angle_dims,kind,b", [([], "linear", 0.5), ([], "rbf", -0.5), ([1], "linear", -0.7),
                                               ([1], "rbf", 0.5)])
def test_objective_gradient_matches_central_differences(angle_dims, kind, b):
    fn, params, m0, S0, terms = _objective_case(angle_dims, kind, b)
    leaves = [p.clone().requires_grad_() for p in params] + [m0.clone().requires_grad_(), S0.clone().requires_grad_()]
    out = fn(leaves[:-2], leaves[-2], leaves[-1])
    assert torch.all(out["step_var"] > 1e-6)                        # the bonus is in play at every step
    grads = torch.autograd.grad(out["reward"], leaves)
    rng = np.random.RandomState(5)
    for k, (leaf, g) in enumerate(zip(leaves, grads)):
        v = torch.tensor(rng.randn(*leaf.shape), dtype=torch.float64)
        if k == len(leaves) - 1:
            v = 0.5 * (v + v.T)                                      # a symmetric direction for S0
        h = 1e-5
        vals = []
        for sgn in (1, -1):
            args = [p.detach().clone() for p in leaves]
            args[k] = args[k] + sgn * h * v
            vals.append(float(fn(args[:-2], args[-2], args[-1])["reward"]))
        fd = (vals[0] - vals[1]) / (2 * h)
        ad = float((g * v).sum())
        assert abs(fd - ad) < 1e-7 * max(1.0, abs(ad)), (k, fd, ad)


def test_objective_definition():
    """b = 0 is the expected reward; the bonus is b sum_t sigma_t; the MULT term does not enter sigma"""
    fn0, params, m0, S0, terms = _objective_case([1], "linear", 0.0)
    fnb = _objective_case([1], "linear", 0.8)[0]
    o0, ob = fn0(params, m0, S0), fnb(params, m0, S0)
    assert torch.equal(o0["step_var"], ob["step_var"]) and torch.equal(o0["traj_m"], ob["traj_m"])
    sig = torch.sqrt(o0["step_var"])
    assert abs(float(ob["reward"] - o0["reward"] - 0.8 * sig.sum())) < 1e-13
    assert aro.sigma(torch.tensor([0.0, 1e-12, 4e-12], dtype=torch.float64)).tolist() == [0.0, 0.0, 2e-6]


# ---- the library -----------------------------------------------------------------------------------------------------
NEW = ("pilco_rollout_explore_workspace_bytes", "pilco_rollout_explore_bwd_workspace_bytes",
       "pilco_rollout_explore_forward", "pilco_rollout_explore_backward")
KERNELS = ("ro_reward_var_kernel", "ro_reward_joint_var_kernel", "ro_reward_explore_sum_kernel", "rb_reward_var_kernel",
           "rb_reward_joint_var_kernel")


def test_library_exports_the_entry_points():
    from pilco_b200 import _lib
    for name in NEW:
        assert hasattr(_lib.lib, name) and name in _lib.SIGNATURES
    header = open(os.path.join(ROOT, "include", "pilco_b200.h")).read()
    assert all(name + "(" in header for name in NEW)


def test_exploration_layout(tmp_path):
    from pilco_b200 import _lib
    src = tmp_path / "ex_layout.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "%s"\nint main(void) { printf("%%zu %%zu %%zu\\n", '
                   'sizeof(pilco_exploration), offsetof(pilco_exploration, b), offsetof(pilco_exploration, step_var)); '
                   'return 0; }\n' % os.path.join(ROOT, "include", "pilco_b200.h"))
    exe = str(tmp_path / "ex_layout")
    subprocess.check_call(["gcc", "-o", exe, str(src)])
    size, ob, osv = map(int, subprocess.check_output([exe], text=True).split())
    assert (ctypes.sizeof(_lib.Exploration), _lib.Exploration.b.offset, _lib.Exploration.step_var.offset) == (size, ob, osv)


def test_new_kernels_do_not_spill():
    nvcc = "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not installed")
    res = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas", "-v",
                          "-cubin", "-o", os.devnull, os.path.join(ROOT, "pilco_b200", "csrc", "rollout_explore.cu")],
                         capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    props = dict(re.findall(r"Function properties for (\S+)\n\s*(.*)", res.stderr))
    for k in KERNELS:
        name = next(n for n in props if k in n)
        assert "0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads" in props[name], (name, props[name])
    if os.path.exists(CUOBJDUMP):
        text = sass("|".join(KERNELS))
        assert len(text) == len(KERNELS), sorted(text)
        for name, t in text.items():
            assert not re.search(r"\b(STL|LDL)\b", t), "local memory traffic in %s" % name


def _ex(b, step_var=None):
    from pilco_b200 import _lib
    return _lib.Exploration(b, step_var)


def test_validation_before_device_work():
    """Every rejected call returns before it enqueues anything (the fake pointers are never dereferenced); an inactive
    call is the call without exploration."""
    from pilco_b200 import _lib
    lib, C = _lib.lib, ctypes
    g = _lib.RolloutGrad()
    fwd = lambda ro, ex: lib.pilco_rollout_explore_forward(C.byref(ro), None, C.byref(ex), None)
    bwd = lambda ro, ex: lib.pilco_rollout_explore_backward(C.byref(ro), None, C.byref(ex), C.byref(g), None)
    ro = _rollout()
    need = lib.pilco_rollout_explore_workspace_bytes(C.byref(ro), None, C.byref(_ex(0.5)))
    base = lib.pilco_rollout_workspace_bytes(C.byref(ro))
    assert need == base + 8 * (ro.R * ro.H + (ro.R * ro.H) % 2)
    for call in (fwd, bwd):
        for bad in (float("nan"), float("inf"), -float("inf")):
            assert call(ro, _ex(bad)) == ERR_DIM
        assert call(ro, _ex(0.5)) == ERR_WS                                      # ws_bytes = 0
        ro.ws_bytes = base
        assert call(ro, _ex(0.5)) == ERR_WS                                      # enough for the call without it only
        assert call(ro, _ex(0.0, FAKE)) == ERR_WS                                # step_var alone makes the call active
        box = _rollout(reward_kind=_lib.REWARD_BOX)
        box.ws_bytes = need
        assert call(box, _ex(0.5)) == ERR_UNSUP                                  # an additive box term
        assert call(box, _ex(0.0, FAKE)) == ERR_UNSUP
        nul = _rollout()
        nul.m0 = None
        assert call(nul, _ex(0.5)) == ERR_NULL                                   # the codes of the underlying call
        ro.ws_bytes = 0
    risk = _rollout(reward_kind=_lib.REWARD_BOX, channel=_lib.CHANNEL_MULT)      # a MULT box term is fine: the
    assert fwd(risk, _ex(0.5)) == ERR_WS                                         # workspace check comes next
    # inactive: NULL, or b = 0 without step_var -> the call without exploration (its status and workspace sizes)
    assert lib.pilco_rollout_explore_forward(C.byref(ro), None, None, None) == ERR_WS
    assert fwd(ro, _ex(0.0)) == ERR_WS
    assert lib.pilco_rollout_explore_forward(C.byref(nul), None, None, None) == ERR_NULL
    for ex in (None, C.byref(_ex(0.0))):
        assert lib.pilco_rollout_explore_workspace_bytes(C.byref(ro), None, ex) == base
        assert (lib.pilco_rollout_explore_bwd_workspace_bytes(C.byref(ro), None, ex)
                == lib.pilco_rollout_bwd_workspace_bytes(C.byref(ro)))
    assert (lib.pilco_rollout_explore_bwd_workspace_bytes(C.byref(ro), None, C.byref(_ex(0.5)))
            == lib.pilco_rollout_bwd_workspace_bytes(C.byref(ro)))


def test_python_validation():
    """RolloutPlan rejects a non-finite b and an additive box term before any device work"""
    from pilco_b200 import engine, _lib
    box = [dict(kind=_lib.REWARD_BOX, coef=-1.0, W=np.array([1.0, 1.0, 1.0, 0.0, -1.0, 1.0]), t=None)]
    with pytest.raises(ValueError, match="finite"):
        engine.RolloutPlan(None, dict(Ds=3, U=1), box, np.zeros(3), np.eye(3), 5, exploration=float("nan"))
    with pytest.raises(ValueError, match="box"):
        engine.RolloutPlan(None, dict(Ds=3, U=1), box, np.zeros(3), np.eye(3), 5, exploration=0.5)
    with pytest.raises(ValueError, match="box"):
        engine.RolloutPlan(None, dict(Ds=3, U=1), box, np.zeros(3), np.eye(3), 5, exploration=0.0)
