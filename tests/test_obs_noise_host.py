"""CPU tests of measurement noise at the policy's input (pilco_rollout_noisy_*, DESIGN.md section 22): the torch
statement (tests/action_reward_oracle.py's cascade with v) against propagate.m's composition
(tests/golden/obs_noise.npz), bitwise the cascade without v at v = 0, against 10^6 Monte Carlo draws in the exact H = 1
case and its autograd gradient against central differences; and the library side that needs no GPU: exported symbols,
the pilco_obs_noise layout, the new kernels' registers and local memory, and validation before any device work."""
import ctypes
import os
import re
import subprocess

import numpy as np
import pytest
import torch

from abi_fakes import ERR_DIM, ERR_NULL, ERR_UNSUP, ERR_WS, FAKE, _rollout
import action_reward_oracle as aro
import particle_oracle as po
from oracle import torch_port as tp
from particle_grad_oracle import T
from util import CUOBJDUMP, ROOT, make_gp_problem, sass

GOLDEN = os.path.join(ROOT, "tests", "golden", "obs_noise.npz")


def _problem(kind, Ds=3, U=2, dims=(), seed=4, n=40, bf=10, squash=True):
    Dh = Ds + len(dims)
    X, Y, ell, sf2, sn2 = make_gp_problem(n, Dh + U, Ds, seed=seed)
    Y = 0.1 * Y
    rng = np.random.RandomState(seed + 1)
    maxa = 0.7 + rng.rand(U) if squash else None
    if kind == "linear":
        prm = [T(0.5 * rng.randn(U, Dh)), T(0.3 * rng.randn(U))]
    else:
        prm = [T(rng.randn(bf, Dh) * 0.5 + 0.5), T(0.1 * rng.randn(bf, U)), T(1.0 + 0.1 * rng.randn(U, Dh))]
    B = rng.randn(Ds, Ds)
    S0 = 0.03 * B @ B.T + 0.02 * np.eye(Ds)
    v = 0.01 + 0.04 * rng.rand(Ds)
    t = 0.3 * rng.randn(Ds)
    terms = [dict(kind=0, coef=1.0, W=np.diag(0.5 + rng.rand(Ds)), t=t), dict(kind=1, coef=0.3, W=rng.randn(Ds), t=None)]
    return dict(kind=kind, prm=prm, X=X, Y=Y, ell=ell, sf2=sf2, sn2=sn2, maxa=maxa, m0=X[0, :Ds], S0=S0, v=v,
                terms=terms, dims=list(dims) or None)


def _run(P, H, b=0.0, v=None, prm=None, m0=None, S0=None):
    return aro.problem_rollout(P["kind"], P["prm"] if prm is None else prm, P["X"], P["Y"], P["ell"], P["sf2"],
                               P["sn2"], P["maxa"], P["terms"], T(P["m0"]) if m0 is None else m0,
                               T(P["S0"]) if S0 is None else S0, H, angle_dims=P["dims"], v=P["v"] if v is None else v,
                               b=b)


# ---- propagate.m ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", ["linear", "rbf"])
def test_oracle_matches_propagate_m(case):
    """one noisy propagate.m step (gp2/conlin + gSin + gp0 composed with ss = S + diag(sn2), q = S C)"""
    if not os.path.exists(GOLDEN):
        pytest.skip("golden fixture not generated")
    g = np.load(GOLDEN)
    pre = case + "_"
    m, s, v = g[pre + "m"].reshape(-1), g[pre + "s"], g[pre + "sn2"].reshape(-1)
    iK, beta = tp.calculate_factorizations(T(g[pre + "X"]), T(g[pre + "Y"]), T(g[pre + "ell"]), T(g[pre + "sf2"]),
                                           T(g[pre + "sn2_dyn"]))
    dyn = lambda mm, ss: tp.predict_given_factorizations(T(g[pre + "X"]), T(g[pre + "ell"]), T(g[pre + "sf2"]), mm, ss,
                                                         iK, beta)
    ma = T(g[pre + "maxU"]).reshape(1, -1)
    if case == "linear":
        act = lambda mm, ss: tp.linear_action(T(g[pre + "W"]), T(g[pre + "b"]).reshape(1, -1), mm, ss, ma)
    else:
        act = lambda mm, ss: tp.rbf_action(T(g[pre + "Xc"]), T(g[pre + "Yc"]), T(g[pre + "lc"]), mm, ss, ma)
    out = aro.mm_rollout(dyn, act, [dict(kind=1, coef=1.0, W=np.zeros(len(m)), t=None)], T(m), T(s), 1, v=T(v))
    for got, ref in ((out["traj_m"][1], g[pre + "Mnext"]), (out["traj_S"][1], g[pre + "Snext"])):
        ref = np.asarray(ref).reshape(tuple(got.shape))
        assert np.max(np.abs(got.numpy() - ref)) <= 1e-12 * max(1.0, np.max(np.abs(ref)))


@pytest.mark.parametrize("kind,dims", [("linear", ()), ("rbf", ()), ("linear", (1,)), ("rbf", (0, 2))])
def test_zero_noise_is_the_noiseless_oracle_bitwise(kind, dims):
    P = _problem(kind, Ds=3, dims=dims)
    H, b = 4, 0.5
    got = _run(P, H, b=b, v=np.zeros(3))
    ref = aro.problem_rollout(kind, P["prm"], P["X"], P["Y"], P["ell"], P["sf2"], P["sn2"], P["maxa"], P["terms"],
                              T(P["m0"]), T(P["S0"]), H, angle_dims=P["dims"], b=b)
    for k in ("traj_m", "traj_S", "step_reward", "step_var", "reward"):
        assert torch.equal(got[k], ref[k]), k


def test_noise_changes_only_what_the_policy_sees():
    """a policy that ignores the state (W = 0) makes the noise irrelevant; one that reads it changes the trajectory"""
    P = _problem("linear", Ds=3)
    H = 3
    zero = [torch.zeros_like(P["prm"][0]), P["prm"][1]]
    a, b_ = _run(P, H, v=P["v"], prm=zero), _run(P, H, v=np.zeros(3), prm=zero)
    assert torch.allclose(a["traj_S"], b_["traj_S"], rtol=0, atol=1e-15)
    c = _run(P, H)
    assert float((c["traj_S"][1:] - _run(P, H, v=np.zeros(3))["traj_S"][1:]).abs().max()) > 1e-6


def test_exact_case_matches_monte_carlo():
    """H = 1, a linear unsquashed policy, no angles: [x, W (x + nu) + b] is exactly Gaussian, so moment matching gives
    the exact first two moments of x_1 = x + f(x, u) + sqrt(var f(x, u)) eps under the latent GP posterior"""
    P = _problem("linear", Ds=3, U=2, squash=False, seed=7)
    P["v"] = np.array([0.05, 0.02, 0.08])
    ref = _run(P, 1)
    iK, beta = tp.calculate_factorizations(T(P["X"]), T(P["Y"]), T(P["ell"]), T(P["sf2"]), T(P["sn2"]))
    dyn = dict(C=P["X"], ell=P["ell"], sf2=P["sf2"], iK=iK.numpy(), beta=beta.numpy())
    rng = np.random.RandomState(11)
    W, b = P["prm"][0].numpy(), P["prm"][1].numpy()
    N, chunks = 10 ** 6, []
    for _ in range(10):
        x = rng.multivariate_normal(P["m0"], P["S0"], size=N // 10)
        z = x + rng.randn(N // 10, 3) * np.sqrt(P["v"])
        u = z @ W.T + b
        mu, var = po.gp_latent(dyn, np.hstack([x, u]))
        chunks.append(x + mu + np.sqrt(np.maximum(var, 0.0)) * rng.randn(N // 10, 3))
    x1 = np.vstack(chunks)
    worst = po.moment_check(x1, ref["traj_m"][1].numpy(), ref["traj_S"][1].numpy())
    assert worst < 5.0, worst
    # without the noise term the covariance is measurably off: the test sees the noise
    bare = _run(P, 1, v=np.zeros(3))
    assert po.moment_check(x1, bare["traj_m"][1].numpy(), bare["traj_S"][1].numpy()) > 5.0


@pytest.mark.parametrize("kind,dims,b", [("linear", (), 0.0), ("rbf", (), 0.5), ("linear", (1,), -0.5), ("rbf", (1,), 0.0)])
def test_gradient_matches_central_differences(kind, dims, b):
    P = _problem(kind, Ds=3, dims=dims, seed=5)
    H = 3
    leaves = [p.clone().requires_grad_(True) for p in P["prm"]]
    m0 = T(P["m0"]).requires_grad_(True)
    S0 = T(P["S0"]).requires_grad_(True)
    out = _run(P, H, b=b, prm=leaves, m0=m0, S0=S0)
    grads = torch.autograd.grad(out["reward"], leaves + [m0, S0])
    rng = np.random.RandomState(3)
    args = [p.detach() for p in leaves] + [m0.detach(), S0.detach()]
    h = 1e-5
    for k, (a, g) in enumerate(zip(args, grads)):
        d = T(rng.randn(*a.shape))
        if k == len(args) - 1:
            d = 0.5 * (d + d.T)                         # S0 is symmetric
        vals = []
        for sgn in (1.0, -1.0):
            pert = list(args)
            pert[k] = a + sgn * h * d
            vals.append(float(_run(P, H, b=b, prm=pert[:-2], m0=pert[-2], S0=pert[-1])["reward"]))
        fd = (vals[0] - vals[1]) / (2 * h)
        ad = float((g * d).sum())
        assert abs(fd - ad) < 1e-7 * max(1.0, abs(ad)), (k, fd, ad)


# ---- the library -----------------------------------------------------------------------------------------------------
NEW = ("pilco_rollout_noisy_workspace_bytes", "pilco_rollout_noisy_bwd_workspace_bytes", "pilco_rollout_noisy_forward",
       "pilco_rollout_noisy_backward")
KERNELS = ("nz_state_kernel", "nz_trig_kernel")


def test_library_exports_the_entry_points():
    from pilco_b200 import _lib
    for name in NEW:
        assert hasattr(_lib.lib, name) and name in _lib.SIGNATURES
    header = open(os.path.join(ROOT, "include", "pilco_b200.h")).read()
    assert all(name + "(" in header for name in NEW)


def test_obs_noise_layout(tmp_path):
    from pilco_b200 import _lib
    src = tmp_path / "nz_layout.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "%s"\nint main(void) { printf("%%zu %%zu\\n", '
                   'sizeof(pilco_obs_noise), offsetof(pilco_obs_noise, var)); return 0; }\n'
                   % os.path.join(ROOT, "include", "pilco_b200.h"))
    exe = str(tmp_path / "nz_layout")
    subprocess.check_call(["gcc", "-o", exe, str(src)])
    size, ov = map(int, subprocess.check_output([exe], text=True).split())
    assert (ctypes.sizeof(_lib.ObsNoise), _lib.ObsNoise.var.offset) == (size, ov) == (16 * 8, 0)


def test_new_kernels_do_not_spill():
    """no spills; the only local memory is the 40-byte frame of the double-precision sin/cos argument reduction that
    the angle cascade's tg_state / tg_trig carry as well (the same STL/LDL count)"""
    nvcc = "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not installed")
    res = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas", "-v",
                          "-cubin", "-o", os.devnull, os.path.join(ROOT, "pilco_b200", "csrc", "rollout_noise.cu")],
                         capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    props = dict(re.findall(r"Function properties for (\S+)\n\s*(.*)", res.stderr))
    for k in KERNELS:
        name = next(n for n in props if k in n)
        assert "40 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads" in props[name], (name, props[name])
    if os.path.exists(CUOBJDUMP):
        text = sass("|".join(KERNELS + ("tg_state_kernel", "tg_trig_kernel")))
        count = {n: (len(re.findall(r"\bSTL\b", t)), len(re.findall(r"\bLDL\b", t))) for n, t in text.items()}
        ref = {v for n, v in count.items() if "tg_" in n}
        assert len(ref) == 1 and all(v in ref for n, v in count.items() if "nz_" in n), count


def _nz(var):
    from pilco_b200 import _lib
    nz = _lib.ObsNoise()
    nz.var[:len(var)] = list(var)
    return nz


def test_validation_before_device_work():
    """Every rejected call returns before it enqueues anything (the fake pointers are never dereferenced); nz == NULL
    is the exploration call"""
    from pilco_b200 import _lib
    lib, C = _lib.lib, ctypes
    g = _lib.RolloutGrad()
    fwd = lambda ro, nz, ex=None: lib.pilco_rollout_noisy_forward(C.byref(ro), None, ex, nz and C.byref(nz), None)
    bwd = lambda ro, nz, ex=None: lib.pilco_rollout_noisy_backward(C.byref(ro), None, ex, nz and C.byref(nz),
                                                                    C.byref(g), None)
    ro = _rollout()
    ok = _nz([0.1, 0.0, 0.2])
    need = lib.pilco_rollout_noisy_workspace_bytes(C.byref(ro), None, None, C.byref(ok))
    base = lib.pilco_rollout_workspace_bytes(C.byref(ro))
    assert need > base
    ex = _lib.Exploration(0.5, None)
    need_ex = lib.pilco_rollout_noisy_workspace_bytes(C.byref(ro), None, C.byref(ex), C.byref(ok))
    assert need_ex == need + 8 * (ro.R * ro.H + (ro.R * ro.H) % 2)
    for call in (fwd, bwd):
        for bad in ([float("nan"), 0, 0], [0, -1e-300, 0], [0, 0, float("inf")]):
            ro.ws_bytes = need
            assert call(ro, _nz(bad)) == ERR_DIM
        ro.ws_bytes = 0
        assert call(ro, _nz([0, 0, 0, -1.0])) == ERR_WS                  # entries from Ds on are not read
        assert call(ro, ok) == ERR_WS
        ro.ws_bytes = base
        assert call(ro, ok) == ERR_WS                                     # enough for the call without noise only
        ro.ws_bytes = need
        assert call(ro, ok, C.byref(ex)) == ERR_WS                        # the exploration slot comes after
        assert call(ro, ok, C.byref(_lib.Exploration(float("nan"), None))) == ERR_DIM
        box = _rollout(reward_kind=_lib.REWARD_BOX)
        box.ws_bytes = need_ex
        assert call(box, ok, C.byref(ex)) == ERR_UNSUP                    # the explore call's codes
        nul = _rollout()
        nul.m0 = None
        assert call(nul, ok) == ERR_NULL
        ro.ws_bytes = 0
    # nz == NULL: the exploration call (its status and workspace sizes)
    assert fwd(ro, None) == ERR_WS
    assert fwd(_rollout(), None, C.byref(ex)) == ERR_WS
    for e in (None, C.byref(ex)):
        assert (lib.pilco_rollout_noisy_workspace_bytes(C.byref(ro), None, e, None)
                == lib.pilco_rollout_explore_workspace_bytes(C.byref(ro), None, e))
        assert (lib.pilco_rollout_noisy_bwd_workspace_bytes(C.byref(ro), None, e, None)
                == lib.pilco_rollout_explore_bwd_workspace_bytes(C.byref(ro), None, e))
    assert (lib.pilco_rollout_noisy_bwd_workspace_bytes(C.byref(ro), None, None, C.byref(ok))
            > lib.pilco_rollout_bwd_workspace_bytes(C.byref(ro)))


def test_python_validation():
    from pilco_b200 import engine, _lib
    terms = [dict(kind=_lib.REWARD_EXP, coef=1.0, W=np.eye(3), t=np.zeros(3))]
    for bad in ([0.1, -0.1, 0.1], [0.1, float("nan"), 0.1], [float("inf")] * 3):
        with pytest.raises(ValueError, match="measurement_noise"):
            engine.RolloutPlan(None, dict(Ds=3, U=1), terms, np.zeros(3), np.eye(3), 5, measurement_noise=bad)
