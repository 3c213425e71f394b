"""CPU tests of the angular-state-dimension stage: the closed forms of pilco_b200/csrc/trig_math.cuh compiled for the
host (against Monte Carlo, the torch statement in tests/angles_oracle.py and torch autograd), the pilco_angles layout,
validation before any device work, and the new kernels' registers."""
import ctypes
import os
import subprocess

import numpy as np
import pytest
import torch

from abi_fakes import ERR_DIM, ERR_NULL, FAKE, _rollout
import angles_oracle as ao
from util import ROOT, TRIG_CASES, host_moments, host_vjp, trig_harness


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    return trig_harness(str(tmp_path_factory.mktemp("trig") / "trig_harness.so"))


@pytest.mark.parametrize("name,m,s,dims", TRIG_CASES, ids=[c[0] + "_%d" % i for i, c in enumerate(TRIG_CASES)])
def test_trig_moments_match_monte_carlo(harness, name, m, s, dims):
    M, S, C = host_moments(harness, m, s, dims)
    rng = np.random.RandomState(11)
    N = 1_000_000
    w, V = np.linalg.eigh(s)
    x = m + (rng.randn(N, len(m)) * np.sqrt(np.clip(w, 0, None))) @ V.T
    from pilco_b200.engine import trig_feature_map
    f = trig_feature_map(x, dims)
    fm = f.mean(0)
    se_m = f.std(0) / np.sqrt(N) + 1e-300
    assert np.all(np.abs(M - fm) <= 5 * se_m + 1e-9), name
    fc = f - fm
    prod = fc[:, :, None] * fc[:, None, :]
    Smc = prod.mean(0)
    se_S = prod.std(0) / np.sqrt(N) + 1e-300
    assert np.all(np.abs(S - Smc) <= 5 * se_S + 1e-9), name
    # s C = cov(x, phi)
    xc = x - x.mean(0)
    cross = xc[:, :, None] * fc[:, None, :]
    se_C = cross.std(0) / np.sqrt(N) + 1e-300
    assert np.all(np.abs(s @ C - cross.mean(0)) <= 5 * se_C + 1e-9), name


@pytest.mark.parametrize("name,m,s,dims", TRIG_CASES, ids=[c[0] + "_%d" % i for i, c in enumerate(TRIG_CASES)])
def test_trig_moments_match_torch_oracle(harness, name, m, s, dims):
    M, S, C = host_moments(harness, m, s, dims)
    Mt, St, Ct = ao.trig_moments(torch.tensor(m), torch.tensor(s), dims)
    assert np.max(np.abs(M - Mt.numpy())) < 1e-14
    assert np.max(np.abs(S - St.numpy())) < 1e-14
    assert np.max(np.abs(C - Ct.numpy())) < 1e-14


@pytest.mark.parametrize("name,m,s,dims", TRIG_CASES, ids=[c[0] + "_%d" % i for i, c in enumerate(TRIG_CASES)])
def test_trig_vjp_matches_autograd(harness, name, m, s, dims):
    Ds, Dh = len(m), len(m) + len(dims)
    rng = np.random.RandomState(3)
    gM, gS, gC = rng.randn(Dh), rng.randn(Dh, Dh), rng.randn(Ds, Dh)
    gm, gs = host_vjp(harness, m, s, dims, gM, gS, gC)
    mt = torch.tensor(m, requires_grad=True)
    st = torch.tensor(s, requires_grad=True)
    Mt, St, Ct = ao.trig_moments(mt, st, dims)
    L = (Mt * torch.tensor(gM)).sum() + (St * torch.tensor(gS)).sum() + (Ct * torch.tensor(gC)).sum()
    rm, rs = torch.autograd.grad(L, (mt, st))
    rs = 0.5 * (rs + rs.T).numpy()
    scale = max(1.0, np.max(np.abs(rs)), np.max(np.abs(rm.numpy())))
    assert np.max(np.abs(gm - rm.numpy())) < 1e-12 * scale
    assert np.max(np.abs(gs - rs)) < 1e-12 * scale
    assert np.array_equal(gs, gs.T)


def test_no_angles_is_identity(harness):
    rng = np.random.RandomState(1)
    m, B = rng.randn(4), rng.randn(4, 4)
    s = B @ B.T
    M, S, C = host_moments(harness, m, s, [])
    assert np.array_equal(M, m) and np.array_equal(S, s) and np.array_equal(C, np.eye(4))


def test_angles_struct_layout(harness):
    from pilco_b200 import _lib
    out = (ctypes.c_size_t * 3)()
    harness.angles_layout(out)
    assert ctypes.sizeof(_lib.Angles) == out[0]
    assert _lib.Angles.A.offset == out[1] and _lib.Angles.dims.offset == out[2]


def _angles(*dims):
    from pilco_b200 import _lib
    a = _lib.Angles()
    a.A = len(dims)
    for i, d in enumerate(dims):
        a.dims[i] = d
    return a


def _angle_rollout(Ds=3, A=1, U=1):
    ro = _rollout()
    ro.dyn.E, ro.dyn.D = Ds, Ds + A + U
    ro.pol.Ds, ro.pol.U = Ds + A, U
    return ro


def test_validation_before_device_work():
    """Every rejected call returns before it enqueues anything (the fake pointers are never dereferenced)."""
    from pilco_b200 import _lib
    lib = _lib.lib
    C = ctypes
    ro = _angle_rollout()
    fwd = lambda ro, a: lib.pilco_rollout_angles_forward(C.byref(ro), C.byref(a), None)
    g = _lib.RolloutGrad()
    bwd = lambda ro, a: lib.pilco_rollout_angles_backward(C.byref(ro), C.byref(a), C.byref(g), None)
    for call in (fwd, bwd):
        assert call(ro, _angles(3)) == ERR_DIM                      # out of range
        assert call(ro, _angles(-1)) == ERR_DIM
        assert call(_angle_rollout(A=2), _angles(1, 1)) == ERR_DIM  # repeated
        assert call(_angle_rollout(Ds=2, A=3), _angles(0, 1, 1)) == ERR_DIM
        big = _angle_rollout(Ds=8, A=4, U=5)                        # Dh + U = 17
        assert call(big, _angles(0, 1, 2, 3)) == ERR_DIM
        wrong = _angle_rollout()
        wrong.pol.Ds = 3                                            # the policy must take Dh = 4 inputs
        assert call(wrong, _angles(0)) == ERR_DIM
        nul = _angle_rollout()
        nul.m0 = None
        assert call(nul, _angles(0)) == ERR_NULL                    # the codes of the call without angles
    assert lib.pilco_trig_moments(3, 1, C.byref(_angles(3)), FAKE, FAKE, FAKE, FAKE, FAKE, None) == ERR_DIM
    assert lib.pilco_trig_moments(3, 0, C.byref(_angles(0)), FAKE, FAKE, FAKE, FAKE, FAKE, None) == ERR_DIM
    assert lib.pilco_trig_moments(3, 1, None, None, FAKE, FAKE, FAKE, FAKE, None) == ERR_NULL
    # without angles the workspace queries are those of the calls without angles
    plain = _rollout()
    assert (lib.pilco_rollout_angles_workspace_bytes(C.byref(plain), None)
            == lib.pilco_rollout_workspace_bytes(C.byref(plain)))
    assert (lib.pilco_rollout_angles_bwd_workspace_bytes(C.byref(plain), C.byref(_angles()))
            == lib.pilco_rollout_bwd_workspace_bytes(C.byref(plain)))


def test_python_validation():
    from pilco_b200 import engine
    with pytest.raises(ValueError, match="distinct"):
        engine.angles_struct([0, 0], 3)
    with pytest.raises(ValueError, match="distinct"):
        engine.angles_struct([3], 3)
    assert engine.angles_struct([], 3) is None
    x = np.array([[0.1, 0.2, 0.3]])
    np.testing.assert_array_equal(engine.trig_feature_map(x, [1]),
                                  [[0.1, 0.3, np.sin(0.2), np.cos(0.2)]])


def test_new_kernels_do_not_spill():
    """ptxas of the angle kernels: no spill stores or loads; the stack frame is at most the double-precision sin/cos
    argument reduction's, which the existing squash stage (ro_state_kernel) carries too."""
    import re
    nvcc = "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not installed")
    out = {}
    for src in ("rollout.cu", "rollout_angles_bwd.cu", "closed_forms.cu"):
        res = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas", "-v",
                              "-cubin", "-o", os.devnull, os.path.join(ROOT, "pilco_b200", "csrc", src)],
                             capture_output=True, text=True)
        assert res.returncode == 0, res.stderr
        for name, props in re.findall(r"Function properties for (\S+)\n\s*(.*)", res.stderr):
            out[name] = props
    tg = {k: v for k, v in out.items() if re.match(r"_Z\d+tg_", k)}
    assert len(tg) >= 8, sorted(tg)
    ref = int(re.search(r"(\d+) bytes stack", out["_Z15ro_state_kernel5RoDev"]).group(1))
    for name, props in tg.items():
        assert "0 bytes spill stores, 0 bytes spill loads" in props, (name, props)
        assert int(re.search(r"(\d+) bytes stack", props).group(1)) <= ref, (name, props)


def _pendulum_data(T=30, seed=0):
    rng = np.random.RandomState(seed)
    X = np.hstack([rng.randn(T, 2), rng.uniform(-2, 2, (T, 1))])
    Y = 0.1 * rng.randn(T, 2)
    return X, Y


def test_pilco_angle_dims_construction_and_data():
    """PILCO(angle_dims=...): the models are built on [phi(x), u]; PILCO.set_data applies phi; the models' own set_data
    rejects raw data; width checks of the controller and the joint reward terms; particle methods refuse angles --
    all before any device work"""
    from pilco.models import PILCO
    from pilco.controllers import RbfController, LinearController
    from pilco.rewards import ExponentialStateActionReward
    X, Y = _pendulum_data()
    p = PILCO((X, Y), controller=RbfController(3, 1, 5), horizon=10, angle_dims=[0])
    assert p.state_dim == 2 and p.policy_input_dim == 3
    assert p.mgpr.models[0].data[0].shape == (30, 4)
    np.testing.assert_array_equal(p.mgpr.models[0].data[0][:, 1], np.sin(X[:, 0]))
    np.testing.assert_array_equal(p.mgpr.models[0].data[0][:, 2], np.cos(X[:, 0]))
    np.testing.assert_array_equal(p.m_init, X[0:1, :2])
    X2, Y2 = _pendulum_data(T=40, seed=1)
    p.set_data((X2, Y2))
    assert p.mgpr.models[1].data[0].shape == (40, 4)
    with pytest.raises(ValueError, match="PILCO.set_data"):
        p.mgpr.set_data((X2, Y2))
    assert isinstance(PILCO((X, Y), angle_dims=[1]).controller, LinearController)
    assert np.asarray(PILCO((X, Y), angle_dims=[1]).controller.W).shape == (1, 3)
    with pytest.raises(ValueError, match="Dh = 3"):
        PILCO((X, Y), controller=RbfController(2, 1, 5), angle_dims=[0])
    with pytest.raises(ValueError, match="Dh = 3"):
        PILCO((X, Y), controller=RbfController(3, 1, 5), reward=ExponentialStateActionReward(2, 1), angle_dims=[0])
    PILCO((X, Y), controller=RbfController(3, 1, 5), reward=ExponentialStateActionReward(3, 1), angle_dims=[0])
    with pytest.raises(ValueError, match="distinct"):
        PILCO((X, Y), angle_dims=[2])
    for call in (lambda: p.sample_trajectories(p.m_init, p.S_init, 5),
                 lambda: p.sample_policy_gradient(p.m_init, p.S_init, 5),
                 lambda: p.optimize_policy_sampled()):
        with pytest.raises(ValueError, match="angle_dims"):
            call()
    # without angles nothing changes
    q = PILCO((X, Y))
    assert q.angle_dims is None and q.mgpr.models[0].data[0].shape == (30, 3)
    q.mgpr.set_data((X2, Y2))
