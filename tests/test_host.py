"""CPU tests of the host-side logic: C-ABI symbols, parameter objects, GP training driver, the lock-step
optimiser, restart sharding / winner selection, the oct2py/gpflow stand-ins, and the loud failure of the
product path without a GPU."""
import ctypes
import os
import re

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_abi_exports_every_declared_symbol():
    hdr = open(os.path.join(ROOT, "include", "pilco_b200.h")).read()
    hdr = re.sub(r"/\*.*?\*/", "", hdr, flags=re.S)
    declared = set(re.findall(r"\b(pilco_[a-z0-9_]+)\s*\(", hdr))
    assert len(declared) >= 18
    lib = ctypes.CDLL(os.path.join(ROOT, "pilco_b200", "libpilco_b200.so"))
    for name in sorted(declared):
        assert hasattr(lib, name), "libpilco_b200.so does not export %s" % name
    from pilco_b200 import _lib
    assert declared == set(_lib.SIGNATURES), "ctypes signature table out of sync with the header"
    assert _lib.lib.pilco_version() == _lib.ABI_VERSION == 3
    assert _lib.lib.pilco_pad_n(300) == 320 and _lib.lib.pilco_pad_n(64) == 64
    assert _lib.lib.pilco_mm_workspace_bytes(300, 12, 10, 2) > 0
    assert _lib.lib.pilco_mm_workspace_bytes(300, 17, 10, 2) == 0          # D > PILCO_MAX_D rejected
    assert b"workspace" in _lib.lib.pilco_status_string(-3)


def test_struct_layouts_match_header_sizes(tmp_path):
    """Compile include/pilco_b200.h with the C compiler and compare every struct's size and field offsets with
    the ctypes mirrors the Python host side passes through the ABI."""
    import subprocess
    from pilco_b200 import _lib
    exe = str(tmp_path / "abi_layout")
    subprocess.check_call(["gcc", "-o", exe, os.path.join(ROOT, "tests", "host_harness", "abi_layout.c")])
    mirror = {"pilco_gp_model": _lib.GpModel, "pilco_policy": _lib.Policy, "pilco_reward_term": _lib.RewardTerm,
              "pilco_rollout": _lib.Rollout, "pilco_rollout_grad": _lib.RolloutGrad}
    nchecked = 0
    for line in subprocess.check_output([exe], text=True).splitlines():
        parts = line.split()
        kind, what, val = parts[0], parts[1] if len(parts) == 3 else "", parts[-1]
        if kind == "sizeof":
            assert ctypes.sizeof(mirror[what]) == int(val), what
        elif kind == "offsetof":
            st, field = what.split(".")
            assert getattr(mirror[st], field).offset == int(val), what
        else:
            assert int(val) == _lib.ABI_VERSION
        nchecked += 1
    assert nchecked >= 40
    assert ctypes.sizeof(_lib.GpModel) == 4 * 4 + 4 * 16 + 16          # ints, 4x(ptr,stride), iK+ldk(+pad)
    assert ctypes.sizeof(_lib.RewardTerm) == 32


def test_box_risk_formulas_on_host(tmp_path):
    """pilco_b200/csrc/risk_math.cuh (the code the device executes for the safe-PILCO risk rewards) compiled
    for the host: value against the numpy restatement of rewards_safe.py, derivatives against torch autograd."""
    import subprocess
    from oracle import safe_port as sp
    so = str(tmp_path / "risk_harness.so")
    subprocess.check_call(["g++", "-O1", "-shared", "-fPIC", "-x", "c++", "-o", so,
                           os.path.join(ROOT, "tests", "host_harness", "risk_harness.cpp")])
    lib = ctypes.CDLL(so)
    dp = ctypes.POINTER(ctypes.c_double)
    lib.risk_box_eval_host.restype = ctypes.c_double
    lib.risk_box_eval_host.argtypes = [ctypes.c_int, dp, dp, dp, dp, dp]
    rng = np.random.RandomState(0)
    Ds = 4
    inf = float("inf")
    cases = [((0, 2), (-0.3, -1.0), (0.4, 0.2), 2.0, True),         # RiskOfCollision
             ((1,), (-0.2,), (inf,), 1.0, True),                      # SingleConstraint, low only
             ((3,), (-inf,), (0.7,), 1.0, True),                      # high only
             ((2,), (-0.5,), (0.6,), 1.0, False)]                     # both, complement
    for dims, lows, highs, sfac, inside in cases:
        m = rng.randn(1, Ds) * 0.3
        a = rng.rand(Ds, Ds); s = 0.3 * a @ a.T + 0.2 * np.eye(Ds)
        prm = np.array([len(dims), float(inside), sfac] + [v for k in range(len(dims)) for v in (dims[k], lows[k], highs[k])])
        dm, dv = np.zeros(16), np.zeros(16)
        c = lambda x: np.ascontiguousarray(x, dtype=np.float64).ctypes.data_as(dp)
        val = lib.risk_box_eval_host(Ds, c(prm), c(m), c(s), dm.ctypes.data_as(dp), dv.ctypes.data_as(dp))
        if len(dims) == 2:
            ref = sp.risk_of_collision(m, s, lows, highs)[0]
        else:
            ref = sp.single_constraint(m, s, dims[0], high=None if highs[0] == inf else highs[0],
                                       low=None if lows[0] == -inf else lows[0], inside=inside)[0]
        assert abs(val - ref) < 1e-14
        mt = torch.tensor(m, requires_grad=True); st = torch.tensor(s, requires_grad=True)
        rt = sp.box_risk_torch(mt, st, dims, lows, highs, sfac, inside)
        assert abs(float(rt.detach()) - val) < 1e-14
        gm, gs = torch.autograd.grad(rt, [mt, st])
        for k, d in enumerate(dims):
            assert abs(dm[k] - float(gm[0, d])) < 1e-12 and abs(dv[k] - float(gs[d, d])) < 1e-12


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the no-GPU failure mode")
def test_product_path_fails_loudly_without_gpu():
    from pilco.models import MGPR
    X = np.random.rand(20, 2); Y = np.random.rand(20, 1)
    m = MGPR((X, Y))
    with pytest.raises(RuntimeError, match="CUDA device"):
        m.predict_on_noisy_inputs(np.zeros((1, 2)), np.eye(2))


def test_parameter_surface():
    from pilco_b200.params import Parameter, Softplus, set_trainable
    p = Parameter(np.ones(3), transform=Softplus(1e-3))
    assert p.shape == (3,) and np.allclose(p.numpy(), 1.0)
    th = p.unconstrained
    assert np.allclose(1e-3 + np.logaddexp(0, th), 1.0)
    p.assign([1.0, 2.0, 3.0])
    assert np.allclose(np.stack([p, p]), [[1, 2, 3], [1, 2, 3]])
    assert np.allclose(p.value() * 2, [2, 4, 6]) and np.allclose(2 * p, [2, 4, 6])
    set_trainable(p, False)
    assert not p.trainable
    q = Parameter(0.5)
    assert isinstance(q.numpy(), float) and q.shape == ()


def test_gp_training_reduces_loss_and_restarts_keep_best():
    """host training driver (the SMGPR / FITC path and the reference for the device NLML kernel)"""
    from pilco.models import MGPR
    np.random.seed(0)
    X = np.random.rand(40, 2)
    Y = np.sin(3 * X).dot(np.random.rand(2, 1)) + 1e-2 * np.random.randn(40, 1)
    m = MGPR((X, Y))
    l0 = m.models[0].training_loss()
    m.optimize_host(restarts=1)
    l1 = m.models[0].training_loss()
    assert l1 < l0 and np.all(m.lengthscales > 0) and np.all(m.noise >= 1e-6)
    m.models[0].likelihood.variance.assign(0.01)
    from gpflow import set_trainable
    set_trainable(m.models[0].likelihood.variance, False)
    m.optimize_host(restarts=0)
    assert abs(m.noise[0] - 0.01) < 1e-12


def test_smgpr_and_controller_host_surface():
    from pilco.models import SMGPR
    from pilco.controllers import RbfController, LinearController
    np.random.seed(0)
    X = np.random.rand(30, 3); Y = np.random.rand(30, 2)
    s = SMGPR((X, Y), num_induced_points=7)
    assert s.Z.numpy().shape == (7, 3) and s.centres.shape == (7, 3)
    s.optimize_host(restarts=0, maxiter=5)                             # host cross-check path (SMGPR.optimize itself runs on the device)
    assert np.all(s.lengthscales > 0)
    rbf = RbfController(3, 2, 11, max_action=2.0)
    assert rbf.models[1].X is rbf.models[0].X                          # shared centres (controllers.py:103-106)
    assert not rbf.models[0].kernel.variance.trainable and not rbf.models[0].likelihood.variance.trainable
    flat = rbf.get_flat()
    assert flat.shape == (11 * 3 + 11 * 2 + 2 * 3,)
    rbf.randomize()
    rbf.set_flat(flat)
    assert np.allclose(rbf.get_flat(), flat)
    rbf.set_data((np.random.rand(11, 3), np.random.rand(11, 2)))
    assert rbf.X.shape == (11, 3) and rbf.Y.shape == (11, 2)
    lin = LinearController(3, 2)
    f = lin.get_flat(); lin.randomize(); lin.set_flat(f)
    assert np.allclose(lin.get_flat(), f)


def test_lockstep_lbfgs_batches_evaluations():
    from pilco_b200.policy_opt import LockstepLBFGS
    A = np.array([1.0, 3.0, 10.0, 0.5])
    c = np.array([[1, 2], [3, -1], [0.5, 0.5], [-2, 4]], dtype=float)
    batches = []

    def ev(x):
        batches.append(x.copy())
        return (A[:, None] * (x - c) ** 2).sum(1), 2 * A[:, None] * (x - c)
    fin = LockstepLBFGS(ev, np.zeros((4, 2)), 50).run()
    for (f, x), ci in zip(fin, c):
        assert f < 1e-12 and np.allclose(x, ci, atol=1e-6)
    assert len(batches) < 12            # evaluations are shared: ~max over restarts, not the sum


def test_lockstep_isolates_nonfinite_restart():
    from pilco_b200.policy_opt import LockstepLBFGS, BIG

    def ev(x):
        f = (x ** 2).sum(1); g = 2 * x
        f[1] = BIG; g[1] = 0.0          # restart 1 always fails (what the evaluator reports for info != 0)
        return f, g
    fin = LockstepLBFGS(ev, np.ones((3, 2)), 20).run()
    assert fin[0][0] < 1e-12 and fin[2][0] < 1e-12 and fin[1][0] == BIG


def test_shard_and_select():
    from pilco_b200.policy_opt import shard_restarts, select_best
    assert shard_restarts(10, 0, 4) == [0, 4, 8] and shard_restarts(10, 3, 4) == [3, 7]
    assert sorted(sum((shard_restarts(7, r, 3) for r in range(3)), [])) == list(range(7))
    t = np.array([[2.0, 0], [1.0, 0], [1.0, 1], [np.nan, 0]])
    assert select_best(t) == 1          # ties -> lowest restart index (pilco.py:105 uses a strict >)


def test_oct2py_stand_in_conventions():
    import oct2py
    oc = oct2py.Oct2Py()
    oc.addpath("whatever")
    s = oct2py.io.Struct(); s.hyp = 1; s.p = oct2py.io.Struct(); s.p.w = 2
    assert s["hyp"] == 1 and s.p.w == 2
    M, S, C = oc.gSin(np.array([[0.1], [0.2]]), 0.1 * np.eye(2), 7.0, nout=3)
    assert M.shape == (2, 1) and S.shape == (2, 2) and C.shape == (2, 2)
    out = oc.reward(np.zeros((2, 1)), np.eye(2), np.zeros((2, 1)), np.eye(2), nout=4)
    assert len(out) == 4 and isinstance(out[0], float)
    from gpflow import config
    assert config.default_float() is np.float64


def test_safe_extension_host_surface():
    """Host logic of the safe-PILCO drop-ins (no device work): the parameter block handed to the box-risk kernel,
    the reference's truthiness handling of missing bounds (rewards_safe.py:44-52), reward-term lowering of
    ObjectiveFunction / SafePILCO (channels, coefficients) and the import paths of the reference package."""
    from safe_pilco_extension.rewards_safe import RiskOfCollision, SingleConstraint, ObjectiveFunction
    from safe_pilco_extension.safe_pilco import SafePILCO
    from pilco.rewards import ExponentialReward, LinearReward, CombinedRewards
    from pilco.controllers import LinearController
    from pilco_b200 import _lib
    inf = float("inf")
    r = RiskOfCollision(4, [-1.0, -2.0], [1.5, 2.5])
    assert np.array_equal(r.prm(), [2, 1, 2.0, 0, -1.0, 1.5, 2, -2.0, 2.5])          # dims 0 and 2, scale 2*diag(s)
    assert np.array_equal(SingleConstraint(3, low=0.2).prm(), [1, 1, 1.0, 3, 0.2, inf])
    assert np.array_equal(SingleConstraint(1, high=0.7, inside=False).prm(), [1, 0, 1.0, 1, -inf, 0.7])
    assert np.array_equal(SingleConstraint(1, high=0.7, low=0.0).prm(), [1, 1, 1.0, 1, -inf, 0.7])   # low=0.0 is falsy upstream
    with pytest.raises(Exception):
        SingleConstraint(0)
    obj = ObjectiveFunction(ExponentialReward(4), r, mu=2.0)
    t = obj.terms(coef=0.5)
    assert [x["kind"] for x in t] == [_lib.REWARD_EXP, _lib.REWARD_BOX] and [x["coef"] for x in t] == [0.5, -1.0]
    assert all(x["channel"] == _lib.CHANNEL_ADD for x in t)
    X = np.random.rand(30, 5); Y = np.random.rand(30, 4)
    comb = CombinedRewards(4, [LinearReward(4, np.ones(4)), ExponentialReward(4)], coefs=[2.0, 3.0])
    sp = SafePILCO((X, Y), controller=LinearController(4, 1), reward_add=comb, reward_mult=r, mu=-7.0, horizon=5)
    terms, mu = sp.reward_spec()
    assert mu == -7.0 and [x["channel"] for x in terms] == [0, 0, 1] and [x["coef"] for x in terms] == [2.0, 3.0, 1.0]
    sp.mu.assign(0.75 * sp.mu.numpy())
    assert sp.reward_spec()[1] == -5.25
    with pytest.raises(Exception):
        SafePILCO((X, Y), reward_add=comb)                                      # reward_mult is mandatory (safe_pilco.py:23-24)
    from pilco.models import PILCO
    assert PILCO((X, Y)).reward_spec()[1] == 0.0


def test_plain_c_caller_links_and_runs(tmp_path):
    """The boundary is a C ABI: a C99 translation unit including only include/pilco_b200.h must compile, link against
    libpilco_b200.so and run its GPU-free calls (tests/host_harness/c_caller.c)."""
    import subprocess
    exe = str(tmp_path / "c_caller")
    libdir = os.path.join(ROOT, "pilco_b200")
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Werror", "-o", exe, os.path.join(ROOT, "tests", "host_harness", "c_caller.c"),
                           "-L" + libdir, "-l:libpilco_b200.so", "-Wl,-rpath," + libdir])
    env = dict(os.environ)
    env["LD_LIBRARY_PATH"] = "/usr/local/cuda/lib64:" + env.get("LD_LIBRARY_PATH", "")
    out = subprocess.run([exe], capture_output=True, text=True, env=env, timeout=120)
    assert out.returncode == 0, (out.returncode, out.stdout, out.stderr)
    assert out.stdout.startswith("abi 3 mm_ws ") and "workspace" in out.stdout


@pytest.mark.parametrize("variant", ["table1024", "table256x16"])
def test_table_exp_on_host(tmp_path, variant):
    """pilco_b200/csrc/exp_table.cuh (the table exp of the tile kernels, shared source) compiled for the host, in both
    table layouts (1024 entries + cubic remainder: 7 fp64 instructions; 256 entries x 16 bank-interleaved copies +
    quartic remainder: 8): accuracy against libm over the range a log-kernel value can take, the row-offset form used
    by the tile rows, and the clamp that turns padding (NEG_PAD) and far-apart centres into ~1e-304 instead of garbage."""
    import subprocess
    so = str(tmp_path / "exp_harness.so")
    flags = ["-DPILCO_EXP256"] if variant == "table256x16" else []
    subprocess.check_call(["g++", "-O2", "-ffp-contract=off", "-shared", "-fPIC", "-x", "c++"] + flags + ["-o", so,
                           os.path.join(ROOT, "tests", "host_harness", "exp_harness.cpp")])
    lib = ctypes.CDLL(so)
    dp = ctypes.POINTER(ctypes.c_double)
    c = lambda a: a.ctypes.data_as(dp)
    lib.exp_harness_scale.restype = ctypes.c_double
    SC = lib.exp_harness_scale()
    NT, STR = lib.exp_harness_entries(), lib.exp_harness_stride()
    assert (NT, STR) == ((256, 16) if variant == "table256x16" else (1024, 1))
    assert abs(SC - NT / np.log(2.0)) < 1e-9
    tab = np.zeros(NT * STR)
    lib.exp_harness_table(c(tab))
    assert tab[0] == 1.0 and abs(tab[(NT // 2) * STR] - np.sqrt(2.0)) < 3e-16
    rng = np.random.RandomState(0)
    LD = np.longdouble                                          # x87 extended precision: reference for 2^(xs/NT)
    ref_of = lambda xs: np.exp2(LD(xs) / LD(float(NT)))
    xs = np.concatenate([rng.uniform(-690.0, 1.0, 200000), rng.uniform(-1e-3, 1e-3, 1000), [0.0, -1.0, 1.0]]) * SC
    out = np.zeros_like(xs)
    lib.exp_harness_scaled(len(xs), c(xs), c(tab), c(out))
    rel = np.abs((LD(out) - ref_of(xs)) / ref_of(xs)).astype(np.float64)
    assert rel.max() < 4e-16, rel.max()                       # observed 3.5e-16 (1.6 ulp): table rounding + polynomial + final rounding
    # row-offset form: c = pre-scaled column part, A = pre-scaled row part (integer part folded into the magic constant)
    for A in (-123456.789, 0.25, 3210.5, -0.49999):
        cc = rng.uniform(-400.0, 10.0, 50000) * SC
        o2 = np.zeros_like(cc)
        rf = ctypes.c_double()
        lib.exp_harness_shifted(len(cc), c(cc), ctypes.c_double(A), c(tab), c(o2), ctypes.byref(rf))
        tot = LD(cc) + LD(A)                                    # exact pre-scaled exponent of the element
        keep = np.asarray(tot / LD(SC) > -690.0)
        ref2 = np.exp2(tot[keep] / LD(float(NT)))
        assert np.abs((LD(o2[keep]) - ref2) / ref2).astype(np.float64).max() < 7e-16      # + the row-factor product and its own rounding
        assert abs(rf.value - np.exp((A - np.rint(A)) / SC)) < 2.3e-16
    # clamp: padding (NEG_PAD = -1e9 pre-scaled) and extreme negatives give a tiny positive number, never NaN/inf/negative
    # (the 2^k field of exp_shifted is taken from 32 bits of the integer part: |pre-scaled exponent| < 2^(31+EXP_SHIFT),
    #  i.e. 2^41 / 2^39 -- log-kernel values of +-1.4e9 in either layout)
    bad = np.array([-1.0e9, -5.0e6, -1.1e6, -1.0e12 if NT == 1024 else -4.0e11])
    o3 = np.zeros_like(bad)
    rf = ctypes.c_double()
    lib.exp_harness_shifted(len(bad), c(bad), ctypes.c_double(0.0), c(tab), c(o3), ctypes.byref(rf))
    assert np.all(np.isfinite(o3)) and np.all(o3 >= 0.0) and np.all(o3 < 1e-300)
    lib.exp_harness_shifted(len(bad), c(np.zeros(4)), ctypes.c_double(-1.0e9), c(tab), c(o3), ctypes.byref(rf))   # padded ROW
    assert np.all(np.isfinite(o3)) and np.all(o3 >= 0.0) and np.all(o3 < 1e-300)
    xneg = np.array([-2000.0, -1e5]) * SC; o4 = np.zeros(2)
    lib.exp_harness_scaled(2, c(xneg), c(tab), c(o4))
    assert np.all(np.isfinite(o4)) and np.all(o4 >= 0.0) and np.all(o4 < 1e-300)


def test_workspace_layouts_on_host(tmp_path):
    """Workspace layouts (csrc/mm_kernels.cuh, mm_backward.cuh) compiled for the host: arrays are laid out in
    ascending, non-overlapping, 16-byte aligned order with the documented sizes, the per-restart stride matches what
    the shared library reports through pilco_mm_workspace_bytes / pilco_mm_bwd_workspace_bytes, and the pair
    indexing helpers invert each other."""
    import subprocess
    from pilco_b200 import _lib
    so = str(tmp_path / "layout_harness.so")
    subprocess.check_call(["g++", "-O1", "-shared", "-fPIC", "-x", "c++", "-I/usr/local/cuda/include", "-o", so,
                           os.path.join(ROOT, "tests", "host_harness", "layout_harness.cpp")])
    lib = ctypes.CDLL(so)
    lib.layout_bwd_per_r.restype = ctypes.c_ulonglong
    buf = (ctypes.c_ulonglong * 10)()
    for n, D, E in [(300, 12, 10), (37, 1, 1), (64, 4, 3), (600, 3, 2), (500, 10, 8), (200, 12, 10), (50, 10, 2), (65, 13, 2)]:
        for ordered in (0, 1):
            np_ = lib.layout_mm(n, D, E, ordered, buf)
            zeta, betap, Bq, Tpart, Wm, Wc, Qab, Ufrag, Arow, per_r = [int(v) for v in buf]
            assert np_ == (n + 63) // 64 * 64 == _lib.lib.pilco_pad_n(n)
            P = E * E if ordered else E * (E + 1) // 2
            ldz, ks = ctypes.c_int(), ctypes.c_int()
            lib.layout_misc(D, ctypes.byref(ldz), ctypes.byref(ks))
            assert ldz.value >= D and ldz.value % 4 == 0 and ks.value == (D + 3) // 4
            order = [zeta, betap, Bq, Tpart, Wm, Wc, Qab, Ufrag, Arow, per_r]
            assert order == sorted(order) and zeta == 0
            assert betap - zeta == np_ * ldz.value and Bq - betap == E * np_ and Tpart - Bq == P * np_
            assert Wm - Tpart >= P * (np_ // 8) and Wm % 2 == 0 and Ufrag % 2 == 0 and per_r % 2 == 0
            assert Qab - Wc >= E and Ufrag - Qab >= P * (2 * 16 * 16 + 2 * 16 + 8)
            if ordered:
                assert Ufrag == Arow == per_r or per_r - Arow <= 1                     # backward derives row operands in-kernel
            else:
                assert Arow - Ufrag == P * (np_ // 8) * ks.value * 32 and per_r - Arow >= P * np_
                for R in (1, 7):
                    assert _lib.lib.pilco_mm_workspace_bytes(n, D, E, R) == per_r * R * 8
        for need in (0, 1):
            assert _lib.lib.pilco_mm_bwd_workspace_bytes(n, D, E, 3, need) == lib.layout_bwd_per_r(n, D, E, need) * 3 * 8
    a, b = ctypes.c_int(), ctypes.c_int()
    seen = set()
    for q in range(136):                                                            # E = 16: 136 unordered pairs
        assert lib.layout_pair(q, ctypes.byref(a), ctypes.byref(b)) == q and 0 <= a.value <= b.value < 16
        seen.add((a.value, b.value))
    assert len(seen) == 136


def test_lockstep_group_bounds():
    """policy_opt deals a rank's restarts to lock-step groups of at least MIN_GROUP restarts (2 by default)."""
    from pilco_b200.policy_opt import group_bounds
    assert group_bounds(32) == [(0, 16), (16, 32)]
    assert group_bounds(20) == [(0, 10), (10, 20)]
    assert group_bounds(15) == [(0, 15)]
    assert group_bounds(1) == [(0, 1)]
    assert group_bounds(64, groups=4) == [(0, 16), (16, 32), (32, 48), (48, 64)]
    assert group_bounds(17, groups=4) == [(0, 8), (8, 17)]


def test_no_test_module_imports_another():
    """Shared fixtures live in particle_cases.py, abi_fakes.py and util.py, and the oracles in their own modules:
    importing a test module would run its top level and tie its private helpers to another file's tests"""
    tests = os.path.join(ROOT, "tests")
    pattern = re.compile(r"^\s*(import\s+test_\w*|from\s+test_\w*\s+import)\b", re.M)
    offenders = []
    for name in sorted(os.listdir(tests)):
        if name.endswith(".py"):
            src = open(os.path.join(tests, name)).read()
            offenders += ["%s: %s" % (name, m.group(0).strip()) for m in pattern.finditer(src)]
    assert not offenders, offenders
