"""Fake C-ABI descriptors for the tests that check argument validation without a GPU: the status codes of
include/pilco_b200.h and builders of pilco_gp_model, pilco_rollout, pilco_particles (plain and with per-restart
policies, with angles or measurement noise) and pilco_particles_grad whose pointers are fake non-null addresses, a
stand-in for a DeviceGP, the rejected calls of the batched score gradient, and the rows of the engine's particle entry
points called with the engine's own argument order.  Every entry point validates its arguments on the host before it
enqueues anything, so only calls that are rejected may be made with them."""
from pilco_b200 import _lib, engine

OK, ERR_NULL, ERR_DIM, ERR_WS, ERR_ALIGN, ERR_LAUNCH, ERR_UNSUP = 0, -1, -2, -3, -4, -5, -6
FAKE = 0x10000          # 16-byte aligned, never dereferenced by the validation code
PT_MAX_P = 65535 * 32   # the particle kernels' largest P (and R P)


def entry_call(key, query=False, **slots):
    """row ``key`` of engine.PARTICLE_ENTRY_POINTS with the arguments engine.particle_args binds to ``slots`` and a
    NULL stream -> its status; ``query``: its size query's result"""
    name = engine.PARTICLE_ENTRY_POINTS[key][1 if query else 0]
    args = engine.particle_args(name, **slots)
    return getattr(_lib.lib, name)(*args) if query else getattr(_lib.lib, name)(*args, None)


SAMPLER = {False: "step", True: "consistent", "resampled": "resampled"}     # the host tests' sampler keys


def _gp(n=50, D=4, E=3, mode=0, iK=FAKE, ldk=64, bs=0):
    g = _lib.GpModel()
    g.n, g.D, g.E, g.mode = n, D, E, mode
    g.X = g.ell = g.sf2 = g.beta = FAKE
    g.X_bs = bs
    g.iK, g.ldk = iK, ldk
    return g


def _rollout(kind=_lib.POLICY_LINEAR, n_rewards=1, reward_kind=_lib.REWARD_EXP, channel=0):
    ro = _lib.Rollout()
    ro.R, ro.H = 2, 5
    ro.dyn = _gp(n=50, D=4, E=3)
    ro.pol.kind, ro.pol.Ds, ro.pol.U, ro.pol.squash = kind, 3, 1, 1
    ro.pol.max_action = ro.pol.W = ro.pol.b = FAKE
    ro.n_rewards = n_rewards
    ro.rewards[0].kind, ro.rewards[0].channel, ro.rewards[0].coef = reward_kind, channel, 1.0
    ro.rewards[0].W = ro.rewards[0].t = FAKE
    ro.m0 = ro.S0 = ro.traj_m = ro.traj_S = ro.reward = ro.ws = FAKE
    ro.ws_bytes = 0
    return ro


def _particles(kind=_lib.POLICY_LINEAR, reward_kind=_lib.REWARD_EXP, channel=0, P=1000, H=5):
    pr = _lib.Particles()
    pr.P, pr.H = P, H
    pr.dyn = _gp()
    pr.pol.kind, pr.pol.Ds, pr.pol.U, pr.pol.squash = kind, 3, 1, 1
    pr.pol.max_action = pr.pol.W = pr.pol.b = FAKE
    if kind == _lib.POLICY_RBF:
        pr.pol.rbf = _gp(n=20, D=3, E=1, mode=1, iK=None, ldk=0)
    pr.n_rewards = 1
    pr.rewards[0].kind, pr.rewards[0].channel, pr.rewards[0].coef = reward_kind, channel, 1.0
    pr.rewards[0].W = pr.rewards[0].t = FAKE
    pr.x0 = pr.eps = pr.traj = pr.act = pr.step_reward = pr.step_risk = pr.ret = pr.ws = FAKE
    pr.ws_bytes = 0
    return pr


def _batched(kind=_lib.POLICY_LINEAR, **kw):
    """a valid description of R policies, each array with its own per-restart block"""
    pr = _particles(kind, **kw)
    if kind == _lib.POLICY_LINEAR:
        pr.pol.W_bs, pr.pol.b_bs = 3, 1
    else:
        r = pr.pol.rbf
        r.X_bs, r.ell_bs, r.sf2_bs, r.beta_bs = 20 * 3, 3, 1, 20
    return pr


def _grad():
    g = _lib.ParticlesGrad()
    g.gW = g.gb = g.gXc = g.gYc = g.gell = g.pol_L = g.value = g.ws = FAKE
    g.ws_bytes = 0
    return g


def _angles(*dims):
    a = _lib.Angles()
    a.A = len(dims)
    for i, d in enumerate(dims):
        a.dims[i] = d
    return a


def _angle_particles(kind=_lib.POLICY_LINEAR, A=1, batched=False, **kw):
    """_particles' description (E = 3 state dimensions, U = 1) with a policy of Dh = 3 + A inputs"""
    pr = (_batched if batched else _particles)(kind, **kw)
    pr.pol.Ds, pr.dyn.D = 3 + A, 3 + A + 1
    if kind == _lib.POLICY_RBF:
        pr.pol.rbf.D = 3 + A
    return pr


def _noise(var=(0.01, 0.02, 0.03), nu=FAKE):
    n = _lib.ParticlesNoise()
    for i, v in enumerate(var):
        n.v.var[i] = v
    n.nu = nu
    return n


class _FakeGP:
    """stands in for a DeviceGP in the engine's checks before device work: struct() only"""
    def __init__(self, n=40, D=6, E=4):
        self.n, self.D, self.E = n, D, E

    def struct(self):
        g = _lib.GpModel()
        g.n, g.D, g.E = self.n, self.D, self.E
        return g


def _score_grad_cases():
    """(description, R, grad, expected status): every call is rejected before anything is enqueued"""
    out = [(None, 3, _grad(), ERR_NULL), (_batched(), 3, None, ERR_NULL)]
    for kind in (_lib.POLICY_LINEAR, _lib.POLICY_RBF):
        for rk in (_lib.REWARD_EXP, _lib.REWARD_LINEAR, _lib.REWARD_BOX):
            for ch in (_lib.CHANNEL_ADD, _lib.CHANNEL_MULT):
                out.append((_batched(kind, reward_kind=rk, channel=ch), 3, _grad(), ERR_WS))
        out.append((_particles(kind), 3, _grad(), ERR_WS))                 # stride 0: one policy shared by all
        out.append((_particles(kind), 1, _grad(), ERR_WS))                 # R = 1, unbatched
    out.append((_particles(H=0), 1, _grad(), ERR_WS))
    out.append((_particles(H=1), 1, _grad(), ERR_WS))
    for R in (0, -1, 65536):
        out.append((_batched(), R, _grad(), ERR_DIM))
    out.append((_batched(P=1000), PT_MAX_P // 1000 + 1, _grad(), ERR_DIM))
    out.append((_batched(P=1), 65535, _grad(), ERR_WS))
    for field in ("W_bs", "b_bs"):
        pr = _batched(); setattr(pr.pol, field, -3)
        out.append((pr, 3, _grad(), ERR_DIM))
    for field in ("X_bs", "ell_bs", "sf2_bs", "beta_bs"):
        pr = _batched(_lib.POLICY_RBF); setattr(pr.pol.rbf, field, -1)
        out.append((pr, 3, _grad(), ERR_DIM))
        pr = _batched(); setattr(pr.dyn, field, 7)                         # batched dynamics
        out.append((pr, 3, _grad(), ERR_UNSUP))
    for P, H in ((0, 5), (PT_MAX_P + 1, 5), (10, -1)):
        out.append((_batched(P=P, H=H), 1, _grad(), ERR_DIM))
    for field in ("x0", "eps", "traj", "act", "step_reward", "step_risk", "ret"):
        pr = _batched(); setattr(pr, field, None)
        out.append((pr, 3, _grad(), ERR_NULL))
    pr = _batched(_lib.POLICY_RBF); pr.pol.rbf.mode = 0
    out.append((pr, 3, _grad(), ERR_UNSUP))
    pr = _batched(); pr.dyn.iK = None
    out.append((pr, 3, _grad(), ERR_UNSUP))
    out.append((_batched(kind=7), 3, _grad(), ERR_UNSUP))
    pr = _batched(); pr.dyn.E = 4
    out.append((pr, 3, _grad(), ERR_DIM))
    pr = _batched(); pr.dyn.iK = FAKE + 8
    out.append((pr, 3, _grad(), ERR_ALIGN))
    for field in ("value", "ws", "gW", "gb"):
        g = _grad(); setattr(g, field, None)
        out.append((_batched(), 3, g, ERR_NULL))
    for field in ("gXc", "gYc", "gell", "pol_L"):
        g = _grad(); setattr(g, field, None)
        out.append((_batched(_lib.POLICY_RBF), 3, g, ERR_NULL))
        out.append((_batched(), 3, g, ERR_WS))                             # not needed by the linear policy
    g = _grad(); g.ws = FAKE + 8; g.ws_bytes = 1 << 40
    out.append((_batched(), 3, g, ERR_ALIGN))
    return out
