"""Fake C-ABI descriptors for the tests that check argument validation without a GPU: the status codes of
include/pilco_b200.h and builders of pilco_gp_model, pilco_rollout, pilco_particles (plain and with per-restart
policies) and pilco_particles_grad whose pointers are fake non-null addresses.  Every entry point validates its
arguments on the host before it enqueues anything, so only calls that are rejected may be made with them."""
from pilco_b200 import _lib

OK, ERR_NULL, ERR_DIM, ERR_WS, ERR_ALIGN, ERR_LAUNCH, ERR_UNSUP = 0, -1, -2, -3, -4, -5, -6
FAKE = 0x10000          # 16-byte aligned, never dereferenced by the validation code
PT_MAX_P = 65535 * 32   # the particle kernels' largest P (and R P)


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
