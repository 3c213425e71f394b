"""Device-side plumbing: PyTorch owns every fp64 device buffer, the C ABI does the math.

Each function mirrors one C entry point; arguments are numpy arrays or CUDA tensors, results are
CUDA tensors (the API classes convert to host arrays at the boundary).  There is no CPU path:
``device()`` raises when no CUDA device is present.
"""
import ctypes as C

import numpy as np
import torch

from . import _lib
from ._lib import lib, check, GpModel

F64 = torch.float64


def device():
    if not torch.cuda.is_available():
        raise RuntimeError("pilco_b200: a CUDA device (H100, sm_90a) is required; "
                           "there is no CPU fallback for the moment-matching path")
    return torch.device("cuda", torch.cuda.current_device())


def stream_ptr():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def dev(x, dtype=F64):
    """numpy / tensor -> contiguous CUDA tensor"""
    if isinstance(x, torch.Tensor):
        return x.to(device=device(), dtype=dtype).contiguous()
    return torch.as_tensor(np.ascontiguousarray(np.asarray(x, dtype=np.float64)), dtype=dtype).to(device())


def ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


def pad_n(n):
    return int(lib.pilco_pad_n(int(n)))


class DeviceGP:
    """Device-resident factorised multi-output GP (what ``pilco_gp_model`` points at).

    ``X`` [B?,n,D], ``ell`` [B?,E,D], ``sf2`` [B?,E], ``beta`` [B?,E,n]; a leading batch dimension
    B (per-restart RBF policies) is optional and must match the rollout batch R.
    """

    def __init__(self, X, ell, sf2, beta, iK=None, ldk=0, mode=0, batched=False):
        self.X, self.ell, self.sf2, self.beta, self.iK = X, ell, sf2, beta, iK
        self.ldk, self.mode, self.batched = int(ldk), int(mode), bool(batched)
        self.n, self.D = int(X.shape[-2]), int(X.shape[-1])
        self.E = int(ell.shape[-2])

    def struct(self):
        g = GpModel()
        g.n, g.D, g.E, g.mode = self.n, self.D, self.E, self.mode
        b = self.batched
        g.X = self.X.data_ptr(); g.X_bs = self.n * self.D if b else 0
        g.ell = self.ell.data_ptr(); g.ell_bs = self.E * self.D if b else 0
        g.sf2 = self.sf2.data_ptr(); g.sf2_bs = self.E if b else 0
        g.beta = self.beta.data_ptr(); g.beta_bs = self.E * self.n if b else 0
        g.iK = self.iK.data_ptr() if self.iK is not None else None
        g.ldk = self.ldk
        return g


def gp_factorize(X, Y, ell, sf2, sn2, need_iK=True, mode=0):
    """pilco_gp_factorize.  Unbatched inputs ([n,D], [n,E], [E,D], [E], [E]) or batched with a leading B."""
    X, Y, ell, sf2, sn2 = dev(X), dev(Y), dev(ell), dev(sf2), dev(sn2)
    batched = X.dim() == 3
    B = X.shape[0] if batched else 1
    n, D = X.shape[-2], X.shape[-1]
    E = Y.shape[-1]
    ldk = pad_n(n)
    d = device()
    beta = torch.empty((B, E, n) if batched else (E, n), dtype=F64, device=d)
    iK = torch.empty((B, E, ldk, ldk) if batched else (E, ldk, ldk), dtype=F64, device=d) if need_iK else None
    info = torch.zeros(B, dtype=torch.int32, device=d)
    wsb = lib.pilco_gp_factorize_workspace_bytes(n, E, B)
    ws = torch.empty(wsb // 8, dtype=F64, device=d)
    bs = lambda t, per: (per if batched else 0)
    check(lib.pilco_gp_factorize(n, D, E, B,
                                 ptr(X), bs(X, n * D), ptr(Y), bs(Y, n * E), ptr(ell), bs(ell, E * D),
                                 ptr(sf2), bs(sf2, E), ptr(sn2), bs(sn2, E),
                                 ptr(iK), ldk, ptr(beta), ptr(info), ptr(ws), wsb, stream_ptr()),
          "gp_factorize")
    gp = DeviceGP(X, ell, sf2, beta, iK, ldk, mode=mode, batched=batched)
    gp.info = info
    gp.fact_ws = ws            # first B*E*ldw*ldw doubles = Cholesky factors (needed by the policy VJP)
    gp.Y, gp.sn2 = Y, sn2
    return gp


def gp_append(gp, X, Y):
    """pilco_gp_append: the factorised (unbatched, exact-GP) model ``gp`` with rows appended to its data and unchanged
    hyper-parameters.  ``X`` [n1,D], ``Y`` [n1,E] hold the old rows first.  Returns a NEW DeviceGP (n changes, so do the
    padded leading dimension and every workspace size downstream); the old inverse is consumed by the O(n^2 k)
    block-inverse update, no Cholesky factorisation of the full matrix is done."""
    if gp.batched or gp.iK is None or gp.mode != 0:
        raise ValueError("gp_append needs an unbatched exact-GP model with its inverse")
    X, Y = dev(X), dev(Y)
    n0, n1 = gp.n, int(X.shape[0])
    k = n1 - n0
    if k < 1:
        raise ValueError("gp_append: no rows appended")
    D, E = gp.D, gp.E
    ldk = pad_n(n1)
    d = device()
    beta = torch.empty((E, n1), dtype=F64, device=d)
    iK = torch.empty((E, ldk, ldk), dtype=F64, device=d)
    info = torch.zeros(1, dtype=torch.int32, device=d)
    wsb = lib.pilco_gp_append_workspace_bytes(n0, k, E)
    ws = torch.empty(wsb // 8, dtype=F64, device=d)
    check(lib.pilco_gp_append(n0, k, D, E, ptr(X), ptr(Y), ptr(gp.ell), ptr(gp.sf2), ptr(gp.sn2),
                              ptr(gp.iK), gp.ldk, ptr(iK), ldk, ptr(beta), ptr(info), ptr(ws), wsb, stream_ptr()),
          "gp_append")
    new = DeviceGP(X, gp.ell, gp.sf2, beta, iK, ldk, mode=0)
    new.info = info
    new.Y, new.sn2 = Y, gp.sn2
    new.appends = getattr(gp, "appends", 0) + 1
    return new


def gp_refactorize(gp):
    """Re-run pilco_gp_factorize in place after gp.X / gp.Y / gp.ell were overwritten (policy optimisation)."""
    B = gp.X.shape[0] if gp.batched else 1
    n, D, E = gp.n, gp.D, gp.E
    bs = lambda per: (per if gp.batched else 0)
    wsb = gp.fact_ws.numel() * 8
    check(lib.pilco_gp_factorize(n, D, E, B, ptr(gp.X), bs(n * D), ptr(gp.Y), bs(n * E), ptr(gp.ell), bs(E * D),
                                 ptr(gp.sf2), bs(E), ptr(gp.sn2), bs(E), ptr(gp.iK), gp.ldk, ptr(gp.beta),
                                 ptr(gp.info), ptr(gp.fact_ws), wsb, stream_ptr()), "gp_factorize")


class GpNlml:
    """pilco_gp_nlml with persistent buffers: -log p(y_e | X, theta) and gradients for B hyper-parameter sets."""

    def __init__(self, X, Y, B):
        d = device()
        self.X, self.Y = dev(X), dev(Y)
        self.n, self.D = self.X.shape
        self.E, self.B = self.Y.shape[1], int(B)
        B, E, D = self.B, self.E, self.D
        self.ell = torch.empty((B, E, D), dtype=F64, device=d)
        self.sf2 = torch.empty((B, E), dtype=F64, device=d)
        self.sn2 = torch.empty((B, E), dtype=F64, device=d)
        self.out = torch.empty((B, E, D + 3), dtype=F64, device=d)       # [g_ell | g_sf2 | g_sn2 | nlml]
        self.nlml = torch.empty((B, E), dtype=F64, device=d)
        self.g_ell = torch.empty((B, E, D), dtype=F64, device=d)
        self.g_sf2 = torch.empty((B, E), dtype=F64, device=d)
        self.g_sn2 = torch.empty((B, E), dtype=F64, device=d)
        self.info = torch.zeros(B, dtype=torch.int32, device=d)
        self.wsb = lib.pilco_gp_nlml_workspace_bytes(self.n, E, B)
        self.ws = torch.empty(self.wsb // 8, dtype=F64, device=d)

    def __call__(self, ell, sf2, sn2):
        """numpy [B,E,D], [B,E], [B,E] -> nlml [B,E], g_ell [B,E,D], g_sf2 [B,E], g_sn2 [B,E], bad [B] (numpy)"""
        self.ell.copy_(torch.as_tensor(ell)); self.sf2.copy_(torch.as_tensor(sf2)); self.sn2.copy_(torch.as_tensor(sn2))
        n, D, E, B = self.n, self.D, self.E, self.B
        check(lib.pilco_gp_nlml(n, D, E, B, ptr(self.X), 0, ptr(self.Y), 0, ptr(self.ell), E * D, ptr(self.sf2), E,
                                ptr(self.sn2), E, ptr(self.nlml), ptr(self.g_ell), ptr(self.g_sf2), ptr(self.g_sn2),
                                ptr(self.info), ptr(self.ws), self.wsb, stream_ptr()), "gp_nlml")
        return (self.nlml.cpu().numpy(), self.g_ell.cpu().numpy(), self.g_sf2.cpu().numpy(), self.g_sn2.cpu().numpy(),
                self.info.cpu().numpy() != 0)


class FitcNlml:
    """pilco_fitc_nlml with persistent buffers: FITC bound and its gradient w.r.t. (ell, sf2, sn2, Z) for B
    hyper-parameter sets x E outputs (each output with its own inducing inputs)."""

    def __init__(self, X, Y, Mi, B):
        d = device()
        self.X, self.Y = dev(X), dev(Y)
        self.N, self.D = self.X.shape
        self.E, self.B, self.Mi = self.Y.shape[1], int(B), int(Mi)
        B, E, D, Mi = self.B, self.E, self.D, self.Mi
        mk = lambda *shape: torch.empty(shape, dtype=F64, device=d)
        self.Z, self.ell, self.sf2, self.sn2 = mk(B, E, Mi, D), mk(B, E, D), mk(B, E), mk(B, E)
        self.nlml, self.g_ell, self.g_sf2, self.g_sn2, self.g_Z = mk(B, E), mk(B, E, D), mk(B, E), mk(B, E), mk(B, E, Mi, D)
        self.info = torch.zeros(B, dtype=torch.int32, device=d)
        self.wsb = lib.pilco_fitc_nlml_workspace_bytes(self.N, Mi, D, E, B)
        self.ws = torch.empty(self.wsb // 8, dtype=F64, device=d)

    def __call__(self, Z, ell, sf2, sn2):
        """numpy [B,E,Mi,D], [B,E,D], [B,E], [B,E] -> nlml, g_ell, g_sf2, g_sn2, g_Z, bad [B] (numpy)"""
        for dst, src in ((self.Z, Z), (self.ell, ell), (self.sf2, sf2), (self.sn2, sn2)):
            dst.copy_(torch.as_tensor(np.ascontiguousarray(src)))
        check(lib.pilco_fitc_nlml(self.N, self.Mi, self.D, self.E, self.B, ptr(self.X), ptr(self.Y), ptr(self.Z),
                                  ptr(self.ell), ptr(self.sf2), ptr(self.sn2), ptr(self.nlml), ptr(self.g_ell),
                                  ptr(self.g_sf2), ptr(self.g_sn2), ptr(self.g_Z), ptr(self.info), ptr(self.ws), self.wsb,
                                  stream_ptr()), "fitc_nlml")
        return (self.nlml.cpu().numpy(), self.g_ell.cpu().numpy(), self.g_sf2.cpu().numpy(), self.g_sn2.cpu().numpy(),
                self.g_Z.cpu().numpy(), self.info.cpu().numpy() != 0)


def fitc_factorize(X, Z, Y, ell, sf2, sn2):
    """pilco_fitc_factorize: FITC over inducing points Z -> DeviceGP centred on Z."""
    X, Z, Y, ell, sf2, sn2 = dev(X), dev(Z), dev(Y), dev(ell), dev(sf2), dev(sn2)
    N, D = X.shape
    Mi = Z.shape[0]
    E = Y.shape[1]
    ldk = pad_n(Mi)
    d = device()
    beta = torch.empty((E, Mi), dtype=F64, device=d)
    iK = torch.empty((E, ldk, ldk), dtype=F64, device=d)
    info = torch.zeros(1, dtype=torch.int32, device=d)
    wsb = lib.pilco_fitc_workspace_bytes(N, Mi, E)
    ws = torch.empty(wsb // 8, dtype=F64, device=d)
    check(lib.pilco_fitc_factorize(N, Mi, D, E, ptr(X), ptr(Z), ptr(Y), ptr(ell), ptr(sf2), ptr(sn2),
                                   ptr(iK), ldk, ptr(beta), ptr(info), ptr(ws), wsb, stream_ptr()),
          "fitc_factorize")
    gp = DeviceGP(Z, ell, sf2, beta, iK, ldk, mode=0)
    gp.info = info
    return gp


def gp_predict(gp, Xnew, e0=0, ne=None, full_cov=False):
    """pilco_gp_predict: posterior of outputs e0 .. e0+ne-1 of the factorised model ``gp`` at deterministic inputs
    Xnew [T,D] -> mean [T,ne] and the latent variance, [T,ne] or with ``full_cov`` the covariance [ne,T,T]."""
    Xs = dev(Xnew)
    if Xs.dim() != 2 or Xs.shape[1] != gp.D:
        raise ValueError("gp_predict: Xnew must be [T, %d], got %s" % (gp.D, tuple(Xs.shape)))
    T = int(Xs.shape[0])
    ne = gp.E - int(e0) if ne is None else int(ne)
    if T < 1 or ne < 1:
        raise ValueError("gp_predict: needs at least one input row and one output (T=%d, ne=%d)" % (T, ne))
    d = device()
    mean = torch.empty((T, ne), dtype=F64, device=d)
    var = torch.empty((ne, T, T) if full_cov else (T, ne), dtype=F64, device=d)
    wsb = lib.pilco_gp_predict_workspace_bytes(gp.n, gp.D, ne, T, 1 if full_cov else 0)
    ws = torch.empty(max(wsb // 8, 2), dtype=F64, device=d)
    g = gp.struct()
    check(lib.pilco_gp_predict(C.byref(g), int(e0), ne, T, ptr(Xs), ptr(mean), ptr(var), 1 if full_cov else 0,
                               ptr(ws), wsb, stream_ptr()), "gp_predict")
    return mean, var


def mm_forward(gp, m, s):
    """pilco_mm_forward: m [R,D], s [R,D,D] -> M [R,E], S [R,E,E], V [R,D,E], info [R]."""
    m, s = dev(m), dev(s)
    R = m.shape[0]
    d = device()
    M = torch.empty((R, gp.E), dtype=F64, device=d)
    S = torch.empty((R, gp.E, gp.E), dtype=F64, device=d)
    V = torch.empty((R, gp.D, gp.E), dtype=F64, device=d)
    info = torch.zeros(R, dtype=torch.int32, device=d)
    wsb = lib.pilco_mm_workspace_bytes(gp.n, gp.D, gp.E, R)
    ws = torch.empty(wsb // 8, dtype=F64, device=d)
    g = gp.struct()
    check(lib.pilco_mm_forward(C.byref(g), R, ptr(m), ptr(s), ptr(M), ptr(S), ptr(V), ptr(info),
                               ptr(ws), wsb, stream_ptr()), "mm_forward")
    return M, S, V, info


def mm_backward(gp, m, s, M, gM, gS, gV, need_param=False):
    """pilco_mm_backward -> gm [R,D], gs [R,D,D] (+ gX [R,n,D], gbeta [R,E,n], gell [R,E,D])."""
    m, s, M, gM, gS, gV = dev(m), dev(s), dev(M), dev(gM), dev(gS), dev(gV)
    R = m.shape[0]
    d = device()
    gm = torch.empty((R, gp.D), dtype=F64, device=d)
    gs = torch.empty((R, gp.D, gp.D), dtype=F64, device=d)
    gX = gb = gl = None
    if need_param:
        gX = torch.empty((R, gp.n, gp.D), dtype=F64, device=d)
        gb = torch.empty((R, gp.E, gp.n), dtype=F64, device=d)
        gl = torch.empty((R, gp.E, gp.D), dtype=F64, device=d)
    wsb = lib.pilco_mm_bwd_workspace_bytes(gp.n, gp.D, gp.E, R, 1 if need_param else 0)
    ws = torch.empty(wsb // 8, dtype=F64, device=d)
    g = gp.struct()
    check(lib.pilco_mm_backward(C.byref(g), R, ptr(m), ptr(s), ptr(M), ptr(gM), ptr(gS), ptr(gV),
                                ptr(gm), ptr(gs), ptr(gX), ptr(gb), ptr(gl), ptr(ws), wsb, stream_ptr()), "mm_backward")
    return gm, gs, gX, gb, gl


def mm_forward_taped(gp, m, s):
    """pilco_mm_forward_taped: as mm_forward, plus the tape (opaque device buffer) for mm_backward_taped."""
    m, s = dev(m), dev(s)
    R = m.shape[0]
    d = device()
    M = torch.empty((R, gp.E), dtype=F64, device=d)
    S = torch.empty((R, gp.E, gp.E), dtype=F64, device=d)
    V = torch.empty((R, gp.D, gp.E), dtype=F64, device=d)
    info = torch.zeros(R, dtype=torch.int32, device=d)
    wsb = lib.pilco_mm_workspace_bytes(gp.n, gp.D, gp.E, R)
    ws = torch.empty(wsb // 8, dtype=F64, device=d)
    tb = lib.pilco_mm_tape_bytes(gp.n, gp.D, gp.E, R)
    if tb == 0:
        raise ValueError("taped moment match: %d centres (D=%d) exceed what its shared-memory staging holds (n <= 1024 for D <= 12)" % (gp.n, gp.D))
    tape = torch.empty(tb // 8, dtype=F64, device=d)
    g = gp.struct()
    check(lib.pilco_mm_forward_taped(C.byref(g), R, ptr(m), ptr(s), ptr(M), ptr(S), ptr(V), ptr(info),
                                     ptr(ws), wsb, ptr(tape), tb, stream_ptr()), "mm_forward_taped")
    return M, S, V, info, tape


def mm_backward_taped(gp, m, s, M, gM, gS, gV, tape):
    """pilco_mm_backward_taped -> gm [R,D], gs [R,D,D] from the tape of mm_forward_taped (no recomputation)."""
    m, s, M, gM, gS, gV = dev(m), dev(s), dev(M), dev(gM), dev(gS), dev(gV)
    R = m.shape[0]
    d = device()
    gm = torch.empty((R, gp.D), dtype=F64, device=d)
    gs = torch.empty((R, gp.D, gp.D), dtype=F64, device=d)
    wsb = lib.pilco_mm_tape_bwd_workspace_bytes(gp.D, gp.E, R)
    ws = torch.empty(wsb // 8, dtype=F64, device=d)
    g = gp.struct()
    check(lib.pilco_mm_backward_taped(C.byref(g), R, ptr(m), ptr(s), ptr(M), ptr(gM), ptr(gS), ptr(gV),
                                      ptr(tape), tape.numel() * 8, ptr(gm), ptr(gs), ptr(ws), wsb, stream_ptr()),
          "mm_backward_taped")
    return gm, gs


def squash_sin(m, s, max_action):
    m, s, e = dev(m), dev(s), dev(max_action)
    R, U = m.shape
    d = device()
    M = torch.empty((R, U), dtype=F64, device=d)
    S = torch.empty((R, U, U), dtype=F64, device=d)
    Cq = torch.empty((R, U, U), dtype=F64, device=d)
    check(lib.pilco_squash_sin(U, R, ptr(m), ptr(s), ptr(e), ptr(M), ptr(S), ptr(Cq), stream_ptr()), "squash_sin")
    return M, S, Cq


def linear_action(W, b, m, s):
    W, b, m, s = dev(W), dev(b), dev(m), dev(s)
    R, Ds = m.shape
    U = W.shape[-2]
    batched = W.dim() == 3
    d = device()
    M = torch.empty((R, U), dtype=F64, device=d)
    S = torch.empty((R, U, U), dtype=F64, device=d)
    V = torch.empty((R, Ds, U), dtype=F64, device=d)
    check(lib.pilco_linear_action(Ds, U, R, ptr(W), U * Ds if batched else 0, ptr(b), U if batched else 0,
                                  ptr(m), ptr(s), ptr(M), ptr(S), ptr(V), stream_ptr()), "linear_action")
    return M, S, V


def exp_reward(W, t, m, s, variance=True):
    W, t, m, s = dev(W), dev(t), dev(m), dev(s)
    R, Ds = m.shape
    d = device()
    mu = torch.empty(R, dtype=F64, device=d)
    sR = torch.empty(R, dtype=F64, device=d) if variance else None
    check(lib.pilco_exp_reward(Ds, R, ptr(W), ptr(t), ptr(m), ptr(s), ptr(mu), ptr(sR), None, stream_ptr()),
          "exp_reward")
    return mu, sR


def box_risk(prm, m, s, grad=False):
    """pilco_box_risk: prm = [nd, inside, sfac, (dim, low, high) x nd]; m [R,Ds], s [R,Ds,Ds] -> risk [R]
    (+ d risk/d m [R,Ds], d risk/d diag(s) [R,Ds] when ``grad``)."""
    prm, m, s = dev(prm), dev(m), dev(s)
    R, Ds = m.shape
    d = device()
    risk = torch.empty(R, dtype=F64, device=d)
    dm = torch.empty((R, Ds), dtype=F64, device=d) if grad else None
    dv = torch.empty((R, Ds), dtype=F64, device=d) if grad else None
    check(lib.pilco_box_risk(Ds, R, ptr(prm), ptr(m), ptr(s), ptr(risk), ptr(dm), ptr(dv), stream_ptr()), "box_risk")
    return (risk, dm, dv) if grad else risk


def _max_action(policy_spec, U):
    """the policy spec's max_action (scalar or [U]) as a [U] device tensor"""
    return dev(np.broadcast_to(np.asarray(policy_spec.get("max_action", 1.0), dtype=np.float64).ravel(), (U,)).copy())


def _fill_policy(pol, policy_spec, batched=None):
    """Fill the pilco_policy ``pol`` from a policy spec: kind, Ds, U, squash, max_action and either the linear W/b
    (batch strides when ``batched``; None: when W has a leading batch dimension) or the RBF policy GP.  Returns the
    device tensors and the policy GP it points to: (max_action, W, b, rbf), W and b None for an RBF policy, rbf None
    for a linear one."""
    pol.kind = policy_spec["kind"]
    pol.Ds, pol.U = Ds, U = int(policy_spec["Ds"]), int(policy_spec["U"])
    pol.squash = 1 if policy_spec.get("squash", True) else 0
    max_action, W, b, rbf = _max_action(policy_spec, U), None, None, None
    pol.max_action = max_action.data_ptr()
    if pol.kind == _lib.POLICY_LINEAR:
        W, b = dev(policy_spec["W"]), dev(policy_spec["b"])
        bat = W.dim() == 3 if batched is None else batched
        pol.W, pol.W_bs = W.data_ptr(), U * Ds if bat else 0
        pol.b, pol.b_bs = b.data_ptr(), U if bat else 0
    else:
        rbf = policy_spec["gp"]
        pol.rbf = rbf.struct()
    return max_action, W, b, rbf


def _fill_rewards(desc, reward_terms):
    """Fill ``desc.n_rewards`` and ``desc.rewards`` from reward-term dicts; returns the device tensors [(W, t)] they
    point to"""
    rw = []
    desc.n_rewards = len(reward_terms)
    for k, rt in enumerate(reward_terms):
        W = dev(rt["W"]); t = dev(rt["t"]) if rt.get("t") is not None else None
        rw.append((W, t))
        desc.rewards[k].kind = rt["kind"]
        desc.rewards[k].channel = int(rt.get("channel", _lib.CHANNEL_ADD))
        desc.rewards[k].coef = float(rt.get("coef", 1.0))
        desc.rewards[k].W = W.data_ptr()
        desc.rewards[k].t = t.data_ptr() if t is not None else None
    return rw


def _policy_grad_buffers(g, pol, rbf, lead):
    """the policy-gradient outputs of ``g`` (pilco_rollout_grad / pilco_particles_grad) for the policy ``pol``, with
    leading dimensions ``lead``: {'W', 'b'} (linear) or {'X', 'Y', 'ell'} and the factors pol_L (RBF policy GP
    ``rbf``).  Zero-filled; the C code overwrites or zeroes them itself."""
    mk = lambda *shape: torch.zeros(shape, dtype=F64, device=device())
    Ds, U = pol.Ds, pol.U
    if pol.kind == _lib.POLICY_LINEAR:
        buf = {"W": mk(*lead, U, Ds), "b": mk(*lead, U)}
        g.gW, g.gb = buf["W"].data_ptr(), buf["b"].data_ptr()
    else:
        buf = {"X": mk(*lead, rbf.n, Ds), "Y": mk(*lead, rbf.n, U), "ell": mk(*lead, U, Ds)}
        g.gXc, g.gYc, g.gell = (buf[k].data_ptr() for k in ("X", "Y", "ell"))
        g.pol_L = rbf.fact_ws.data_ptr()
    return buf


class RolloutPlan:
    """Owns the buffers of one ``pilco_rollout`` description (batch R, horizon H) and launches it.

    ``reward_terms``: dicts ``kind, coef, W, t`` (+ ``channel``: additive terms accumulate as in PILCO.predict,
    pilco.py:130-134; multiplicative ones form the per-step risk of SafePILCO.predict, safe_pilco.py:29-50, and
    enter the returned reward as ``mult_mu * (1 - prod_t (1 - risk_t))``)."""

    def __init__(self, dyn, policy_spec, reward_terms, m0, S0, H, R=1, mult_mu=0.0, grad=False):
        """``grad=True``: the forward cascade runs the TAPED dynamics tile pass (pilco_rollout.tape), so that
        ``backward()`` needs no recomputation; without it ``backward()`` still works (recomputing path)."""
        d = device()
        self.dyn = dyn
        self.R, self.H = int(R), int(H)
        self.Ds, self.U = policy_spec["Ds"], policy_spec["U"]
        self.keep = [dyn, policy_spec, reward_terms]            # keep device tensors alive
        ro = _lib.Rollout()
        ro.R, ro.H = self.R, self.H
        ro.dyn = dyn.struct()
        self.max_action, self.W, self.b, self.rbf = _fill_policy(ro.pol, policy_spec)
        self.rw = _fill_rewards(ro, reward_terms)
        self.m0, self.S0 = dev(m0), dev(S0)
        # per-restart initial moments: leading dimension R (and R > 1); [1, ...] or unbatched = shared by the batch
        def _batched(t, tail, what):
            if t.numel() == int(np.prod(tail)):
                return False
            if t.numel() == self.R * int(np.prod(tail)) and t.shape[0] == self.R:
                return True
            raise ValueError("%s: expected shape %s or [R=%d, ...], got %s" % (what, tuple(tail), self.R, tuple(t.shape)))
        bat0 = _batched(self.m0, (self.Ds,), "m0")
        self.m0 = self.m0.reshape(self.R, self.Ds) if bat0 else self.m0.reshape(self.Ds)
        ro.m0 = self.m0.data_ptr(); ro.m0_bs = self.Ds if bat0 else 0
        batS = _batched(self.S0, (self.Ds, self.Ds), "S0")
        self.S0 = self.S0.reshape(self.R, self.Ds, self.Ds) if batS else self.S0.reshape(self.Ds, self.Ds)
        ro.S0 = self.S0.data_ptr(); ro.S0_bs = self.Ds * self.Ds if batS else 0
        self.traj_m = torch.empty((self.R, self.H + 1, self.Ds), dtype=F64, device=d)
        self.traj_S = torch.empty((self.R, self.H + 1, self.Ds, self.Ds), dtype=F64, device=d)
        self.reward = torch.empty(self.R, dtype=F64, device=d)
        self.step_reward = torch.empty((self.R, max(self.H, 1)), dtype=F64, device=d)
        self.step_risk = torch.zeros((self.R, max(self.H, 1)), dtype=F64, device=d)
        ro.mult_mu = float(mult_mu)
        ro.step_risk = self.step_risk.data_ptr()
        self.info = torch.zeros(self.R, dtype=torch.int32, device=d)
        ro.traj_m, ro.traj_S = self.traj_m.data_ptr(), self.traj_S.data_ptr()
        ro.reward, ro.step_reward, ro.info = self.reward.data_ptr(), self.step_reward.data_ptr(), self.info.data_ptr()
        wsb = lib.pilco_rollout_workspace_bytes(C.byref(ro))
        self.ws = torch.empty(max(wsb // 8, 2), dtype=F64, device=d)
        ro.ws, ro.ws_bytes = self.ws.data_ptr(), wsb
        self.tape = None
        if grad and self.H > 0:
            tb = lib.pilco_rollout_tape_bytes(C.byref(ro))
            if tb:                                              # (0: more than 2048 centres -> recomputing backward)
                self.tape = torch.empty(tb // 8, dtype=F64, device=d)
                ro.tape, ro.tape_bytes = self.tape.data_ptr(), tb
        self.ro = ro

    def forward(self):
        check(lib.pilco_rollout_forward(C.byref(self.ro), stream_ptr()), "rollout_forward")
        return self.traj_m, self.traj_S, self.reward

    # ---- CUDA graph: the whole H-step loop (6H+1 launches forward, ~10H backward) as one graph launch -------
    def capture(self, backward=False):
        """Capture forward (and optionally the reverse sweep) into a CUDA graph.  Buffers are static, the C
        entry points only enqueue work on the current stream, so stream capture records every launch."""
        self.forward()                       # warm-up: one-time function attributes are set here
        if backward:
            self.backward()
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            self.forward()
            if backward:
                self.backward()
        self.graph = g
        return g

    def replay(self):
        self.graph.replay()
        return self.traj_m, self.traj_S, self.reward

    def backward(self):
        """pilco_rollout_backward: d reward[r] / d policy parameters (call after forward()).
        Linear: {'W': [R,U,Ds], 'b': [R,U]};  RBF: {'X': [R,bf,Ds], 'Y': [R,bf,U], 'ell': [R,U,Ds]}."""
        d = device()
        if not hasattr(self, "grad"):
            g = _lib.RolloutGrad()
            R, Ds = self.R, self.Ds
            self.gbuf = _policy_grad_buffers(g, self.ro.pol, self.rbf, (R,))
            self.gbuf["m0"] = torch.empty((R, Ds), dtype=F64, device=d)
            self.gbuf["S0"] = torch.empty((R, Ds, Ds), dtype=F64, device=d)
            g.gm0, g.gS0 = self.gbuf["m0"].data_ptr(), self.gbuf["S0"].data_ptr()
            wsb = lib.pilco_rollout_bwd_workspace_bytes(C.byref(self.ro))
            self.bws = torch.empty(max(wsb // 8, 2), dtype=F64, device=d)
            g.ws, g.ws_bytes = self.bws.data_ptr(), wsb
            self.grad = g
        check(lib.pilco_rollout_backward(C.byref(self.ro), C.byref(self.grad), stream_ptr()), "rollout_backward")
        return self.gbuf


class ParticlePlan:
    """Owns the buffers of one ``pilco_particles`` description (P particles, horizon H) and launches it.

    ``x0`` [P,Ds] and ``eps`` [P,H,Ds] are static device buffers: fill them (``set_inputs``) and ``launch()``, or
    capture ``launch()`` in a CUDA graph.  Policy and reward terms as for ``RolloutPlan``; one policy is unbatched.
    ``grad=True`` also allocates the buffers of ``launch_grad()`` (pilco_particles_rollout_grad).

    A batch of policies (``R > 1``, or an RBF policy factorised with a leading batch dimension) takes a policy spec
    with a leading R, as ``RolloutPlan`` does, and needs ``grad=True``: ``launch_grad()`` then runs the R policies over
    the same x0 and eps (pilco_particles_rollout_batch_grad) and every output has a leading R.

    ``consistent=True``: ``launch()`` samples each particle's dynamics as ONE function drawn from the GP posterior
    (pilco_particles_rollout_consistent, DESIGN.md section 14) instead of fresh noise at every step; its workspace is
    O(P H E n).  Its gradient is ``ConsistentGradPlan``; ``grad=True`` with ``consistent=True`` is a ValueError.

    ``estimator`` picks what ``launch_grad()`` estimates d E[return] with: ``"pathwise"`` (the default) differentiates
    the sampled trajectories; ``"score"`` is the score-function estimator (pilco_particles_rollout_score_grad, DESIGN.md
    section 16), which differentiates no trajectory, so box terms enter its gradient.  Both give the same rollout and
    value.  ``"score"`` with ``consistent=True``, or an unknown estimator, is a ValueError."""

    ESTIMATORS = ("pathwise", "score")

    def __init__(self, dyn, policy_spec, reward_terms, P, H, mult_mu=0.0, grad=False, R=1, consistent=False,
                 estimator="pathwise"):
        if estimator not in self.ESTIMATORS:
            raise ValueError("particles: estimator must be one of %s, not %r" % (self.ESTIMATORS, estimator))
        if consistent and estimator == "score":
            raise ValueError("particles: the score-function gradient of the consistent (function-sample) rollout "
                             "is not available; use estimator='pathwise'")
        self.estimator = estimator
        if consistent and grad:
            raise ValueError("particles: the gradient of the consistent (function-sample) rollout is "
                             "ConsistentGradPlan, not ParticlePlan(grad=True)")
        self.consistent = bool(consistent)
        self._describe(dyn, policy_spec, reward_terms, P, H, mult_mu, R, grad)
        pr, d = self.pr, device()
        P, H = self.P, self.H
        if self.consistent:
            wsb = lib.pilco_particles_consistent_workspace_bytes(C.byref(pr))
            if wsb == 0:
                raise ValueError("particles: unsupported sizes (P=%d, H=%d, D=%d)" % (P, H, dyn.D))
            self.ws = torch.empty(max(wsb // 8, 2), dtype=F64, device=d)
            pr.ws, pr.ws_bytes = self.ws.data_ptr(), wsb
        elif not self.batched:                                  # the forward-only rollout (a batch has none)
            wsb = lib.pilco_particles_workspace_bytes(C.byref(pr))
            if wsb == 0:
                raise ValueError("particles: unsupported sizes (P=%d, H=%d, D=%d)" % (P, H, dyn.D))
            self.ws = torch.empty(max(wsb // 8, 2), dtype=F64, device=d)
            pr.ws, pr.ws_bytes = self.ws.data_ptr(), wsb
        self.grad = None
        if grad:
            self._grad_buffers(self._grad_ws_bytes(P))

    def _grad_ws_bytes(self, P):
        """the gradient workspace of this plan's call with P particles per restart (0: unsupported sizes)"""
        pr = _lib.Particles.from_buffer_copy(self.pr)
        pr.P = int(P)
        if self.estimator == "score":
            return int(lib.pilco_particles_score_grad_workspace_bytes(C.byref(pr), self.R))
        if self.batched:
            return int(lib.pilco_particles_batch_grad_workspace_bytes(C.byref(pr), self.R))
        return int(lib.pilco_particles_grad_workspace_bytes(C.byref(pr)))

    def _describe(self, dyn, policy_spec, reward_terms, P, H, mult_mu, R, grad):
        """the pilco_particles description, its input and output buffers (self.pr)"""
        d = device()
        self.P, self.H, self.R = int(P), int(H), int(R)
        self.Ds, self.U = int(policy_spec["Ds"]), int(policy_spec["U"])
        P, H, Ds, U, R = self.P, self.H, self.Ds, self.U, self.R
        if P < 1 or H < 0 or R < 1:
            raise ValueError("particles: needs P >= 1, H >= 0 and R >= 1 (P=%d, H=%d, R=%d)" % (P, H, R))
        rbf_batched = policy_spec["kind"] == _lib.POLICY_RBF and policy_spec["gp"].batched
        self.batched = R > 1 or rbf_batched
        if self.batched and not grad:
            raise ValueError("particles: a batch of policies runs the gradient path only (grad=True)")
        lead = (R,) if self.batched else ()
        self.lead = lead
        self.keep = [dyn, policy_spec, reward_terms]            # keep device tensors alive
        pr = _lib.Particles()
        pr.P, pr.H = P, H
        pr.dyn = dyn.struct()
        self.max_action, self.W, self.b, self.rbf = _fill_policy(pr.pol, policy_spec, self.batched)
        if pr.pol.kind == _lib.POLICY_LINEAR:
            if self.W.numel() != R * U * Ds or self.b.numel() != R * U:
                raise ValueError("particles: expected W [R,U,Ds] and b [R,U] with R=%d (unbatched: [U,Ds], [U])" % R)
        elif self.rbf.batched != self.batched or (self.batched and self.rbf.X.shape[0] != R):
            raise ValueError("particles: the RBF policy must be factorised with a leading R=%d (unbatched: none)" % R)
        self.rw = _fill_rewards(pr, reward_terms)
        pr.mult_mu = float(mult_mu)
        mk = lambda *shape: torch.zeros(shape, dtype=F64, device=d)
        Hb = max(H, 1)                                          # H = 0: every buffer still has an address
        self.x0, self.eps_buf = mk(P, Ds), mk(P, Hb, Ds)                  # shared by the R policies
        self.traj, self.act_buf = mk(*lead, P, H + 1, Ds), mk(*lead, P, Hb, U)
        self.rew_buf, self.risk_buf, self.ret = mk(*lead, P, Hb), mk(*lead, P, Hb), mk(*lead, P)
        pr.x0, pr.eps = self.x0.data_ptr(), self.eps_buf.data_ptr()
        pr.traj, pr.act = self.traj.data_ptr(), self.act_buf.data_ptr()
        pr.step_reward, pr.step_risk, pr.ret = self.rew_buf.data_ptr(), self.risk_buf.data_ptr(), self.ret.data_ptr()
        self.pr = pr

    def _grad_buffers(self, gwsb):
        """the pilco_particles_grad outputs and a gradient workspace of gwsb bytes (self.grad)"""
        d, pr = device(), self.pr
        if gwsb == 0:
            raise ValueError("particles: unsupported sizes (P=%d, H=%d, D=%d, R=%d)" % (self.P, self.H, pr.dyn.D, self.R))
        g = _lib.ParticlesGrad()
        self.gbuf = _policy_grad_buffers(g, pr.pol, self.rbf, self.lead)
        self.gbuf["value"] = torch.zeros(self.R if self.batched else 1, dtype=F64, device=d)
        g.value = self.gbuf["value"].data_ptr()
        self.gws = torch.empty(max(gwsb // 8, 2), dtype=F64, device=d)
        g.ws, g.ws_bytes = self.gws.data_ptr(), gwsb
        self.grad = g

    def launch_grad(self):
        """pilco_particles_rollout_grad: the rollout (``outputs()`` as after ``launch()``, bitwise) and the pathwise
        gradient of value = mean return w.r.t. the policy parameters with x0 and eps fixed.  Returns the device tensors
        {'value' [1], 'W' [U,Ds], 'b' [U]} (linear) or {'value', 'X' [bf,Ds], 'Y' [bf,U], 'ell' [U,Ds]} (RBF, constrained
        lengthscales), like ``RolloutPlan.backward``.  A batched plan returns them with a leading R ('value' [R]).
        ``estimator="score"``: the score-function gradient (pilco_particles_rollout_score_grad) in the same layout."""
        if self.grad is None:
            raise RuntimeError("ParticlePlan: constructed without grad=True")
        if self.estimator == "score":
            check(lib.pilco_particles_rollout_score_grad(C.byref(self.pr), self.R, C.byref(self.grad), stream_ptr()),
                  "particles_rollout_score_grad")
        elif self.batched:
            check(lib.pilco_particles_rollout_batch_grad(C.byref(self.pr), self.R, C.byref(self.grad), stream_ptr()),
                  "particles_rollout_batch_grad")
        else:
            check(lib.pilco_particles_rollout_grad(C.byref(self.pr), C.byref(self.grad), stream_ptr()),
                  "particles_rollout_grad")
        return self.gbuf

    def set_inputs(self, x0, eps):
        self.x0.copy_(dev(x0).reshape(self.P, self.Ds))
        if self.H > 0:
            self.eps_buf.copy_(dev(eps).reshape(self.P, self.H, self.Ds))

    def launch(self):
        if self.batched:
            raise RuntimeError("ParticlePlan: a batch of policies runs launch_grad()")
        if self.consistent:
            check(lib.pilco_particles_rollout_consistent(C.byref(self.pr), stream_ptr()), "particles_rollout_consistent")
            return
        check(lib.pilco_particles_rollout(C.byref(self.pr), stream_ptr()), "particles_rollout")

    def outputs(self):
        """(traj [P,H+1,Ds], act [P,H,U], step_reward [P,H], step_risk [P,H], ret [P]) device tensors (views), each
        with a leading R for a batched plan"""
        H = self.H
        return self.traj, self.act_buf[..., :H, :], self.rew_buf[..., :H], self.risk_buf[..., :H], self.ret


class ConsistentGradPlan(ParticlePlan):
    """The consistent (function-sample) rollout of ``ParticlePlan(consistent=True)`` and the pathwise gradient of its
    mean return w.r.t. the policy parameters with x0 and eps fixed (pilco_particles_rollout_consistent_grad, DESIGN.md
    section 15): ``set_inputs``, ``launch_grad()`` and ``outputs()`` in ``ParticlePlan``'s layout, each with a leading
    R for a batch of policies (``R > 1`` or a batched RBF policy; the R policies share x0 and eps).  The forward
    outputs are bitwise those of ``ParticlePlan(consistent=True).launch()`` with the same policy.

    The workspace is O(R P H E n) and is not chunked: chunking the particles would reorder the gradient's fixed-order
    sums.  A plan whose workspace exceeds ``max_ws_bytes`` (default: half the free device memory) is a ValueError
    that names the bytes needed and the number of particles that would fit, raised before anything is allocated."""

    def __init__(self, dyn, policy_spec, reward_terms, P, H, mult_mu=0.0, R=1, max_ws_bytes=None):
        self.consistent = True
        self._describe(dyn, policy_spec, reward_terms, P, H, mult_mu, R, True)
        need = self._grad_ws_bytes(self.P)
        if need == 0:
            raise ValueError("particles: unsupported sizes (P=%d, H=%d, D=%d, R=%d)" % (self.P, self.H, dyn.D, self.R))
        if max_ws_bytes is None:
            max_ws_bytes = torch.cuda.mem_get_info(device())[0] // 2
        if need > max_ws_bytes:
            lo = _largest_fitting(lambda p: 0 < self._grad_ws_bytes(p) <= max_ws_bytes, 0, self.P - 1)
            raise ValueError("particles: the consistent gradient of %d restarts x %d particles over H=%d steps needs %d "
                             "workspace bytes, more than max_ws_bytes=%d (half the free device memory by default); "
                             "num_samples=%d would fit" % (self.R, self.P, self.H, need, max_ws_bytes, lo))
        self._grad_buffers(need)

    def _grad_ws_bytes(self, P):
        if P < 1:
            return 0
        pr = _lib.Particles.from_buffer_copy(self.pr)
        pr.P = int(P)
        return int(lib.pilco_particles_consistent_grad_workspace_bytes(C.byref(pr), self.R))

    def launch(self):
        raise RuntimeError("ConsistentGradPlan: the rollout runs with its gradient, launch_grad()")

    def launch_grad(self):
        """pilco_particles_rollout_consistent_grad: the consistent rollout (``outputs()``) and the pathwise gradient
        of value = mean return, returned as ``ParticlePlan.launch_grad`` returns it"""
        check(lib.pilco_particles_rollout_consistent_grad(C.byref(self.pr), self.R, C.byref(self.grad), stream_ptr()),
              "particles_rollout_consistent_grad")
        return self.gbuf


def _largest_fitting(fits, lo, hi):
    """the largest p in [lo, hi] with fits(p), by bisection; fits must be monotone and hold at lo (or lo is returned)"""
    while lo < hi:
        mid = (lo + hi + 1) // 2
        lo, hi = (mid, hi) if fits(mid) else (lo, mid - 1)
    return lo


def gp_predict_vjp(gp, Xs, gmean, gvar):
    """pilco_gp_predict_vjp: d/dXs of sum(gmean * mean + gvar * var) over all E outputs of the (unbatched, mode-0)
    factorised model ``gp`` at Xs [T,D]; gmean, gvar [T,E] -> [T,D] device tensor."""
    Xs, gmean, gvar = dev(Xs), dev(gmean), dev(gvar)
    T = int(Xs.shape[0])
    if Xs.shape != (T, gp.D) or gmean.shape != (T, gp.E) or gvar.shape != (T, gp.E):
        raise ValueError("gp_predict_vjp: expected Xs [T,%d], gmean and gvar [T,%d]" % (gp.D, gp.E))
    out = torch.empty((T, gp.D), dtype=F64, device=device())
    wsb = lib.pilco_gp_predict_vjp_workspace_bytes(gp.n, gp.D, gp.E, T)
    if wsb == 0:
        raise ValueError("gp_predict_vjp: unsupported sizes (n=%d, D=%d, E=%d, T=%d)" % (gp.n, gp.D, gp.E, T))
    ws = torch.empty(wsb // 8, dtype=F64, device=device())
    g = gp.struct()
    check(lib.pilco_gp_predict_vjp(C.byref(g), T, ptr(Xs), ptr(gmean), ptr(gvar), ptr(out), ptr(ws), wsb,
                                   stream_ptr()), "gp_predict_vjp")
    return out


def particles_rollout(dyn, policy_spec, reward_terms, x0, eps, mult_mu=0.0, consistent=False, max_ws_bytes=None):
    """pilco_particles_rollout: P particles from x0 [P,Ds] driven by the standard normals eps [P,H,Ds] through the
    factorised dynamics ``dyn`` under the (unbatched) policy -> (traj [P,H+1,Ds], act [P,H,U], step_reward [P,H],
    step_risk [P,H], ret [P]) device tensors.

    ``consistent=True``: pilco_particles_rollout_consistent, one posterior function per particle.  Its workspace is
    O(P H E n), so the particles run in chunks whose workspace fits ``max_ws_bytes`` (default: half the free device
    memory).  A particle's outputs do not depend on its batch, so the chunking does not change them."""
    x0, eps = dev(x0), dev(eps)
    if x0.dim() != 2 or eps.dim() != 3 or eps.shape[0] != x0.shape[0] or eps.shape[2] != x0.shape[1]:
        raise ValueError("particles_rollout: x0 must be [P,Ds] and eps [P,H,Ds], got %s and %s"
                         % (tuple(x0.shape), tuple(eps.shape)))
    if consistent:
        return _particles_rollout_consistent(dyn, policy_spec, reward_terms, x0, eps, mult_mu, max_ws_bytes)
    plan = ParticlePlan(dyn, policy_spec, reward_terms, x0.shape[0], eps.shape[1], mult_mu=mult_mu)
    plan.set_inputs(x0, eps)
    plan.launch()
    return plan.outputs()


def consistent_workspace_bytes(dyn, Ds, U, P, H):
    """pilco_particles_consistent_workspace_bytes of P particles over H steps (0: unsupported sizes)"""
    pr = _lib.Particles()
    pr.P, pr.H = int(P), int(H)
    pr.dyn = dyn.struct()
    pr.pol.Ds, pr.pol.U = int(Ds), int(U)
    return int(lib.pilco_particles_consistent_workspace_bytes(C.byref(pr)))


def _particles_rollout_consistent(dyn, policy_spec, reward_terms, x0, eps, mult_mu, max_ws_bytes):
    P, H = int(x0.shape[0]), int(eps.shape[1])
    Ds, U = int(policy_spec["Ds"]), int(policy_spec["U"])
    if max_ws_bytes is None:
        max_ws_bytes = torch.cuda.mem_get_info(device())[0] // 2
    fits = lambda p: 0 < consistent_workspace_bytes(dyn, Ds, U, p, H) <= max_ws_bytes
    if not fits(1):
        raise ValueError("particles_rollout: the consistent rollout of one particle (H=%d, n=%d) needs %d workspace "
                         "bytes, more than max_ws_bytes=%d" % (H, dyn.n, consistent_workspace_bytes(dyn, Ds, U, 1, H),
                                                               max_ws_bytes))
    lo = _largest_fitting(fits, 1, P)
    if lo == P:
        plan = ParticlePlan(dyn, policy_spec, reward_terms, P, H, mult_mu=mult_mu, consistent=True)
        plan.set_inputs(x0, eps)
        plan.launch()
        return plan.outputs()
    d = device()
    Hb = max(H, 1)
    out = (torch.empty((P, H + 1, Ds), dtype=F64, device=d), torch.empty((P, Hb, U), dtype=F64, device=d)[:, :H],
           torch.empty((P, Hb), dtype=F64, device=d)[:, :H], torch.empty((P, Hb), dtype=F64, device=d)[:, :H],
           torch.empty(P, dtype=F64, device=d))
    plan = None
    for p0 in range(0, P, lo):
        p1 = min(P, p0 + lo)
        if plan is None or plan.P != p1 - p0:
            plan = None                                     # free the previous chunk's workspace first
            plan = ParticlePlan(dyn, policy_spec, reward_terms, p1 - p0, H, mult_mu=mult_mu, consistent=True)
        plan.set_inputs(x0[p0:p1], eps[p0:p1])
        plan.launch()
        for o, c in zip(out, plan.outputs()):
            o[p0:p1].copy_(c)
    return out


class PredictPlan:
    """``PILCO.predict(m, S, n)`` as ONE graph launch: host moments -> device, n-step cascade (R = 1), final
    moments + reward + status -> pinned host memory.  Built once per (model, policy, reward, n) state by
    ``PILCO`` and replayed for every call with new initial moments (pilco/models/pilco.py:118-136)."""

    def __init__(self, dyn, policy_spec, reward_terms, Ds, n, mult_mu=0.0):
        d = device()
        self.Ds, self.n = int(Ds), int(n)
        Ds = self.Ds
        self.h_in = torch.zeros(Ds + Ds * Ds, dtype=F64).pin_memory()
        self.h_out = torch.zeros(Ds + Ds * Ds + 2, dtype=F64).pin_memory()       # [m | S | reward | info]
        self.d_in = torch.zeros(Ds + Ds * Ds, dtype=F64, device=d)
        self.d_out = torch.zeros(Ds + Ds * Ds + 2, dtype=F64, device=d)
        self.plan = RolloutPlan(dyn, policy_spec, reward_terms, np.zeros(Ds), np.eye(Ds), self.n, R=1, mult_mu=mult_mu)
        self._enqueue()                                    # eager warm-up (one-time kernel attributes)
        torch.cuda.synchronize()
        self.graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.graph):
            self._enqueue()

    def _enqueue(self):
        Ds, p = self.Ds, self.plan
        self.d_in.copy_(self.h_in, non_blocking=True)
        p.m0.copy_(self.d_in[:Ds])
        p.S0.copy_(self.d_in[Ds:].reshape(Ds, Ds))
        p.forward()
        out = self.d_out
        out[:Ds] = p.traj_m[0, -1]
        out[Ds:Ds + Ds * Ds] = p.traj_S[0, -1].reshape(-1)
        out[Ds + Ds * Ds] = p.reward[0]
        out[Ds + Ds * Ds + 1] = p.info[0].to(F64)
        self.h_out.copy_(out, non_blocking=True)

    def __call__(self, m, S):
        """m [Ds] / [1,Ds], S [Ds,Ds] (host) -> (m_n [1,Ds], S_n [Ds,Ds], reward [1,1]) host ndarrays"""
        Ds = self.Ds
        hin = self.h_in.numpy()
        hin[:Ds] = np.asarray(m, dtype=np.float64).reshape(Ds)
        hin[Ds:] = np.asarray(S, dtype=np.float64).reshape(Ds * Ds)
        self.graph.replay()
        torch.cuda.current_stream().synchronize()
        res = self.h_out.numpy()
        if res[-1] != 0.0:
            raise RuntimeError("moment-matching rollout failed: covariance not positive definite")
        return (res[:Ds].reshape(1, Ds).copy(), res[Ds:Ds + Ds * Ds].reshape(Ds, Ds).copy(),
                res[Ds + Ds * Ds].reshape(1, 1).copy())


class SplitRollout:
    """R independent rollouts as ``nsplit`` sub-batches on parallel streams inside ONE captured CUDA graph.

    Within a rollout the per-step kernels are strictly sequential, and several of them (state/policy glue,
    the D x D Cholesky stage) are latency-bound on a handful of SMs; running sub-batches on separate streams lets
    those overlap another sub-batch's tile kernel.  ``make_plan(lo, hi)`` must build the RolloutPlan of restarts
    [lo, hi)."""

    def __init__(self, make_plan, R, nsplit=4, backward=False):
        nsplit = max(1, min(int(nsplit), int(R)))
        bounds = [round(k * R / nsplit) for k in range(nsplit + 1)]
        self.slices = [(bounds[k], bounds[k + 1]) for k in range(nsplit) if bounds[k + 1] > bounds[k]]
        self.plans = [make_plan(lo, hi) for lo, hi in self.slices]
        self.backward = backward
        self.R = R
        for p in self.plans:                       # eager warm-up (one-time attributes, allocations)
            p.forward()
            if backward:
                p.backward()
        torch.cuda.synchronize()
        self.side = [torch.cuda.Stream() for _ in self.plans[1:]]
        self.graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.graph):
            cur = torch.cuda.current_stream()
            for st in self.side:
                st.wait_stream(cur)
            self._run(self.plans[0])
            for st, p in zip(self.side, self.plans[1:]):
                with torch.cuda.stream(st):
                    self._run(p)
            for st in self.side:
                cur.wait_stream(st)
        self.reward = torch.empty(R, dtype=F64, device=device())

    def _run(self, p):
        p.forward()
        if self.backward:
            p.backward()

    def replay(self):
        self.graph.replay()
        for (lo, hi), p in zip(self.slices, self.plans):
            self.reward[lo:hi].copy_(p.reward, non_blocking=True)
        return self.reward

    @property
    def info(self):
        return torch.cat([p.info for p in self.plans])


class ActionPlan:
    """Low-latency policy evaluation at a deterministic state: u = E[pi(x)] with s = 0, the call
    ``PILCO.compute_action`` makes once per control step when a learnt policy drives the plant
    (pilco/models/pilco.py:115-116, examples/utils.py:32-36).

    All buffers are allocated once; host->device copy of the state, the policy moment match
    (``pilco_mm_forward`` in deterministic-GP mode or ``pilco_linear_action``), ``pilco_squash_sin`` and the
    device->host copy of the action are captured in ONE CUDA graph, so a control step costs one graph launch and
    one stream synchronisation instead of ~10 allocations and 4-6 separate launches."""

    def __init__(self, policy_spec):
        d = device()
        self.Ds, self.U = int(policy_spec["Ds"]), int(policy_spec["U"])
        Ds, U = self.Ds, self.U
        self.kind = policy_spec["kind"]
        self.squash = bool(policy_spec.get("squash", True))
        self.h_x = torch.zeros((1, Ds), dtype=F64).pin_memory()
        self.h_out = torch.zeros((1, U + 1), dtype=F64).pin_memory()          # [action | info]
        self.m = torch.zeros((1, Ds), dtype=F64, device=d)
        self.s = torch.zeros((1, Ds, Ds), dtype=F64, device=d)
        self.M = torch.empty((1, U), dtype=F64, device=d)
        self.S = torch.empty((1, U, U), dtype=F64, device=d)
        self.V = torch.empty((1, Ds, U), dtype=F64, device=d)
        self.Mu = torch.empty((1, U), dtype=F64, device=d)
        self.Su = torch.empty((1, U, U), dtype=F64, device=d)
        self.Cq = torch.empty((1, U, U), dtype=F64, device=d)
        self.out = torch.zeros((1, U + 1), dtype=F64, device=d)
        self.info = torch.zeros(1, dtype=torch.int32, device=d)
        self.maxa = _max_action(policy_spec, U)
        if self.kind == _lib.POLICY_LINEAR:
            self.W, self.b = dev(policy_spec["W"]).reshape(U, Ds), dev(policy_spec["b"]).reshape(U)
        else:
            self.gp = policy_spec["gp"]
            if self.gp.batched:
                raise ValueError("ActionPlan evaluates ONE policy (unbatched parameters)")
            self.gps = self.gp.struct()
            self.wsb = lib.pilco_mm_workspace_bytes(self.gp.n, self.gp.D, self.gp.E, 1)
            self.ws = torch.empty(self.wsb // 8, dtype=F64, device=d)
        self._enqueue()                                    # eager warm-up (one-time kernel attributes)
        torch.cuda.synchronize()
        self.graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.graph):
            self._enqueue()

    def _enqueue(self):
        U = self.U
        self.info.zero_()                                  # the kernels only OR failure bits into info
        self.m.copy_(self.h_x, non_blocking=True)
        if self.kind == _lib.POLICY_LINEAR:
            check(lib.pilco_linear_action(self.Ds, U, 1, ptr(self.W), 0, ptr(self.b), 0, ptr(self.m), ptr(self.s),
                                          ptr(self.M), ptr(self.S), ptr(self.V), stream_ptr()), "linear_action")
        else:
            check(lib.pilco_mm_forward(C.byref(self.gps), 1, ptr(self.m), ptr(self.s), ptr(self.M), ptr(self.S),
                                       ptr(self.V), ptr(self.info), ptr(self.ws), self.wsb, stream_ptr()), "mm_forward")
        if self.squash:
            check(lib.pilco_squash_sin(U, 1, ptr(self.M), ptr(self.S), ptr(self.maxa), ptr(self.Mu), ptr(self.Su),
                                       ptr(self.Cq), stream_ptr()), "squash_sin")
            self.out[:, :U] = self.Mu
        else:
            self.out[:, :U] = self.M
        self.out[:, U] = self.info.to(F64)
        self.h_out.copy_(self.out, non_blocking=True)

    def __call__(self, x):
        """x [Ds] or [1,Ds] (host) -> action [1,U] (host ndarray)"""
        self.h_x.copy_(torch.as_tensor(np.asarray(x, dtype=np.float64).reshape(1, self.Ds)))
        self.graph.replay()
        torch.cuda.current_stream().synchronize()
        res = self.h_out.numpy()
        if res[0, self.U] != 0.0:
            raise RuntimeError("policy moment match failed (info=%d)" % int(res[0, self.U]))
        return res[:, :self.U].copy()
