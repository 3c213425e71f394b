"""Device-side plumbing: PyTorch owns every fp64 device buffer, the C ABI does the math.

Each function mirrors one C entry point; arguments are numpy arrays or CUDA tensors, results are
CUDA tensors (the API classes convert to host arrays at the boundary).  There is no CPU path:
``device()`` raises when no CUDA device is present.
"""
import ctypes as C
import gc

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
    # with iK, the next B*E*ldw*ldw doubles = R = L^-1 (what gp_append extends)
    gp.R = ws[B * E * ldk * ldk:2 * B * E * ldk * ldk].view(iK.shape) if need_iK else None
    gp.Y, gp.sn2 = Y, sn2
    return gp


def gp_append(gp, X, Y):
    """pilco_gp_append_tri: the factorised (unbatched, exact-GP) model ``gp`` with rows appended to its data and unchanged
    hyper-parameters.  ``X`` [n1,D], ``Y`` [n1,E] hold the old rows first.  Returns a NEW DeviceGP (n changes, so do the
    padded leading dimension and every workspace size downstream): the old model's triangular inverse R = L^-1 is
    extended by one block row in O(n^2 k), no Cholesky factorisation of the full matrix is done."""
    if gp.batched or gp.iK is None or gp.mode != 0 or getattr(gp, "R", None) is None:
        raise ValueError("gp_append needs an unbatched exact-GP model with its inverse and triangular inverse")
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
    R = torch.empty((E, ldk, ldk), dtype=F64, device=d)
    info = torch.zeros(1, dtype=torch.int32, device=d)
    wsb = lib.pilco_gp_append_tri_workspace_bytes(n0, k, E)
    ws = torch.empty(wsb // 8, dtype=F64, device=d)
    check(lib.pilco_gp_append_tri(n0, k, D, E, ptr(X), ptr(Y), ptr(gp.ell), ptr(gp.sf2), ptr(gp.sn2),
                              ptr(gp.R), gp.ldk, ptr(gp.iK), gp.ldk, ptr(R), ldk, ptr(iK), ldk, ptr(beta), ptr(info),
                              ptr(ws), wsb, stream_ptr()),
          "gp_append")
    new = DeviceGP(X, gp.ell, gp.sf2, beta, iK, ldk, mode=0)
    new.info = info
    new.R = R
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


def predict_samples_workspace_bytes(gp, T, S, ne=None, full_cov=True):
    """pilco_gp_predict_samples_workspace_bytes (0: unsupported sizes)"""
    ne = gp.E if ne is None else int(ne)
    return int(lib.pilco_gp_predict_samples_workspace_bytes(gp.n, gp.D, ne, int(T), int(S), 1 if full_cov else 0))


def gp_predict_samples(gp, Xnew, eps, e0=0, ne=None, full_cov=True, jitter=1e-6, max_ws_bytes=None):
    """pilco_gp_predict_samples: posterior function samples of outputs e0 .. e0+ne-1 of the factorised model ``gp`` at
    Xnew [T,D] given standard normals eps [S,T,ne] -> (samples [S,T,ne], info [ne]) device tensors; info[e] != 0 where
    the covariance + jitter I of output e is not positive definite.  ``full_cov=False`` draws each point independently
    from its marginal.  A workspace above ``max_ws_bytes`` (default: half the free device memory) is a ValueError that
    names the bytes needed and the largest T that would fit, raised before anything is allocated."""
    Xs, eps = dev(Xnew), dev(eps)
    if Xs.dim() != 2 or Xs.shape[1] != gp.D:
        raise ValueError("gp_predict_samples: Xnew must be [T, %d], got %s" % (gp.D, tuple(Xs.shape)))
    T = int(Xs.shape[0])
    ne = gp.E - int(e0) if ne is None else int(ne)
    if eps.dim() != 3 or eps.shape[1:] != (T, ne):
        raise ValueError("gp_predict_samples: eps must be [S, %d, %d], got %s" % (T, ne, tuple(eps.shape)))
    S = int(eps.shape[0])
    if T < 1 or ne < 1 or S < 1:
        raise ValueError("gp_predict_samples: needs T, ne, S >= 1 (T=%d, ne=%d, S=%d)" % (T, ne, S))
    wsb = predict_samples_workspace_bytes(gp, T, S, ne, full_cov)
    if wsb == 0:
        raise ValueError("gp_predict_samples: unsupported sizes (n=%d, D=%d, ne=%d, T=%d, S=%d)" % (gp.n, gp.D, ne, T, S))
    _largest_fitting(lambda t: predict_samples_workspace_bytes(gp, t, S, ne, full_cov), T, max_ws_bytes,
                     "gp_predict_samples: %d samples of %d outputs at T=%d points (full_cov=%s)"
                     % (S, ne, T, bool(full_cov)), whole="T")
    d = device()
    samples = torch.empty((S, T, ne), dtype=F64, device=d)
    info = torch.empty(ne, dtype=torch.int32, device=d)
    ws = torch.empty(wsb // 8, dtype=F64, device=d)
    g = gp.struct()
    check(lib.pilco_gp_predict_samples(C.byref(g), int(e0), ne, T, S, ptr(Xs), ptr(eps), ptr(samples),
                                       1 if full_cov else 0, float(jitter), ptr(info), ptr(ws), wsb, stream_ptr()),
          "gp_predict_samples")
    return samples, info


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


def angles_struct(angle_dims, Ds):
    """``pilco_angles`` for the angular state dimensions ``angle_dims`` of a state of dimension ``Ds`` (None or empty:
    no angles -> None).  ValueError for a dimension out of range or repeated."""
    if angle_dims is None or len(angle_dims) == 0:
        return None
    dims = [int(a) for a in angle_dims]
    if len(set(dims)) != len(dims) or any(a < 0 or a >= Ds for a in dims):
        raise ValueError("angle_dims %s: expected distinct indices into a state of dimension %d" % (list(angle_dims), Ds))
    ang = _lib.Angles()
    ang.A = len(dims)
    for i, a in enumerate(dims):
        ang.dims[i] = a
    return ang


def trig_feature_map(x, angle_dims):
    """phi(x) on the host (numpy, last axis = state): the pass-through dimensions in increasing order, then
    sin, cos of every angle in ``angle_dims`` order -- the map the device applies to the state Gaussian."""
    x = np.asarray(x, dtype=np.float64)
    Ds = x.shape[-1]
    dims = [int(a) for a in (angle_dims or [])]
    keep = [j for j in range(Ds) if j not in dims]
    parts = [x[..., keep]]
    for a in dims:
        parts += [np.sin(x[..., a:a + 1]), np.cos(x[..., a:a + 1])]
    return np.concatenate(parts, axis=-1)


def trig_moments(m, s, angle_dims):
    """pilco_trig_moments: moments of phi(x) for x ~ N(m [R,Ds], s [R,Ds,Ds]) -> M [R,Dh], S [R,Dh,Dh] and
    C = inv(s) cov(x, phi) [R,Ds,Dh] (Dh = Ds + len(angle_dims))."""
    m, s = dev(m), dev(s)
    R, Ds = m.shape
    ang = angles_struct(angle_dims, Ds)
    Dh = Ds + (ang.A if ang is not None else 0)
    d = device()
    M = torch.empty((R, Dh), dtype=F64, device=d)
    S = torch.empty((R, Dh, Dh), dtype=F64, device=d)
    Cx = torch.empty((R, Ds, Dh), dtype=F64, device=d)
    check(lib.pilco_trig_moments(Ds, R, C.byref(ang) if ang is not None else None, ptr(m), ptr(s), ptr(M), ptr(S),
                                 ptr(Cx), stream_ptr()), "trig_moments")
    return M, S, Cx


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
    elif pol.kind == _lib.POLICY_RBF:
        rbf = policy_spec["gp"]
        pol.rbf = rbf.struct()
    return max_action, W, b, rbf


MLP_MAX_WIDTH = 64                                       # the widest hidden layer the MLP kernels take


def mlp_theta_size(Ds, U, hidden):
    """the length of a tanh MLP's flat parameter vector: A_1 [w1, Ds+1], (A_2 [w2, w1+1],) A_out [U, w_L+1]"""
    widths = [int(Ds)] + [int(w) for w in hidden]
    return sum(widths[l + 1] * (widths[l] + 1) for l in range(len(hidden))) + int(U) * (widths[-1] + 1)


def _is_mlp(policy_spec):
    return isinstance(policy_spec, dict) and policy_spec.get("kind") == _lib.POLICY_MLP


def _refuse_mlp(policy_spec, what):
    """the moment-matching plans take no MLP spec (it has no closed-form moments): ValueError before any allocation"""
    if _is_mlp(policy_spec):
        raise ValueError("%s: an MLP policy runs in the particle rollouts only (ParticlePlan, ConsistentGradPlan, "
                         "particles_rollout); moment matching has no closed form for it" % what)


def _particle_mlp(policy_spec, what, R=1, angles=None, measurement_noise=None, schedule=False, estimator="pathwise"):
    """An MLP spec's refusals and checks for the particle plans, before any allocation (ValueError): no angles,
    measurement noise, schedule or score estimator; 1 or 2 hidden layers of 1 .. 64 units; theta [n_theta] or
    [R, n_theta].  Returns (L, widths, n_theta, batched) for an MLP spec, else None."""
    if not _is_mlp(policy_spec):
        return None
    for on, feat in ((angles is not None and len(angles) > 0, "angles"),
                     (measurement_noise is not None, "measurement_noise"), (bool(schedule), "schedule=True"),
                     (estimator == "score", "estimator='score'")):
        if on:
            raise ValueError("%s: an MLP policy does not combine with %s" % (what, feat))
    hidden = tuple(int(w) for w in policy_spec["hidden"])
    if len(hidden) not in (1, 2) or any(w < 1 or w > MLP_MAX_WIDTH for w in hidden):
        raise ValueError("%s: an MLP policy has 1 or 2 hidden layers of 1 .. %d units, got hidden=%s"
                         % (what, MLP_MAX_WIDTH, hidden))
    n = mlp_theta_size(policy_spec["Ds"], policy_spec["U"], hidden)
    shape = tuple(np.shape(policy_spec["theta"]))
    if shape not in ((n,), (int(R), n)) or (int(R) > 1 and shape != (int(R), n)):
        raise ValueError("%s: the MLP (Ds=%d, hidden=%s, U=%d) has %d parameters: theta must be [%s%d], got %s"
                         % (what, int(policy_spec["Ds"]), hidden, int(policy_spec["U"]), n,
                            "%d, " % int(R) if int(R) > 1 else "R?, ", n, shape))
    return len(hidden), hidden, n, len(shape) == 2


def _schedule_check(policy_spec, H, schedule):
    """A scheduled spec (a time-varying linear policy: W [R?,Hw,U,Ds], b [R?,Hw,U]) against RolloutPlan's ``schedule``
    and horizon H, before any allocation: ValueError.  Returns the (batched, Hw) of a scheduled spec, else None."""
    if not schedule:
        if isinstance(policy_spec, dict) and policy_spec.get("schedule", False):
            raise ValueError("the policy spec is a time-varying linear policy (a schedule): pass schedule=True")
        return None
    if policy_spec["kind"] != _lib.POLICY_LINEAR:
        raise ValueError("schedule=True takes a linear policy (time-varying W_t, b_t); an RBF policy has no schedule")
    U, Ds = int(policy_spec["U"]), int(policy_spec["Ds"])
    Ws, bs = np.shape(policy_spec["W"]), np.shape(policy_spec["b"])
    if len(Ws) not in (3, 4) or Ws[-2:] != (U, Ds) or bs != Ws[:-2] + (U,):
        raise ValueError("schedule=True: expected W [R?, H, U=%d, Ds=%d] and b [R?, H, U], got W %s, b %s"
                         % (U, Ds, Ws, bs))
    Hw = int(Ws[-3])
    if Hw < int(H):
        raise ValueError("schedule=True: the schedule has %d steps, fewer than the rollout's H=%d" % (Hw, int(H)))
    return len(Ws) == 4, Hw


def _particle_schedule(policy_spec, H, schedule, what):
    """``_schedule_check`` for the particle plans, before any allocation: a scheduled spec without ``schedule=True`` is
    a ValueError that names ``what``"""
    if not schedule and isinstance(policy_spec, dict) and policy_spec.get("schedule", False):
        raise ValueError("%s: the policy spec is a time-varying linear policy (a schedule): pass schedule=True" % what)
    return _schedule_check(policy_spec, H, schedule)


def _reward_count(reward_terms):
    if len(reward_terms) > 8:
        raise ValueError("at most 8 reward terms per rollout, got %d" % len(reward_terms))


def _fill_rewards(desc, reward_terms):
    """Fill ``desc.n_rewards`` and ``desc.rewards`` from reward-term dicts (``desc.pol`` already filled); returns the
    device tensors [(W, t)] they point to.  The shapes of a joint state-action term are checked against the policy
    here, before any device work: ValueError."""
    rw = []
    _reward_count(reward_terms)
    desc.n_rewards = len(reward_terms)
    Ds, U = int(desc.pol.Ds), int(desc.pol.U)
    for k, rt in enumerate(reward_terms):
        if rt["kind"] in _lib.JOINT_REWARDS:
            D = Ds + U
            if (rt.get("state_dim", Ds), rt.get("control_dim", U)) != (Ds, U):
                raise ValueError("reward term %d is built for state_dim=%s, control_dim=%s; the policy has %d and %d"
                                 % (k, rt.get("state_dim"), rt.get("control_dim"), Ds, U))
            wshape = (D, D) if rt["kind"] == _lib.REWARD_EXP_SA else (D,)
            if np.shape(rt["W"]) != wshape or (rt["kind"] == _lib.REWARD_EXP_SA and np.shape(rt.get("t")) != (D,)):
                raise ValueError("reward term %d on the joint [x, u]: W must be %s%s for state_dim=%d, control_dim=%d, "
                                 "got W %s, t %s" % (k, list(wshape), " and t [%d]" % D if len(wshape) == 2 else "", Ds, U,
                                                     np.shape(rt["W"]), np.shape(rt.get("t"))))
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

    def __init__(self, dyn, policy_spec, reward_terms, m0, S0, H, R=1, mult_mu=0.0, grad=False, angles=None,
                 exploration=None, measurement_noise=None, schedule=False):
        """``grad=True``: the forward cascade runs the TAPED dynamics tile pass (pilco_rollout.tape), so that
        ``backward()`` needs no recomputation; without it ``backward()`` still works (recomputing path).

        ``angles``: angular state dimensions (pilco_rollout_angles_*).  The state dimension is then the dynamics GP's
        output count E; the policy (``policy_spec["Ds"]``) and the joint state-action terms see phi(x) of dimension
        Dh = E + len(angles), the dynamics GP [phi(x), u].

        ``exploration``: a float b selects the exploration objective (pilco_rollout_explore_*, DESIGN.md section 21):
        ``reward`` = sum_t (E[r_t] + b sigma_t) (+ the multiplicative channel's term), sigma_t^2 = sum_k c_k^2 Var[r_k]
        over the additive terms, written to ``step_var`` [R, max(H,1)]; its gradient is ``backward()``'s.  b = 0.0 fills
        ``step_var`` and leaves every other output and gradient as without exploration.  ``None``: no exploration.
        A non-finite b, or an additive box term (it has no variance closed form), is a ValueError.

        ``measurement_noise``: variances v [Ds] >= 0 of a noisy state measurement z = x + nu, nu ~ N(0, diag(v)), that
        the policy sees in place of the state (pilco_rollout_noisy_*, DESIGN.md section 22): the policy is moment-matched
        at N(m, S + diag(v)) (phi of it with angles), the dynamics and the rewards see the true state's moments.  Ds is
        the raw state dimension.  ``None``: the policy sees the state.

        ``schedule=True``: a time-varying linear policy u_t = sq(W_t x + b_t) (pilco_rollout_scheduled_*, DESIGN.md
        section 27); the spec's W is [Hw, U, Ds] or [R, Hw, U, Ds] and b [Hw, U] or [R, Hw, U], Hw >= H (step t < H reads
        W[..., t, :, :]).  ``backward()`` then returns the per-step cotangents W [R, H, U, Ds] and b [R, H, U].  An RBF
        spec or Hw < H is a ValueError."""
        _refuse_mlp(policy_spec, "RolloutPlan")
        sched = _schedule_check(policy_spec, H, schedule)
        b = None
        if exploration is not None:
            b = float(exploration)
            if not np.isfinite(b):
                raise ValueError("exploration: b must be finite, got %r" % exploration)
            for k, rt in enumerate(reward_terms):
                if rt["kind"] == _lib.REWARD_BOX and int(rt.get("channel", _lib.CHANNEL_ADD)) == _lib.CHANNEL_ADD:
                    raise ValueError("exploration: reward term %d is an additive box term, which has no variance closed "
                                     "form; use it in the multiplicative channel (SafePILCO) or leave exploration off"
                                     % k)
        nz_var = None
        if measurement_noise is not None:
            nz_var = np.asarray(measurement_noise, dtype=np.float64).reshape(-1)
            if not np.all(np.isfinite(nz_var)) or np.any(nz_var < 0.0):
                raise ValueError("measurement_noise: the variances must be finite and >= 0, got %r" % nz_var)
        d = device()
        self.dyn = dyn
        self.R, self.H = int(R), int(H)
        self.Ds, self.U = policy_spec["Ds"], policy_spec["U"]
        self.ang = None
        if angles is not None and len(angles) > 0:
            self.Ds = int(dyn.struct().E)
            self.ang = angles_struct(angles, self.Ds)
            Dh = self.Ds + self.ang.A
            if int(policy_spec["Ds"]) != Dh:
                raise ValueError("with %d angle dimension(s) the policy must take %d inputs (phi(x)), got %d"
                                 % (self.ang.A, Dh, int(policy_spec["Ds"])))
        self.nz = None
        if nz_var is not None:
            if nz_var.shape[0] != int(self.Ds):
                raise ValueError("measurement_noise: expected %d variances (the state dimension), got %d"
                                 % (int(self.Ds), nz_var.shape[0]))
            self.nz = _lib.ObsNoise()
            self.nz.var[:len(nz_var)] = nz_var.tolist()
        self.keep = [dyn, policy_spec, reward_terms]            # keep device tensors alive
        ro = _lib.Rollout()
        ro.R, ro.H = self.R, self.H
        ro.dyn = dyn.struct()
        self.max_action, self.W, self.b, self.rbf = _fill_policy(ro.pol, policy_spec,
                                                                 batched=None if sched is None else False)
        self.sch = None
        if sched is not None:                                   # step t reads W[..., t, :, :], b[..., t, :]
            U, Ds = int(policy_spec["U"]), int(policy_spec["Ds"])
            ro.pol.W_bs, ro.pol.b_bs = (sched[1] * U * Ds, sched[1] * U) if sched[0] else (0, 0)
            self.sch = _lib.PolicySchedule(U * Ds, U)
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
        self.ex, self.step_var = None, None
        if b is not None:
            self.step_var = torch.zeros((self.R, max(self.H, 1)), dtype=F64, device=d)
            self.ex = _lib.Exploration(b, self.step_var.data_ptr())
        wsb = self._call("workspace_bytes", ro)
        self.ws = torch.empty(max(wsb // 8, 2), dtype=F64, device=d)
        ro.ws, ro.ws_bytes = self.ws.data_ptr(), wsb
        self.tape = None
        if grad and self.H > 0:
            tb = lib.pilco_rollout_tape_bytes(C.byref(ro))
            if tb:                                              # (0: more than 2048 centres -> recomputing backward)
                self.tape = torch.empty(tb // 8, dtype=F64, device=d)
                ro.tape, ro.tape_bytes = self.tape.data_ptr(), tb
        self.ro = ro

    def _ang_ref(self):
        return C.byref(self.ang) if self.ang is not None else None

    def _ex_ref(self):
        return C.byref(self.ex) if self.ex is not None else None

    def _nz_ref(self):
        return C.byref(self.nz) if self.nz is not None else None

    def _call(self, what, ro, *rest):
        """pilco_rollout_noisy_<what>, or with a schedule pilco_rollout_scheduled_<what>"""
        args = (C.byref(ro), self._ang_ref(), self._ex_ref(), self._nz_ref())
        if self.sch is not None:
            return getattr(lib, "pilco_rollout_scheduled_" + what)(*args, C.byref(self.sch), *rest)
        return getattr(lib, "pilco_rollout_noisy_" + what)(*args, *rest)

    def forward(self):
        check(self._call("forward", self.ro, stream_ptr()),
              "rollout_noisy_forward" if self.sch is None else "rollout_scheduled_forward")
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
        Linear: {'W': [R,U,Ds], 'b': [R,U]} (with a schedule per step: [R,H,U,Ds], [R,H,U]);
        RBF: {'X': [R,bf,Ds], 'Y': [R,bf,U], 'ell': [R,U,Ds]}."""
        d = device()
        if not hasattr(self, "grad"):
            g = _lib.RolloutGrad()
            R, Ds = self.R, self.Ds
            self.gbuf = _policy_grad_buffers(g, self.ro.pol, self.rbf, (R,) if self.sch is None else (R, self.H))
            self.gbuf["m0"] = torch.empty((R, Ds), dtype=F64, device=d)
            self.gbuf["S0"] = torch.empty((R, Ds, Ds), dtype=F64, device=d)
            g.gm0, g.gS0 = self.gbuf["m0"].data_ptr(), self.gbuf["S0"].data_ptr()
            wsb = self._call("bwd_workspace_bytes", self.ro)
            self.bws = torch.empty(max(wsb // 8, 2), dtype=F64, device=d)
            g.ws, g.ws_bytes = self.bws.data_ptr(), wsb
            self.grad = g
        check(self._call("backward", self.ro, C.byref(self.grad), stream_ptr()),
              "rollout_noisy_backward" if self.sch is None else "rollout_scheduled_backward")
        return self.gbuf


# (policy family, sampler, call) -> the C rollout and its size query, pilco_particles_<stem>_rollout and
# pilco_particles_<stem>_workspace_bytes.  Families: "plain" (linear or RBF), "scheduled" (a time-varying linear policy,
# DESIGN.md section 28) and "mlp" (section 29); samplers: "step", "consistent" (section 14), "resampled" (section 26) and
# "features" (section 30); calls: "forward", the gradients "pathwise" and "score", and "batch", R policies forward only
# (sections 31 and 33).  Each row is the most general entry point of its kind, given NULL for the angles, noise or
# exploration a plan lacks; the pathwise call of an unbatched plan is the batched one at R = 1.
PARTICLE_ENTRY_POINTS = {key: ("pilco_particles_%s_rollout" % stem, "pilco_particles_%s_workspace_bytes" % stem)
                         for key, stem in {
    ("plain", "step", "forward"): "noisy",
    ("plain", "consistent", "forward"): "noisy_consistent",
    ("plain", "step", "pathwise"): "explore_batch_grad",
    ("plain", "consistent", "pathwise"): "explore_consistent_grad",
    ("plain", "step", "score"): "noisy_score_grad",
    ("plain", "consistent", "score"): "consistent_score_grad",
    ("plain", "resampled", "forward"): "resampled",
    ("plain", "resampled", "pathwise"): "resampled_grad",
    ("plain", "features", "forward"): "features",
    ("plain", "features", "pathwise"): "features_grad",
    ("plain", "step", "batch"): "batch",
    ("plain", "consistent", "batch"): "consistent_batch",
    ("scheduled", "step", "forward"): "scheduled",
    ("scheduled", "consistent", "forward"): "scheduled_consistent",
    ("scheduled", "step", "pathwise"): "scheduled_batch_grad",
    ("scheduled", "consistent", "pathwise"): "scheduled_consistent_grad",
    ("scheduled", "step", "score"): "scheduled_score_grad",
    ("scheduled", "consistent", "score"): "scheduled_consistent_score_grad",
    ("scheduled", "resampled", "forward"): "scheduled_resampled",
    ("scheduled", "resampled", "pathwise"): "scheduled_resampled_grad",
    ("scheduled", "step", "batch"): "scheduled_batch",
    ("scheduled", "consistent", "batch"): "scheduled_consistent_batch",
    ("mlp", "step", "forward"): "mlp",
    ("mlp", "consistent", "forward"): "mlp_consistent",
    ("mlp", "step", "pathwise"): "mlp_batch_grad",
    ("mlp", "consistent", "pathwise"): "mlp_consistent_grad",
    ("mlp", "resampled", "forward"): "mlp_resampled",
    ("mlp", "resampled", "pathwise"): "mlp_resampled_grad",
    ("mlp", "features", "forward"): "mlp_features",
    ("mlp", "features", "pathwise"): "mlp_features_grad",
    ("mlp", "step", "batch"): "mlp_batch",
    ("mlp", "consistent", "batch"): "mlp_consistent_batch",
}.items()}


def _view(keep, key):
    """the rows of PARTICLE_ENTRY_POINTS that keep(family, sampler, call) selects, under key(family, sampler, call),
    their names after "pilco_particles_": the per-family tables that callers index"""
    return {key(*k): tuple(n[len("pilco_particles_"):] for n in v) for k, v in PARTICLE_ENTRY_POINTS.items() if keep(*k)}


_SAMPLER_KEY = {"step": False, "consistent": True}             # the views' sampler keys: the consistent flag, or the name
PARTICLE_CALLS = _view(lambda f, s, c: f == "plain" and s != "features" and c != "batch",
                       lambda f, s, c: (_SAMPLER_KEY.get(s, s), c))
PARTICLE_FEATURE_CALLS = _view(lambda f, s, c: f == "plain" and s == "features", lambda f, s, c: (s, c))
PARTICLE_SCHEDULED_CALLS = _view(lambda f, s, c: f == "scheduled" and c != "batch",
                                 lambda f, s, c: (_SAMPLER_KEY.get(s, s), c))
PARTICLE_MLP_CALLS = _view(lambda f, s, c: f == "mlp" and c != "batch", lambda f, s, c: (_SAMPLER_KEY.get(s, s), c))
PARTICLE_BATCH_CALLS = _view(lambda f, s, c: f == "scheduled" and c == "batch", lambda f, s, c: s == "consistent")
PARTICLE_STATIONARY_BATCH_CALLS = _view(lambda f, s, c: f != "scheduled" and c == "batch",
                                        lambda f, s, c: (f == "mlp", s == "consistent"))

# the slot each argtype of a particle entry point takes (a rollout's final c_dp is the stream, which each launch passes)
_SLOTS = {C.POINTER(_lib.Particles): "pr", C.POINTER(_lib.Angles): "ang", C.POINTER(_lib.ParticlesNoise): "nz",
          C.POINTER(_lib.Exploration): "ex", C.POINTER(_lib.PolicySchedule): "sch", C.POINTER(_lib.Mlp): "mlp",
          C.POINTER(_lib.ParticlesResample): "rs", C.POINTER(_lib.FeatureDraws): "fd",
          C.POINTER(_lib.ParticlesGrad): "grad", C.c_int: "R", _lib.c_dp: "value"}


def particle_args(name, **slots):
    """The arguments of the particle entry point ``name`` before its stream, in the order of its ``_lib.SIGNATURES``
    argtypes (the header's): the structs ``pr`` (the pilco_particles description), ``ang``, ``nz``, ``ex``, ``sch``,
    ``mlp``, ``rs``, ``fd`` and ``grad`` by reference, NULL where ``slots`` has none; ``R`` for the c_int; ``value``
    for a c_dp before the stream."""
    res, types = _lib.SIGNATURES[name]
    args = [slots.get(_SLOTS[t]) for t in (types[:-1] if res is C.c_int else types)]
    return tuple(C.byref(a) if isinstance(a, C.Structure) else a for a in args)


class _Entry:
    """Row ``key`` of PARTICLE_ENTRY_POINTS with its arguments bound once (``particle_args``): ``query()`` is the
    workspace size, a call enqueues the rollout on the current stream."""

    def __init__(self, key, **slots):
        run, query = PARTICLE_ENTRY_POINTS[key]
        self.name = run[len("pilco_"):]
        self.run, self.args = getattr(lib, run), particle_args(run, **slots)
        self.size, self.size_args = getattr(lib, query), particle_args(query, **slots)

    def query(self):
        return int(self.size(*self.size_args))

    def __call__(self):
        check(self.run(*self.args, stream_ptr()), self.name)


def _policy_width(dyn, spec, angles, what):
    """(E, the pilco_angles of ``angles`` or None): the policy takes the state's E dimensions and one more per angle
    (phi(x)); ValueError otherwise, before any allocation"""
    E = int(dyn.struct().E)
    ang = angles_struct(angles, E) if angles is not None and len(angles) > 0 else None
    A = ang.A if ang is not None else 0
    if int(spec["Ds"]) != E + A:
        raise ValueError("%s: with %d angle dimension(s) the policy must take %d inputs (phi(x)), got %d"
                         % (what, A, E + A, int(spec["Ds"])))
    return E, ang


def _noise_struct(measurement_noise, E):
    """the pilco_particles_noise of the measurement variances (None: no noise; ``_particle_noise``'s refusals).  Its
    nu is a placeholder, which the size queries check but do not read, until ``_buffers`` points it at the plan's nu"""
    v = _particle_noise(measurement_noise, E)
    if v is None:
        return None
    nz = _lib.ParticlesNoise()
    for i, x in enumerate(v):
        nz.v.var[i] = float(x)
    nz.nu = 16
    return nz


class _Particles:
    """What the particle plans share: one ``pilco_particles`` description ``pr``, the structs the entry points take
    beside it and the device tensors they point to.  ``_structs`` allocates nothing, so that a plan can query sizes and
    refuse before any allocation; ``_buffers`` allocates."""

    ang = nz = ex = sch = mlp = rs = fd = grad = None
    R = 1

    def _structs(self, dyn, spec, P, H, ang=None, nz=None, schedule=False, mlp=None, batched=False):
        """the description with what the size queries read (sizes, model, the policy's kind and widths, an RBF
        policy's model), the schedule (step t reads W[t], b[t]) and the MLP (``_particle_mlp``'s (L, widths,
        n_theta, _); theta strides by n_theta when ``batched``)"""
        self.keep = [dyn, spec]                                 # keep device tensors alive
        self.P, self.H, self.E, self.U = int(P), int(H), int(dyn.struct().E), int(spec["U"])
        self.ang, self.nz = ang, nz
        pr = self.pr = _lib.Particles()
        pr.P, pr.H = self.P, self.H
        pr.dyn = dyn.struct()
        pr.pol.kind, pr.pol.Ds, pr.pol.U = spec.get("kind", _lib.POLICY_LINEAR), int(spec["Ds"]), self.U
        if pr.pol.kind == _lib.POLICY_RBF:
            pr.pol.rbf = spec["gp"].struct()
        if schedule:
            self.sch = _lib.PolicySchedule(self.U * pr.pol.Ds, self.U)
        if mlp is not None:
            L, hidden, self.n_theta, _ = mlp
            self.mlp = _lib.Mlp(L, (C.c_int * 2)(hidden[0], hidden[-1] if L == 2 else 0), None,
                                self.n_theta if batched else 0, None)

    def _buffers(self, spec, reward_terms, mult_mu, lead, batched):
        """the policy's device tensors (``_fill_policy``; a batched schedule strides by its steps, an MLP's theta is
        [R?, n_theta]), the reward terms and mult_mu, the inputs x0 [P,E], eps [P,Hb,E] and with measurement noise nu
        [P,Hb,E], shared by the policies, and the outputs traj [*lead,P,H+1,E], act_buf [*lead,P,Hb,U], rew_buf and
        risk_buf [*lead,P,Hb] and ret [*lead,P] (Hb = max(H, 1): H = 0 still has addresses)"""
        pr, d = self.pr, device()
        P, H, Hb, E, U = self.P, self.H, max(self.H, 1), self.E, self.U
        self.keep.append(reward_terms)
        self.max_action, self.W, self.b, self.rbf = _fill_policy(pr.pol, spec, batched)
        if self.sch is not None and batched:                    # W [R,Hw,U,Ds], b [R,Hw,U]
            pr.pol.W_bs, pr.pol.b_bs = self.W[0].numel(), self.b[0].numel()
        if self.mlp is not None:
            self.theta = dev(spec["theta"]).reshape(*((self.R,) if batched else ()), self.n_theta)
            self.mlp.theta = self.theta.data_ptr()
        self.rw = _fill_rewards(pr, reward_terms)
        pr.mult_mu = float(mult_mu)
        mk = lambda *shape: torch.zeros(shape, dtype=F64, device=d)
        self.x0, self.eps_buf = mk(P, E), mk(P, Hb, E)
        self.traj, self.act_buf = mk(*lead, P, H + 1, E), mk(*lead, P, Hb, U)
        self.rew_buf, self.risk_buf, self.ret = mk(*lead, P, Hb), mk(*lead, P, Hb), mk(*lead, P)
        pr.x0, pr.eps = self.x0.data_ptr(), self.eps_buf.data_ptr()
        pr.traj, pr.act = self.traj.data_ptr(), self.act_buf.data_ptr()
        pr.step_reward, pr.step_risk, pr.ret = self.rew_buf.data_ptr(), self.risk_buf.data_ptr(), self.ret.data_ptr()
        if self.nz is not None:
            self.nu_buf = mk(P, Hb, E)
            self.nz.nu = self.nu_buf.data_ptr()

    def _ang_ref(self):
        return C.byref(self.ang) if self.ang is not None else None

    def _nz_ref(self):
        return C.byref(self.nz) if self.nz is not None else None

    def _entry(self, key, **slots):
        """row ``key`` of PARTICLE_ENTRY_POINTS bound to this description's structs (``slots`` replace them)"""
        return _Entry(key, **dict(dict(pr=self.pr, ang=self.ang, nz=self.nz, ex=self.ex, sch=self.sch, mlp=self.mlp,
                                       rs=self.rs, fd=self.fd, grad=self.grad, R=self.R), **slots))


def _largest_fitting(need, n, max_ws_bytes, what, whole=None):
    """The largest count c in 1 .. n whose workspace of need(c) bytes fits max_ws_bytes (default: half the free device
    memory), by bisection: need(c) grows with c and is 0 for sizes the call does not support.  Not even c = 1 fitting
    is a ValueError that names ``what`` and the bytes needed.  ``whole`` (the count's name): all n must fit, and the
    ValueError also names the largest count that would."""
    if max_ws_bytes is None:
        max_ws_bytes = torch.cuda.mem_get_info(device())[0] // 2
    fits = lambda c: 0 < need(c) <= max_ws_bytes
    lo, hi = (n, n) if fits(n) else (0, n - 1)
    while lo < hi:
        mid = (lo + hi + 1) // 2
        lo, hi = (mid, hi) if fits(mid) else (lo, mid - 1)
    if lo < (n if whole else 1):
        raise ValueError("%s: need %d workspace bytes, more than max_ws_bytes=%d (half the free device memory by "
                         "default)%s" % (what, need(n if whole else 1), max_ws_bytes,
                                         "; %s=%d would fit" % (whole, lo) if whole else ""))
    return lo


class FeatureDraws:
    """What ``feature_draws`` returns: the device tensors of P particles' function draws (DESIGN.md section 30),
    omega [E,F,D], w [P,E,2F] and v [P,E,n].  A plan draws once and rolls out many times on them."""

    def __init__(self, F, omega, w, v):
        self.F, self.omega, self.w, self.v = int(F), omega, w, v
        self.P, self.E, self.n = int(w.shape[0]), int(w.shape[1]), int(v.shape[2])
        self.D = int(omega.shape[2]) if len(np.shape(omega)) == 3 else -1
        if tuple(np.shape(omega)) != (self.E, self.F, self.D) or tuple(np.shape(w)) != (self.P, self.E, 2 * self.F) \
                or tuple(np.shape(v)) != (self.P, self.E, self.n):
            raise ValueError("FeatureDraws: expected omega [E,F,D], w [P,E,2F] and v [P,E,n], got %s, %s and %s"
                             % (tuple(np.shape(omega)), tuple(np.shape(w)), tuple(np.shape(v))))

    def struct(self, p0=0):
        """the pilco_feature_draws of the particles from p0 on (the draws of one particle are contiguous)"""
        return _lib.FeatureDraws(self.F, self.omega.data_ptr(), self.w[p0:].data_ptr(), self.v[p0:].data_ptr())


def _features_check(dyn, num_features):
    """the feature sampler's refusals on the model and F (ValueError), before any allocation"""
    F = int(num_features)
    if getattr(dyn, "sn2", None) is None or dyn.mode != 0 or dyn.iK is None or dyn.batched:
        raise ValueError("features: the function draws need the exact GP gp_factorize returns (with its sn2); a FITC "
                         "(SMGPR) model is not supported")
    if F < 1 or F > _lib.MAX_FEATURES:
        raise ValueError("features: num_features must be in 1 .. %d, got %d" % (_lib.MAX_FEATURES, F))
    return F


def feature_draws(dyn, P, F, zeta, w, eps_y, out=None):
    """pilco_particles_features_draw: P particles' dynamics functions f_pe = phi_e' w_pe + k_e(., X) v_pe drawn from
    the caller's standard normals zeta [E,F,D] (the frequencies, shared by all particles), w [P,E,2F] (the feature
    weights) and eps_y [P,E,n] (the data update's noise), through the exact GP ``dyn`` (``gp_factorize``'s, with its
    sn2) -> ``FeatureDraws``.  ValueError, before any allocation, for a model without sn2 (FITC), F outside
    1 .. 8192 or a wrong shape.  ``out``: an earlier call's draws of the same sizes over the same w tensor, redrawn in
    place with nothing allocated, so that the call can be captured in a CUDA graph."""
    F = _features_check(dyn, F)
    P, E, n, D = int(P), dyn.E, dyn.n, dyn.D
    for a, shape, what in ((zeta, (E, F, D), "zeta"), (w, (P, E, 2 * F), "w"), (eps_y, (P, E, n), "eps_y")):
        if tuple(np.shape(a)) != shape:
            raise ValueError("feature_draws: %s must be %s, got %s" % (what, shape, tuple(np.shape(a))))
    g = dyn.struct()
    wsb = int(lib.pilco_particles_features_draw_workspace_bytes(C.byref(g), P, F))
    if wsb == 0:
        raise ValueError("feature_draws: unsupported sizes (P=%d, F=%d, n=%d, D=%d, E=%d)" % (P, F, n, D, E))
    zeta, w, eps_y = dev(zeta).contiguous(), dev(w).contiguous(), dev(eps_y).contiguous()
    if out is None:
        d = device()
        out = FeatureDraws(F, torch.empty((E, F, D), dtype=F64, device=d), w,
                           torch.empty((P, E, n), dtype=F64, device=d))
        out.ws = torch.empty(max(wsb // 8, 2), dtype=F64, device=d)
    elif (out.P, out.F, out.E, out.n, out.D) != (P, F, E, n, D) or out.w.data_ptr() != w.data_ptr():
        raise ValueError("feature_draws: out holds the draws of other sizes or another w")
    check(lib.pilco_particles_features_draw(C.byref(g), ptr(dyn.sn2), P, F, ptr(zeta), ptr(w), ptr(eps_y),
                                            ptr(out.omega), ptr(out.v), ptr(out.ws), wsb, stream_ptr()),
          "particles_features_draw")
    return out


class ParticlePlan(_Particles):
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
    value.  ``"score"`` with ``consistent=True``, or an unknown estimator, is a ValueError.

    ``angles``: angular state dimensions (pilco_particles_angles_*, DESIGN.md section 20).  The state x0, eps and traj
    then have the dynamics GP's output count E as their last dimension; the policy (``policy_spec["Ds"]`` = E +
    len(angles)) and the joint state-action terms see phi(x), the dynamics GP [phi(x), u].  The gradient of an unbatched
    plan runs the batch-gradient call at R = 1.

    ``measurement_noise``: variances v [E] >= 0 of a noisy state measurement (pilco_particles_noisy_*, DESIGN.md section
    23): the policy sees phi(z_t), z_t = x_t + sqrt(v) o nu_t, while the dynamics GP and the rewards see the true state.
    The plan then owns a nu buffer [P,H,E] of standard normals shared by the R policies, which ``set_inputs`` fills
    (its ``nu`` is then required).  The gradients are conditioned on nu, as on x0 and eps.

    ``exploration``: a float b (0.0 included) selects PILCO's exploration objective in ``launch_grad()``
    (pilco_particles_explore_*, DESIGN.md section 24): value = mean return + b sum_t sigma_t, sigma_t^2 the sum over the
    additive terms of c_k^2 times the sample variance of term k over the restart's P particles at step t, with its
    pathwise gradient.  The plan then owns ``step_var`` [R, max(H,1)], which each ``launch_grad()`` fills with
    sigma_t^2.  At b = 0 every other output and gradient is bitwise the plan's without exploration.  It needs
    ``grad=True``, P >= 2 and no additive box term; ``estimator="score"`` with it is a ValueError.  ``None``: no
    exploration.

    ``resample=True``: Deep PILCO's Gaussian refit (pilco_particles_resampled_*, DESIGN.md section 26).  At every step
    t >= 1 each restart's particles are replaced by draws mu^_t + L^_t xi_t from the Gaussian fitted to them (sample
    mean and unbiased covariance, L^_t its Cholesky factor with degenerate columns zeroed), and the rewards and the
    policy are evaluated at the redrawn particles.  The plan then owns ``xi`` [P,H,Ds] (standard normals shared by the
    R policies, which ``set_inputs`` fills: its ``xi`` is then required), ``step_mean`` [R?,H+1,Ds] and ``step_cov``
    [R?,H+1,Ds,Ds] (the fitted moments; t = 0: those of x0), which every launch fills.  ``launch_grad()`` gives the
    pathwise gradient through the refit.  It needs P >= 2; with ``consistent``, ``estimator="score"``, ``angles``,
    ``measurement_noise`` or ``exploration`` it is a ValueError raised before any allocation.

    ``schedule=True``: a time-varying linear policy u_t = sq(W_t x + b_t) (pilco_particles_scheduled_*, DESIGN.md
    section 28), with every sampler, estimator and feature above.  The spec's W is [Hw, U, Ds] or [R, Hw, U, Ds] and b
    [Hw, U] or [R, Hw, U], Hw >= H (step t < H reads W[..., t, :, :]); ``launch_grad()`` then returns the per-step
    gradients 'W' [R?, H, U, Ds] and 'b' [R?, H, U].  An RBF spec or Hw < H is a ValueError raised before any
    allocation, and so is a scheduled spec without ``schedule=True``.

    A tanh MLP policy (pilco_particles_mlp_*, DESIGN.md section 29): ``dict(kind=POLICY_MLP, Ds, U, squash,
    max_action, hidden=(w1[, w2]), theta)``, theta [n_theta] or [R, n_theta] in ``mlp_theta_size``'s flat layout (A_1,
    (A_2,) A_out, each row-major [out, in + 1] with the bias last).  Every sampler, forward and pathwise, with
    exploration; ``launch_grad()`` returns {'value', 'theta' [R?, n_theta]}.  With ``angles``, ``measurement_noise``,
    ``schedule=True`` or ``estimator="score"``, or a theta of the wrong length, it is a ValueError raised before any
    allocation.

    ``num_features=F`` with ``consistent=True``: each particle's functions are random-feature draws with an exact
    data update (pilco_particles_features_*, DESIGN.md section 30), which ``set_inputs(x0, None, features=draws)``
    takes from ``feature_draws`` in place of eps; the workspace does not grow with n or F.  Its gradient is
    ``ConsistentGradPlan(num_features=F)``.  Without ``consistent=True``, with ``estimator="score"``, ``resample``
    or ``schedule``, or with a model without sn2 (FITC), it is a ValueError raised before any allocation."""

    ESTIMATORS = ("pathwise", "score")

    def __init__(self, dyn, policy_spec, reward_terms, P, H, mult_mu=0.0, grad=False, R=1, consistent=False,
                 estimator="pathwise", angles=None, measurement_noise=None, exploration=None, resample=False,
                 schedule=False, num_features=None):
        mlp = _particle_mlp(policy_spec, "ParticlePlan", R, angles, measurement_noise, schedule, estimator)
        sched = _particle_schedule(policy_spec, H, schedule, "ParticlePlan")
        self.fd = _features_plan_check(dyn, num_features, consistent, estimator, resample, schedule)
        if estimator not in self.ESTIMATORS:
            raise ValueError("particles: estimator must be one of %s, not %r" % (self.ESTIMATORS, estimator))
        self.resample = bool(resample)
        if self.resample:
            _resample_check(P, consistent, estimator, angles, measurement_noise, exploration)
        if exploration is not None and (estimator == "score" or not grad):
            raise ValueError("particles: exploration is an objective of the pathwise gradient: it needs grad=True and "
                             "estimator='pathwise' (the score-function estimate of sigma_t's gradient is not available)")
        if consistent and estimator == "score":
            raise ValueError("particles: the score-function gradient of the consistent (function-sample) rollout "
                             "is engine.ConsistentGradPlan(..., estimator='score'), not ParticlePlan")
        self.estimator = estimator
        if consistent and grad:
            raise ValueError("particles: the gradient of the consistent (function-sample) rollout is "
                             "ConsistentGradPlan, not ParticlePlan(grad=True)")
        self.consistent = bool(consistent)
        self._describe(dyn, policy_spec, reward_terms, P, H, mult_mu, R, grad, angles, measurement_noise, exploration,
                       sched, mlp)
        pr, d = self.pr, device()
        if not self.batched:                                    # the forward-only rollout (a batch has none)
            self.fwd = self._entry(self._key("forward"))
            wsb = self.fwd.query()
            if wsb == 0:
                raise ValueError("particles: unsupported sizes (P=%d, H=%d, D=%d)" % (self.P, self.H, dyn.D))
            self.ws = torch.empty(max(wsb // 8, 2), dtype=F64, device=d)
            pr.ws, pr.ws_bytes = self.ws.data_ptr(), wsb
        self.grad = None
        if grad:
            self._grad_buffers(self._grad_ws_bytes(self.P))

    def _key(self, call):
        """the PARTICLE_ENTRY_POINTS row of this plan's ``call``"""
        family = "mlp" if self.mlp is not None else "scheduled" if self.sch is not None else "plain"
        sampler = "resampled" if self.resample else "features" if self.fd is not None else \
            "consistent" if self.consistent else "step"
        return family, sampler, call

    def _grad_ws_bytes(self, P):
        """the gradient workspace of this plan's call with P particles per restart (0: unsupported sizes)"""
        pr = _lib.Particles.from_buffer_copy(self.pr)
        pr.P = int(P)
        return self._entry(self._key(self.estimator), pr=pr).query()

    def _describe(self, dyn, policy_spec, reward_terms, P, H, mult_mu, R, grad, angles=None, measurement_noise=None,
                  exploration=None, sched=None, mlp=None):
        """the pilco_particles description, its input and output buffers (self.pr); self.Ds is the state's width.
        The angles, the policy's width, the measurement noise, the exploration weight and the policy's shapes are
        checked first, before any device work.  ``sched``: ``_schedule_check``'s (batched, Hw) of a scheduled spec, or
        None; ``mlp``: ``_particle_mlp``'s (L, widths, n_theta, batched) of an MLP spec, or None."""
        b = _particle_exploration(exploration, reward_terms, P)
        E, ang = _policy_width(dyn, policy_spec, angles, "particles")
        nz = _noise_struct(measurement_noise, E)
        P, H, R = int(P), int(H), int(R)
        if P < 1 or H < 0 or R < 1:
            raise ValueError("particles: needs P >= 1, H >= 0 and R >= 1 (P=%d, H=%d, R=%d)" % (P, H, R))
        Ds, U = E + (ang.A if ang is not None else 0), int(policy_spec["U"])
        rbf_batched = policy_spec["kind"] == _lib.POLICY_RBF and policy_spec["gp"].batched
        self.R, self.batched = R, R > 1 or rbf_batched or (mlp is not None and mlp[3])
        if self.batched and not grad:
            raise ValueError("particles: a batch of policies runs the gradient path only (grad=True)")
        size = lambda k: int(np.prod(np.shape(policy_spec[k])))
        if sched is not None:                                   # step t reads W[..., t, :, :], b[..., t, :]
            Hw = sched[1]
            if size("W") != R * Hw * U * Ds or size("b") != R * Hw * U:
                raise ValueError("particles: schedule=True expects W [R,Hw,U,Ds] and b [R,Hw,U] with R=%d (unbatched: "
                                 "[Hw,U,Ds], [Hw,U])" % R)
        elif mlp is None and policy_spec["kind"] == _lib.POLICY_LINEAR:
            if size("W") != R * U * Ds or size("b") != R * U:
                raise ValueError("particles: expected W [R,U,Ds] and b [R,U] with R=%d (unbatched: [U,Ds], [U])" % R)
        elif mlp is None and (rbf_batched != self.batched or (self.batched and policy_spec["gp"].X.shape[0] != R)):
            raise ValueError("particles: the RBF policy must be factorised with a leading R=%d (unbatched: none)" % R)
        self.lead = (R,) if self.batched else ()
        self._structs(dyn, policy_spec, P, H, ang, nz, sched is not None, mlp, self.batched)
        self.Ds = E
        self._buffers(policy_spec, reward_terms, mult_mu, self.lead, self.batched)
        mk = lambda *shape: torch.zeros(shape, dtype=F64, device=device())
        Hb, lead = max(H, 1), self.lead
        if b is not None:                                       # sigma_t^2 [R, max(H,1)], also for an unbatched plan
            self.step_var = mk(R, Hb)
            self.ex = _lib.Exploration(b, self.step_var.data_ptr())
        if self.resample:                                       # xi shared by the R policies; the fitted moments
            self.xi_buf = mk(P, Hb, E)
            self._step_mean, self._step_cov = mk(R, H + 1, E), mk(R, H + 1, E, E)
            self.step_mean = self._step_mean.view(*lead, H + 1, E)
            self.step_cov = self._step_cov.view(*lead, H + 1, E, E)
            self.rs = _lib.ParticlesResample(self.xi_buf.data_ptr(), self._step_mean.data_ptr(),
                                             self._step_cov.data_ptr())

    def _grad_buffers(self, gwsb):
        """the pilco_particles_grad outputs and a gradient workspace of gwsb bytes (self.grad)"""
        d, pr = device(), self.pr
        if gwsb == 0:
            raise ValueError("particles: unsupported sizes (P=%d, H=%d, D=%d, R=%d)" % (self.P, self.H, pr.dyn.D, self.R))
        g = _lib.ParticlesGrad()
        if self.mlp is not None:                                # d value / d theta [R?, n_theta]
            self.gbuf = {"theta": torch.zeros((*self.lead, self.n_theta), dtype=F64, device=d)}
            self.mlp.gtheta = self.gbuf["theta"].data_ptr()
        elif self.sch is None:
            self.gbuf = _policy_grad_buffers(g, pr.pol, self.rbf, self.lead)
        else:                                                   # per step; H = 0 still has an address
            self.gbuf = _policy_grad_buffers(g, pr.pol, self.rbf, self.lead + (max(self.H, 1),))
            self.gbuf["W"], self.gbuf["b"] = self.gbuf["W"][..., :self.H, :, :], self.gbuf["b"][..., :self.H, :]
        self.gbuf["value"] = torch.zeros(self.R if self.batched else 1, dtype=F64, device=d)
        g.value = self.gbuf["value"].data_ptr()
        self.gws = torch.empty(max(gwsb // 8, 2), dtype=F64, device=d)
        g.ws, g.ws_bytes = self.gws.data_ptr(), gwsb
        self.grad = g
        self.bwd = self._entry(self._key(self.estimator))

    def launch_grad(self):
        """pilco_particles_rollout_grad: the rollout (``outputs()`` as after ``launch()``, bitwise) and the pathwise
        gradient of value = mean return w.r.t. the policy parameters with x0 and eps fixed.  Returns the device tensors
        {'value' [1], 'W' [U,Ds], 'b' [U]} (linear) or {'value', 'X' [bf,Ds], 'Y' [bf,U], 'ell' [U,Ds]} (RBF, constrained
        lengthscales), like ``RolloutPlan.backward``.  A batched plan returns them with a leading R ('value' [R]).
        ``estimator="score"``: the score-function gradient (pilco_particles_rollout_score_grad) in the same layout.
        With ``exploration``: value and gradient of the exploration objective, and sigma_t^2 in ``step_var``.  With
        ``schedule``: 'W' [R?,H,U,Ds] and 'b' [R?,H,U], one gradient per step.  An MLP policy: {'value', 'theta'
        [R?, n_theta]}."""
        if self.grad is None:
            raise RuntimeError("ParticlePlan: constructed without grad=True")
        self.bwd()
        return self.gbuf

    def set_inputs(self, x0, eps, nu=None, xi=None, features=None):
        """x0 [P,Ds], eps [P,H,Ds], with measurement noise nu [P,H,E] and with ``resample`` xi [P,H,Ds] (each required
        then, and only then).  With ``num_features``: ``features`` (``feature_draws`` of P particles at that F) in
        place of eps, which is then not read (None)."""
        if (features is None) != (self.fd is None):
            raise ValueError("particles: features (feature_draws) are required with num_features and only then")
        if features is not None:
            dyn = self.pr.dyn
            have, want = (features.P, features.F, features.E, features.n, features.D), \
                (self.P, self.fd.F, dyn.E, dyn.n, dyn.D)
            if have != want:
                raise ValueError("particles: the feature draws are for (P, F, E, n, D) = %s; the plan has %s"
                                 % (have, want))
            self.features = features                            # keeps the draws alive
            st = features.struct()                              # in place: the bound calls point at self.fd
            self.fd.omega, self.fd.w, self.fd.v = st.omega, st.w, st.v
        if (nu is None) != (self.nz is None):
            raise ValueError("particles: nu [P,H,E] is required with measurement_noise and only then")
        if (xi is None) == self.resample:
            raise ValueError("particles: xi [P,H,Ds] is required with resample=True and only then")
        self.x0.copy_(dev(x0).reshape(self.P, self.Ds))
        if self.H > 0:
            if features is None:
                self.eps_buf.copy_(dev(eps).reshape(self.P, self.H, self.Ds))
            if nu is not None:
                self.nu_buf.copy_(dev(nu).reshape(self.nu_buf.shape))
            if xi is not None:
                self.xi_buf.copy_(dev(xi).reshape(self.P, self.H, self.Ds))

    def launch(self):
        if self.batched:
            raise RuntimeError("ParticlePlan: a batch of policies runs launch_grad()")
        self.fwd()

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
    that names the bytes needed and the number of particles that would fit, raised before anything is allocated.

    ``angles``, ``measurement_noise``, ``exploration``: as ``ParticlePlan`` (pilco_particles_explore_consistent_grad_*
    with exploration).

    ``estimator``: ``"pathwise"`` (the default) or ``"score"``, the score-function estimator over the same function
    samples (pilco_particles_consistent_score_grad_rollout, DESIGN.md section 25), which differentiates the log-density
    of each particle's whole path under its draw instead of the path itself, so box terms enter its gradient.  The same
    rollout, value and output layout; its estimate is unbiased on rollouts without degenerate pivots.  ``"score"`` with
    ``exploration``, or an unknown estimator, is a ValueError raised before any allocation.

    ``schedule=True``: a time-varying linear policy, as ``ParticlePlan``.  A tanh MLP policy: as ``ParticlePlan``.

    ``num_features=F``: the functions are random-feature draws with an exact data update (DESIGN.md section 30), taken
    by ``set_inputs(x0, None, nu=None, features=draws)``; the workspace is O(R P H (D + E)), whatever n and F.  With
    ``estimator="score"`` or ``schedule`` it is a ValueError raised before any allocation."""

    def __init__(self, dyn, policy_spec, reward_terms, P, H, mult_mu=0.0, R=1, max_ws_bytes=None, angles=None,
                 measurement_noise=None, exploration=None, estimator="pathwise", schedule=False, num_features=None):
        mlp = _particle_mlp(policy_spec, "ConsistentGradPlan", R, angles, measurement_noise, schedule, estimator)
        sched = _particle_schedule(policy_spec, H, schedule, "ConsistentGradPlan")
        self.fd = _features_plan_check(dyn, num_features, True, estimator, False, schedule)
        if estimator not in self.ESTIMATORS:
            raise ValueError("particles: estimator must be one of %s, not %r" % (self.ESTIMATORS, estimator))
        if exploration is not None and estimator == "score":
            raise ValueError("particles: exploration is an objective of the pathwise gradient: it needs "
                             "estimator='pathwise' (the score-function estimate of sigma_t's gradient is not available)")
        self.estimator = estimator
        self.consistent, self.resample = True, False
        self._describe(dyn, policy_spec, reward_terms, P, H, mult_mu, R, True, angles, measurement_noise, exploration,
                       sched, mlp)
        need = self._grad_ws_bytes(self.P)
        if need == 0:
            raise ValueError("particles: unsupported sizes (P=%d, H=%d, D=%d, R=%d)" % (self.P, self.H, dyn.D, self.R))
        _largest_fitting(self._grad_ws_bytes, self.P, max_ws_bytes, "particles: the consistent gradient of %d restarts "
                         "x %d particles over H=%d steps" % (self.R, self.P, self.H), whole="num_samples")
        self._grad_buffers(need)

    def launch(self):
        raise RuntimeError("ConsistentGradPlan: the rollout runs with its gradient, launch_grad()")

    def launch_grad(self):
        """pilco_particles_rollout_consistent_grad: the consistent rollout (``outputs()``) and the pathwise gradient
        of value = mean return (with ``exploration``: the exploration objective, and sigma_t^2 in ``step_var``),
        returned as ``ParticlePlan.launch_grad`` returns it.  ``estimator="score"``: the score-function gradient
        (pilco_particles_consistent_score_grad_rollout) in the same layout"""
        return super().launch_grad()


def _features_plan_check(dyn, num_features, consistent, estimator, resample, schedule):
    """a plan's feature sampler (ValueError before any allocation): None without num_features, else the
    pilco_feature_draws its size queries take (F set; set_inputs points it at the draws)"""
    if num_features is None:
        return None
    for on, what in ((not consistent, "consistent=False (the draws are whole functions: consistent=True)"),
                     (estimator == "score", "estimator='score' (a function sample has no per-step path density)"),
                     (resample, "resample=True"), (schedule, "schedule=True")):
        if on:
            raise ValueError("particles: num_features does not combine with %s" % what)
    return _lib.FeatureDraws(_features_check(dyn, num_features), None, None, None)


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


def _particle_noise(measurement_noise, E):
    """the measurement variances v [E] of the particle plans as a numpy array (None: no noise).  ValueError for a
    wrong length, a non-finite or a negative value"""
    if measurement_noise is None:
        return None
    v = np.asarray(measurement_noise, dtype=np.float64).reshape(-1)
    if v.shape[0] != E:
        raise ValueError("measurement_noise: expected %d variances (the state dimension), got %d" % (E, v.shape[0]))
    if not np.all(np.isfinite(v)) or np.any(v < 0.0):
        raise ValueError("measurement_noise: the variances must be finite and >= 0, got %r" % v)
    return v


def _particle_exploration(exploration, reward_terms, P):
    """the exploration weight b of the particle plans as a float (None: no exploration).  ValueError for a non-finite
    b, an additive box term (no gradient, and section 21's rule) or fewer than 2 particles (no sample variance)"""
    if exploration is None:
        return None
    b = float(exploration)
    if not np.isfinite(b):
        raise ValueError("exploration: b must be finite, got %r" % exploration)
    _no_additive_box(reward_terms)
    if int(P) < 2:
        raise ValueError("exploration: the sample variance of the step rewards needs P >= 2 particles, got %d" % int(P))
    return b


def _resample_check(P, consistent, estimator, angles, measurement_noise, exploration):
    """the Gaussian refit's refusals (ValueError), before any allocation: it runs on the step-wise sampler with the
    pathwise gradient only, without angles, measurement noise or exploration, and needs P >= 2"""
    for on, what in ((consistent, "consistent=True (redrawing breaks a particle's identity with its function)"),
                     (estimator == "score", "estimator='score' (the path density no longer factorises per particle)"),
                     (angles is not None and len(angles) > 0, "angles"),
                     (measurement_noise is not None, "measurement_noise"), (exploration is not None, "exploration")):
        if on:
            raise ValueError("particles: resample=True does not combine with %s" % what)
    if int(P) < 2:
        raise ValueError("particles: resample=True fits a covariance to the particles: it needs P >= 2, got %d" % int(P))


def _no_additive_box(reward_terms):
    for k, rt in enumerate(reward_terms):
        if rt["kind"] == _lib.REWARD_BOX and int(rt.get("channel", _lib.CHANNEL_ADD)) == _lib.CHANNEL_ADD:
            raise ValueError("exploration: reward term %d is an additive box term, which the reward variance leaves "
                             "out of its rule; use it in the multiplicative channel (SafePILCO) or leave exploration "
                             "off" % k)


def particle_reward_moments(reward_terms, traj, act, angles=None):
    """pilco_particles_reward_moments: the per-step sample moments of the reward over particles that have already been
    rolled out -> (mean [..., H], var [..., H]) device tensors.  ``traj`` [..., P, H+1, E] and ``act`` [..., P, H, U]
    are any sampler's outputs (a leading restart dimension, or none), chunked or not.  mean_t = sum_k c_k rbar_kt and
    var_t = sum_k c_k^2 s_kt^2 over the additive terms, s_kt^2 the unbiased variance of term k over the P particles
    (DESIGN.md section 24): the sampled counterparts of the moment-matching rollout's E[r_t] and sigma_t^2.
    ``angles``: the angular state dimensions the policy saw (the joint terms are evaluated at [phi(x), u])."""
    if len(traj.shape) < 3 or len(act.shape) != len(traj.shape) or tuple(act.shape[:-2]) != tuple(traj.shape[:-2]) \
            or act.shape[-2] != traj.shape[-2] - 1:
        raise ValueError("particle_reward_moments: expected traj [..., P, H+1, E] and act [..., P, H, U], got %s and %s"
                         % (tuple(traj.shape), tuple(act.shape)))
    lead = tuple(traj.shape[:-3])
    P, H, E, U = int(traj.shape[-3]), int(traj.shape[-2]) - 1, int(traj.shape[-1]), int(act.shape[-1])
    if P < 2:
        raise ValueError("particle_reward_moments: the sample variance needs P >= 2 particles, got %d" % P)
    _no_additive_box(reward_terms)
    traj, act = dev(traj), dev(act)
    R = int(np.prod(lead)) if lead else 1
    ang = angles_struct(angles, E)
    pr = _lib.Particles()
    pr.P, pr.H = P, H
    pr.dyn.E = E
    pr.pol.Ds, pr.pol.U = E + (ang.A if ang is not None else 0), U
    keep = _fill_rewards(pr, reward_terms)                     # noqa: F841 -- the terms' device tensors stay alive
    Hb = max(H, 1)
    mean = torch.zeros((R, Hb), dtype=F64, device=device())
    var = torch.zeros((R, Hb), dtype=F64, device=device())
    pr.traj, pr.act = traj.data_ptr(), act.data_ptr()
    check(lib.pilco_particles_reward_moments(C.byref(pr), C.byref(ang) if ang is not None else None, R, ptr(mean),
                                             ptr(var), stream_ptr()), "particles_reward_moments")
    return mean[:, :H].reshape(*lead, H), var[:, :H].reshape(*lead, H)


def particles_rollout(dyn, policy_spec, reward_terms, x0, eps, mult_mu=0.0, consistent=False, max_ws_bytes=None,
                      angles=None, measurement_noise=None, nu=None, resample=False, xi=None, schedule=False,
                      features=None, horizon=None):
    """pilco_particles_rollout: P particles from x0 [P,Ds] driven by the standard normals eps [P,H,Ds] through the
    factorised dynamics ``dyn`` under the (unbatched) policy -> (traj [P,H+1,Ds], act [P,H,U], step_reward [P,H],
    step_risk [P,H], ret [P]) device tensors.

    ``consistent=True``: pilco_particles_rollout_consistent, one posterior function per particle.  Its workspace is
    O(P H E n), so the particles run in chunks whose workspace fits ``max_ws_bytes`` (default: half the free device
    memory).  A particle's outputs do not depend on its batch, so the chunking does not change them.

    ``angles``: angular state dimensions, as ``ParticlePlan``: Ds is then the dynamics GP's output count E and the
    policy takes E + len(angles) inputs.

    ``measurement_noise``: variances v [E] of the policy's measurement z = x + sqrt(v) o nu, as ``ParticlePlan``; ``nu``
    [P,H,E] are its standard normals (required with it, for both samplers).

    ``resample=True``: the Gaussian refit at every step, as ``ParticlePlan(resample=True)``; ``xi`` [P,H,Ds] are the
    redraw's standard normals (required with it, and only then).  The result then also has the fitted moments:
    (traj, act, step_reward, step_risk, ret, step_mean [H+1,Ds], step_cov [H+1,Ds,Ds]).

    ``schedule=True``: a time-varying linear policy (W [Hw,U,Ds], b [Hw,U], Hw >= H), as ``ParticlePlan``.

    A tanh MLP spec (theta [n_theta]) runs every sampler, as ``ParticlePlan``.

    ``features`` (``feature_draws`` of the P particles) with ``consistent=True``: the functions are those random-feature
    draws with an exact data update (DESIGN.md section 30) and eps is not read: pass None and the horizon as
    ``horizon``.  The particles run in chunks under ``max_ws_bytes`` as with the exact consistent sampler.  Without
    ``consistent=True``, or with ``resample`` or ``schedule``, it is a ValueError."""
    if features is not None:
        return _particles_rollout_features(dyn, policy_spec, reward_terms, x0, mult_mu, consistent, max_ws_bytes,
                                           angles, measurement_noise, nu, resample, schedule, features, horizon)
    _particle_mlp(policy_spec, "particles_rollout", 1, angles, measurement_noise, schedule)
    _particle_schedule(policy_spec, eps.shape[1] if len(np.shape(eps)) == 3 else 0, schedule, "particles_rollout")
    if resample:
        _resample_check(x0.shape[0], consistent, "pathwise", angles, measurement_noise, None)
    if (xi is None) == bool(resample):
        raise ValueError("particles_rollout: xi [P,H,Ds] is required with resample=True and only then")
    x0, eps = dev(x0), dev(eps)
    if x0.dim() != 2 or eps.dim() != 3 or eps.shape[0] != x0.shape[0] or eps.shape[2] != x0.shape[1]:
        raise ValueError("particles_rollout: x0 must be [P,Ds] and eps [P,H,Ds], got %s and %s"
                         % (tuple(x0.shape), tuple(eps.shape)))
    if (nu is None) != (measurement_noise is None):
        raise ValueError("particles_rollout: nu [P,H,E] is required with measurement_noise and only then")
    if nu is not None:
        nu = dev(nu)
        if tuple(nu.shape) != tuple(eps.shape):
            raise ValueError("particles_rollout: nu must be [P,H,E] like eps, got %s" % (tuple(nu.shape),))
    if consistent:
        return _particles_rollout_consistent(dyn, policy_spec, reward_terms, x0, eps, mult_mu, max_ws_bytes, angles,
                                             measurement_noise, nu, schedule)
    if resample:
        xi = dev(xi)
        if tuple(xi.shape) != tuple(eps.shape):
            raise ValueError("particles_rollout: xi must be [P,H,Ds] like eps, got %s" % (tuple(xi.shape),))
    plan = ParticlePlan(dyn, policy_spec, reward_terms, x0.shape[0], eps.shape[1], mult_mu=mult_mu, angles=angles,
                        measurement_noise=measurement_noise, resample=resample, schedule=schedule)
    plan.set_inputs(x0, eps, nu, xi)
    plan.launch()
    return plan.outputs() + ((plan.step_mean, plan.step_cov) if resample else ())


def _particles_rollout_features(dyn, policy_spec, reward_terms, x0, mult_mu, consistent, max_ws_bytes, angles,
                                measurement_noise, nu, resample, schedule, features, horizon):
    """particles_rollout with feature draws: every check on the host shapes first, then the chunked consistent path
    with no eps"""
    _features_plan_check(dyn, features.F, consistent, "pathwise", resample, schedule)
    _particle_mlp(policy_spec, "particles_rollout", 1, angles, measurement_noise, schedule)
    if horizon is None or int(horizon) < 0:
        raise ValueError("particles_rollout: with features the horizon (>= 0) is required, got %r" % (horizon,))
    H = int(horizon)
    if len(np.shape(x0)) != 2 or np.shape(x0)[0] != features.P:
        raise ValueError("particles_rollout: x0 must be [P,Ds] with P=%d (the draws'), got %s"
                         % (features.P, tuple(np.shape(x0))))
    if (nu is None) != (measurement_noise is None):
        raise ValueError("particles_rollout: nu [P,H,E] is required with measurement_noise and only then")
    if nu is not None and tuple(np.shape(nu)) != (features.P, H, int(np.shape(x0)[1])):
        raise ValueError("particles_rollout: nu must be [P,H,E], got %s" % (tuple(np.shape(nu)),))
    return _particles_rollout_consistent(dyn, policy_spec, reward_terms, dev(x0), None, mult_mu, max_ws_bytes, angles,
                                         measurement_noise, None if nu is None else dev(nu), schedule, features, H)


def consistent_workspace_bytes(dyn, Ds, U, P, H, angles=None, num_features=None):
    """pilco_particles_consistent_workspace_bytes of P particles over H steps (0: unsupported sizes); ``Ds`` is the
    policy's input width (with ``angles``: E + len(angles)).  ``num_features``: the feature sampler's
    (pilco_particles_features_workspace_bytes)."""
    d = _Particles()
    d._structs(dyn, dict(Ds=Ds, U=U), P, H, angles_struct(angles, int(dyn.struct().E)))
    if num_features is not None:
        d.fd = _lib.FeatureDraws(int(num_features), None, None, None)
    return d._entry(("plain", "consistent" if d.fd is None else "features", "forward")).query()


def _particles_rollout_consistent(dyn, policy_spec, reward_terms, x0, eps, mult_mu, max_ws_bytes, angles=None,
                                  measurement_noise=None, nu=None, schedule=False, features=None, H=None):
    """the consistent rollout in chunks of particles; with ``features`` eps is None and H is given"""
    P, H = int(x0.shape[0]), int(eps.shape[1]) if H is None else int(H)
    Ds, U = int(policy_spec["Ds"]), int(policy_spec["U"])
    E, _ = _policy_width(dyn, policy_spec, angles, "particles_rollout")
    _particle_noise(measurement_noise, E)
    F = features.F if features is not None else None
    lo = _largest_fitting(lambda p: consistent_workspace_bytes(dyn, Ds, U, p, H, angles, F), P, max_ws_bytes,
                          "particles_rollout: the consistent rollout of one particle (H=%d, n=%d)" % (H, dyn.n))
    if lo == P:
        plan = ParticlePlan(dyn, policy_spec, reward_terms, P, H, mult_mu=mult_mu, consistent=True, angles=angles,
                            measurement_noise=measurement_noise, schedule=schedule, num_features=F)
        plan.set_inputs(x0, None if F else eps, nu, features=features)
        plan.launch()
        return plan.outputs()
    d = device()
    Hb, Ds = max(H, 1), int(x0.shape[1])
    out = (torch.empty((P, H + 1, Ds), dtype=F64, device=d), torch.empty((P, Hb, U), dtype=F64, device=d)[:, :H],
           torch.empty((P, Hb), dtype=F64, device=d)[:, :H], torch.empty((P, Hb), dtype=F64, device=d)[:, :H],
           torch.empty(P, dtype=F64, device=d))
    plan = None
    for p0 in range(0, P, lo):
        p1 = min(P, p0 + lo)
        if plan is None or plan.P != p1 - p0:
            plan = None                                     # free the previous chunk's workspace first
            plan = ParticlePlan(dyn, policy_spec, reward_terms, p1 - p0, H, mult_mu=mult_mu, consistent=True,
                                angles=angles, measurement_noise=measurement_noise, schedule=schedule, num_features=F)
        part = None if features is None else FeatureDraws(F, features.omega, features.w[p0:p1], features.v[p0:p1])
        plan.set_inputs(x0[p0:p1], None if F else eps[p0:p1], None if nu is None else nu[p0:p1], features=part)
        plan.launch()
        for o, c in zip(out, plan.outputs()):
            o[p0:p1].copy_(c)
    return out


class CemLoop:
    """The cross-entropy method's loop on the device (DESIGN.md sections 31 and 33), shared by ``CemPlan`` and
    ``policy_opt.CemPolicySearch``: the K candidates ``cand`` [K,H,U], the diagonal Gaussian ``mean`` and ``std`` [H,U]
    they are drawn from, the best so far (``best`` [H,U], ``best_value`` [1]) and ``trace`` [iters,2], with the
    pilco_cem structs of the first draw and of every iteration's update and the update's workspace.  The candidates'
    values are ``value`` [K]; population i is drawn from the normals ``xi[i]`` (i < iters), clipped to [-bound,
    bound]."""

    def __init__(self, K, H, U, elites, iters, alpha, bound, value, xi, mean0, std0):
        mk = lambda *shape: torch.zeros(shape, dtype=F64, device=device())
        self.mean0, self.std0 = mean0, std0
        self.cand, self.mean, self.std, self.best = mk(K, H, U), mk(H, U), mk(H, U), mk(H, U)
        self.best_value, self.trace = mk(1), mk(iters, 2)
        cem = lambda xi, trace: _lib.Cem(K, H, U, elites, alpha, -bound, bound, value.data_ptr(), self.cand.data_ptr(),
                                         xi, self.mean.data_ptr(), self.std.data_ptr(), self.best_value.data_ptr(),
                                         self.best.data_ptr(), trace)
        self.draw = cem(xi[0].data_ptr(), None)                 # the first population, then each update's next one
        self.updates = [cem(xi[i + 1].data_ptr() if i + 1 < iters else None, self.trace[i].data_ptr())
                        for i in range(iters)]
        self.uws_bytes = int(lib.pilco_cem_update_workspace_bytes(K))
        self.uws = torch.empty(max(self.uws_bytes // 8, 2), dtype=F64, device=device())

    def launch(self, evaluate, redraw=None):
        """the whole loop on the current stream, with no host synchronisation: mean, std and the best back to the
        start, (``redraw(0)``,) the first draw, then per iteration i ``evaluate()`` (the candidates' values), (before
        every update but the last ``redraw(i + 1)``, the normals of the next population,) and the update"""
        self.mean.copy_(self.mean0)
        self.std.copy_(self.std0)
        self.best.copy_(self.mean0)
        self.best_value.fill_(-float("inf"))
        if redraw is not None:
            redraw(0)
        check(lib.pilco_cem_draw(C.byref(self.draw), stream_ptr()), "cem_draw")
        for i, u in enumerate(self.updates):
            evaluate()
            if redraw is not None and i + 1 < len(self.updates):
                redraw(i + 1)
            check(lib.pilco_cem_update(C.byref(u), self.uws.data_ptr(), self.uws_bytes, stream_ptr()), "cem_update")

    def capture(self, evaluate, redraw=None):
        """``launch`` eagerly (a warm-up that sets one-time kernel attributes), then recorded as one CUDA graph, which
        is returned.  Unreachable cycles are collected first: one that holds an earlier graph would otherwise be freed
        inside the capture, and freeing a graph's memory there invalidates it."""
        self.launch(evaluate, redraw)
        torch.cuda.synchronize()
        gc.collect()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            self.launch(evaluate, redraw)
        return g


CEM_BOUND = 0.5 * np.pi          # the candidates' b lie in [-pi/2, pi/2], where u = maxa sin(b) is monotone and onto


class CemPlan(_Particles):
    """The cross-entropy method (CEM) over open-loop action sequences on the sampled return, as trajectory-sampling MPC
    plans on a learnt model (PETS, Chua et al. 2018; DESIGN.md section 31), every iteration on the device.

    ``spec`` is a scheduled linear policy: W [Hw,U,Ds] (Hw >= H), shared by every candidate and held fixed (zero for the
    open-loop sequences u_t = maxa sin(b_t)), and b [Hw,U], whose first H steps are the initial sampling mean.  Each of
    ``iters`` iterations rolls out the ``population`` = K candidate schedules b [K,H,U] over the same P particles (x0,
    eps and, with ``measurement_noise``, nu; pilco_particles_scheduled_batch_rollout, or _consistent_ with
    ``consistent=True``), scores each by its mean return and refits a diagonal Gaussian to the ``elites`` best with
    smoothing ``alpha`` (pilco_cem_update).  The candidates are clipped to [-pi/2, pi/2]; row 0 of every population is
    the clipped sampling mean, so the plan is at least as good as its warm start on the same particles.  Every reward
    term works, box terms and the SafePILCO channel (``mult_mu``) included, since nothing is differentiated.
    ``angles``: as ``ParticlePlan`` (the state is then the dynamics GP's E outputs, the policy takes E + len(angles)).

    ``set_inputs(x0, eps, xi, nu=None, std0=None)`` fills the static buffers; ``launch()`` enqueues the whole loop (a
    draw, then per iteration the batched rollout and the update) and ``capture()`` records it as one CUDA graph that
    ``replay()`` runs.  Afterwards ``best_b`` [H,U] and ``best_value`` [1] hold the best candidate so far and its value,
    ``mean`` and ``std`` [H,U] the sampling distribution, ``trace`` [iters,2] each iteration's top value and elites'
    mean value, and ``outputs()`` the last population's rollouts.

    ``consistent=True`` rolls the candidates out in chunks whose O(R P H E n) workspace fits ``max_ws_bytes`` (default:
    half the free device memory); restarts are independent, so the chunking changes no bit.  An RBF or MLP spec, a W
    with a leading batch dimension, an unsquashed policy, ``num_features``, ``resample``, any ``estimator``, K outside
    1 .. 8192, elites outside 1 .. K, iters < 1, alpha outside [0, 1) or H < 1 is a ValueError raised before any
    allocation."""

    def __init__(self, dyn, spec, reward_terms, P, H, population, elites, iters, mult_mu=0.0, consistent=False,
                 angles=None, measurement_noise=None, alpha=0.1, max_ws_bytes=None, num_features=None, resample=False,
                 estimator=None):
        if _is_mlp(spec) or spec.get("kind") != _lib.POLICY_LINEAR:
            raise ValueError("CemPlan: the candidates are the b of a scheduled linear policy; an %s policy has none"
                             % ("MLP" if _is_mlp(spec) else "RBF"))
        for on, what in ((num_features is not None, "num_features (the feature sampler)"),
                         (bool(resample), "resample=True"),
                         (estimator is not None, "an estimator (estimator=%r): CEM differentiates nothing" % (estimator,))):
            if on:
                raise ValueError("CemPlan: the batched forward rollout does not combine with %s" % what)
        K, ke, iters, P, H, alpha = int(population), int(elites), int(iters), int(P), int(H), float(alpha)
        if not 1 <= K <= _lib.CEM_MAX_K:
            raise ValueError("CemPlan: population must be in 1 .. %d, got %d" % (_lib.CEM_MAX_K, K))
        if not 1 <= ke <= K:
            raise ValueError("CemPlan: elites must be in 1 .. population=%d, got %d" % (K, ke))
        if iters < 1 or P < 1 or H < 1:
            raise ValueError("CemPlan: needs iters >= 1, P >= 1 and H >= 1 (iters=%d, P=%d, H=%d)" % (iters, P, H))
        if not 0.0 <= alpha < 1.0:
            raise ValueError("CemPlan: alpha must be in [0, 1), got %r" % alpha)
        batched, _ = _schedule_check(spec, H, True)
        if batched:
            raise ValueError("CemPlan: W [Hw,U,Ds] is shared by every candidate: no leading batch dimension")
        if not spec.get("squash", True):
            raise ValueError("CemPlan: the bounds [-pi/2, pi/2] need the squashed policy u = maxa sin(b)")
        E, ang = _policy_width(dyn, spec, angles, "CemPlan")
        nz = _noise_struct(measurement_noise, E)
        self.K, self.elites, self.iters, self.alpha, self.consistent = K, ke, iters, alpha, bool(consistent)
        self._structs(dyn, spec, P, H, ang, nz, schedule=True)
        entry = lambda R, **slots: self._entry(("scheduled", "consistent" if self.consistent else "step", "batch"),
                                               R=int(R), **slots)
        if entry(1).query() == 0:
            raise ValueError("CemPlan: unsupported sizes (P=%d, H=%d, D=%d)" % (P, H, self.pr.dyn.D))
        _reward_count(reward_terms)
        Rc = _largest_fitting(lambda R: entry(R).query(), K, max_ws_bytes,
                              "CemPlan: the rollout of one candidate (P=%d, H=%d, n=%d)" % (P, H, self.pr.dyn.n))
        self._buffers(spec, reward_terms, mult_mu, (K,), False)
        pr, U, d = self.pr, self.U, device()
        pr.pol.b_bs = H * U                                     # step t: W[t], cand[r, t]
        self.value = torch.zeros(K, dtype=F64, device=d)
        self.xi = torch.zeros((iters, K, H, U), dtype=F64, device=d)
        self.mean0, self.std0 = self.b[:H].clone(), torch.zeros((H, U), dtype=F64, device=d)
        self.loop = CemLoop(K, H, U, ke, iters, alpha, CEM_BOUND, self.value, list(self.xi), self.mean0, self.std0)
        self.cand, self.mean, self.std, self.best_b = self.loop.cand, self.loop.mean, self.loop.std, self.loop.best
        self.best_value, self.trace = self.loop.best_value, self.loop.trace
        self.draw, self.updates, self.uws, self.uws_bytes = self.loop.draw, self.loop.updates, self.loop.uws, \
            self.loop.uws_bytes
        wsb = entry(Rc).query()
        self.ws = torch.empty(max(wsb // 8, 2), dtype=F64, device=d)
        pr.ws, pr.ws_bytes = self.ws.data_ptr(), wsb
        self.chunks = []                                        # the bound rollout of each chunk of candidates
        for r0 in range(0, K, Rc):
            c = _lib.Particles.from_buffer_copy(pr)
            c.pol.b = self.cand[r0].data_ptr()
            c.traj, c.act = self.traj[r0].data_ptr(), self.act_buf[r0].data_ptr()
            c.step_reward, c.step_risk = self.rew_buf[r0].data_ptr(), self.risk_buf[r0].data_ptr()
            c.ret = self.ret[r0].data_ptr()
            self.chunks.append(entry(min(Rc, K - r0), pr=c, value=self.value[r0].data_ptr()))
        self.chunk = Rc
        self.graph = None

    def set_inputs(self, x0, eps, xi, nu=None, std0=None):
        """x0 [P,E], eps [P,H,E], xi [iters,K,H,U] (iteration i's population draws xi[i]; row 0 is unread), with
        measurement noise nu [P,H,E] (required then, and only then); std0: the initial sampling std (a scalar or
        [H,U]; default (hi - lo) / 4 = pi/4)"""
        if (nu is None) != (self.nz is None):
            raise ValueError("CemPlan: nu [P,H,E] is required with measurement_noise and only then")
        self.x0.copy_(dev(x0).reshape(self.P, self.E))
        self.eps_buf.copy_(dev(eps).reshape(self.eps_buf.shape))
        self.xi.copy_(dev(xi).reshape(self.xi.shape))
        if nu is not None:
            self.nu_buf.copy_(dev(nu).reshape(self.nu_buf.shape))
        self.std0.copy_(dev(np.broadcast_to(np.asarray(0.5 * CEM_BOUND if std0 is None else std0, dtype=np.float64),
                                            (self.H, self.U)).copy()))

    def rollout(self):
        """the batched rollout of the current population: value [K] and ``outputs()``"""
        for c in self.chunks:
            c()
        return self.value

    def launch(self):
        """the whole plan on the current stream, from the initial mean and std0: no host synchronisation"""
        self.loop.launch(self.rollout)
        return self.best_b, self.best_value

    def capture(self):
        """record ``launch()`` as one CUDA graph (``CemLoop.capture``)"""
        self.graph = self.loop.capture(self.rollout)
        return self.graph

    def replay(self):
        self.graph.replay()
        return self.best_b, self.best_value

    def outputs(self):
        """(traj [K,P,H+1,E], act [K,P,H,U], step_reward [K,P,H], step_risk [K,P,H], ret [K,P]) of the last population
        rolled out"""
        return self.traj, self.act_buf, self.rew_buf, self.risk_buf, self.ret


# the batched forward-only rollouts of stationary policies (DESIGN.md section 33) per (MLP, consistent): (rollout, size
# query) after "pilco_particles_"
PARTICLE_STATIONARY_BATCH_CALLS = {
    (False, False): ("batch_rollout", "batch_workspace_bytes"),
    (False, True): ("consistent_batch_rollout", "consistent_batch_workspace_bytes"),
    (True, False): ("mlp_batch_rollout", "mlp_batch_workspace_bytes"),
    (True, True): ("mlp_consistent_batch_rollout", "mlp_consistent_batch_workspace_bytes"),
}


class ParticleBatchPlan(_Particles):
    """R stationary policies rolled out forward only over the same P particles (DESIGN.md section 33): the value of
    each, without the reverse sweep or its histories, for the cross-entropy method over policy parameters
    (``policy_opt.CemPolicySearch``).

    ``spec`` is a linear (W [R,U,Ds], b [R,U]), RBF (``gp`` factorised with a leading R) or tanh MLP (theta
    [R,n_theta]) policy spec, as ``ParticlePlan`` takes for a batch.  The plan owns x0 [P,E], eps [P,H,E] and, with
    ``measurement_noise``, nu [P,H,E], shared by the R policies and filled by ``set_inputs``; and the policies' device
    buffers under the names ``policy_opt``'s flat-row unpacking writes: ``W`` and ``b``, ``theta``, or the batched
    RBF model ``rbf``.  ``launch()`` enqueues the R rollouts (pilco_particles_batch_rollout, _consistent_batch_rollout
    with ``consistent=True``, or their MLP calls) with no host synchronisation, and returns ``value`` [R], each
    policy's mean return.

    The policies run in chunks of ``chunk`` whose workspace plus their trajectory buffers fit ``max_ws_bytes`` (default:
    half the free device memory); those buffers are the chunk's and are reused, so memory does not grow with R.  The
    restarts are independent, so the chunking changes no bit.  ``outputs()`` are the last chunk's rollouts;
    ``bytes_needed(r)`` is what a chunk of r policies needs.

    ``angles`` and ``measurement_noise``: as ``ParticlePlan``, for linear and RBF policies.  A scheduled spec, an MLP
    with angles or noise, ``num_features``, ``resample``, ``exploration``, a spec of the wrong shape, or R, P or H below 1
    is a ValueError raised before any allocation."""

    def __init__(self, dyn, spec, reward_terms, P, H, R, mult_mu=0.0, consistent=False, angles=None,
                 measurement_noise=None, max_ws_bytes=None, num_features=None, resample=False, exploration=None):
        P, H, R = int(P), int(H), int(R)
        if R < 1 or P < 1 or H < 1:
            raise ValueError("ParticleBatchPlan: needs R >= 1, P >= 1 and H >= 1 (R=%d, P=%d, H=%d)" % (R, P, H))
        if isinstance(spec, dict) and spec.get("schedule", False):
            raise ValueError("ParticleBatchPlan: the policies are stationary; a time-varying linear policy (a schedule) "
                             "runs in engine.CemPlan")
        for on, what in ((num_features is not None, "num_features (the feature sampler)"),
                         (bool(resample), "resample=True"), (exploration is not None, "exploration")):
            if on:
                raise ValueError("ParticleBatchPlan: the batched forward rollout does not combine with %s" % what)
        mlp = _particle_mlp(spec, "ParticleBatchPlan", R, angles, measurement_noise)
        E, ang = _policy_width(dyn, spec, angles, "ParticleBatchPlan")
        Ds, U, kind = int(spec["Ds"]), int(spec["U"]), spec["kind"]
        if kind == _lib.POLICY_LINEAR:
            if np.shape(spec["W"]) != (R, U, Ds) or np.shape(spec["b"]) != (R, U):
                raise ValueError("ParticleBatchPlan: expected W [R,U,Ds] = %s and b [R,U] = %s, got %s and %s"
                                 % ((R, U, Ds), (R, U), np.shape(spec["W"]), np.shape(spec["b"])))
        elif kind == _lib.POLICY_RBF:
            g = spec["gp"]
            if not g.batched or tuple(g.X.shape[:1]) != (R,) or g.D != Ds or g.E != U:
                raise ValueError("ParticleBatchPlan: the RBF policy must be factorised with a leading R=%d, Ds=%d "
                                 "inputs and U=%d outputs" % (R, Ds, U))
        elif mlp is None:
            raise ValueError("ParticleBatchPlan: unknown policy kind %r" % (kind,))
        nz = _noise_struct(measurement_noise, E)
        _reward_count(reward_terms)
        self.R, self.Ds, self.consistent = R, Ds, bool(consistent)
        self._structs(dyn, spec, P, H, ang, nz, mlp=mlp, batched=True)
        entry = lambda r, **slots: self._entry(("mlp" if mlp is not None else "plain",
                                                "consistent" if self.consistent else "step", "batch"), R=int(r),
                                               **slots)
        if entry(1).query() == 0:
            raise ValueError("ParticleBatchPlan: unsupported sizes (P=%d, H=%d, D=%d)" % (P, H, self.pr.dyn.D))
        per = 8 * P * ((H + 1) * E + H * U + 2 * H + 1)          # one restart's trajectory buffers, in bytes
        self.bytes_needed = lambda r: q + r * per if (q := entry(r).query()) else 0
        Rc = _largest_fitting(self.bytes_needed, R, max_ws_bytes, "ParticleBatchPlan: the rollout of one policy (P=%d, "
                              "H=%d, n=%d)" % (P, H, self.pr.dyn.n))
        self._buffers(spec, reward_terms, mult_mu, (Rc,), True)
        pr, d = self.pr, device()
        self.value = torch.zeros(R, dtype=F64, device=d)
        wsb = entry(Rc).query()
        self.ws = torch.empty(max(wsb // 8, 2), dtype=F64, device=d)
        pr.ws, pr.ws_bytes = self.ws.data_ptr(), wsb
        self.chunk, self.chunks = Rc, []                        # the bound rollout of each chunk
        for r0 in range(0, R, Rc):
            c, m = _lib.Particles.from_buffer_copy(pr), None
            if self.mlp is not None:
                m = _lib.Mlp.from_buffer_copy(self.mlp)
                m.theta = self.theta[r0].data_ptr()
            elif kind == _lib.POLICY_LINEAR:
                c.pol.W, c.pol.b = self.W[r0].data_ptr(), self.b[r0].data_ptr()
            else:
                g = self.rbf
                c.pol.rbf.X, c.pol.rbf.ell = g.X[r0].data_ptr(), g.ell[r0].data_ptr()
                c.pol.rbf.sf2, c.pol.rbf.beta = g.sf2[r0].data_ptr(), g.beta[r0].data_ptr()
            self.chunks.append(entry(min(Rc, R - r0), pr=c, mlp=m, value=self.value[r0].data_ptr()))

    def set_inputs(self, x0, eps, nu=None):
        """x0 [P,E], eps [P,H,E] and, with measurement noise, nu [P,H,E] (required then, and only then)"""
        if (nu is None) != (self.nz is None):
            raise ValueError("ParticleBatchPlan: nu [P,H,E] is required with measurement_noise and only then")
        self.x0.copy_(dev(x0).reshape(self.P, self.E))
        self.eps_buf.copy_(dev(eps).reshape(self.eps_buf.shape))
        if nu is not None:
            self.nu_buf.copy_(dev(nu).reshape(self.nu_buf.shape))

    def launch(self):
        """the R rollouts on the current stream, chunk by chunk: no host synchronisation -> value [R]"""
        for c in self.chunks:
            c()
        return self.value

    def outputs(self):
        """(traj [Rc,P,H+1,E], act [Rc,P,H,U], step_reward [Rc,P,H], step_risk [Rc,P,H], ret [Rc,P]) of the last chunk
        rolled out (Rc = ``chunk``; the first R - r0 rows of a shorter last chunk)"""
        return self.traj, self.act_buf, self.rew_buf, self.risk_buf, self.ret


def _device_tensor(t, dtype, what):
    if not isinstance(t, torch.Tensor) or t.dtype != dtype or not t.is_cuda or not t.is_contiguous():
        raise ValueError("%s must be a contiguous %s CUDA tensor" % (what, dtype))


def normals(out, seed, stream_id, iter):
    """pilco_normals (DESIGN.md section 32): fill ``out`` (a contiguous fp64 CUDA tensor) with standard normals, each a
    pure function of (seed, stream_id, iteration, its index): Philox4x32-10 and Box-Muller.  The iteration is read from
    ``iter`` (an int64 CUDA tensor of one element) when the kernel runs, so a captured graph draws new normals at every
    replay once something advances it (``AdamState.step``).  seed is taken modulo 2^64; stream_id must be in
    0 .. 2^32 - 1.  The first k elements do not depend on out's size.  Returns out; ValueError before any device work
    for a bad tensor or stream_id."""
    _device_tensor(out, F64, "normals: out")
    if not isinstance(iter, torch.Tensor) or iter.dtype != torch.int64 or iter.numel() != 1 or not iter.is_cuda:
        raise ValueError("normals: iter must be an int64 CUDA tensor of one element")
    if not 0 <= int(stream_id) < 2 ** 32:
        raise ValueError("normals: stream_id must be in 0 .. 2^32 - 1, got %d" % int(stream_id))
    check(lib.pilco_normals(int(seed) % 2 ** 64, int(stream_id), iter.data_ptr(), out.numel(), out.data_ptr(),
                            stream_ptr()), "normals")
    return out


def adam_hyperparameters(lr, betas, eps, max_norm):
    """(lr, b1, b2, eps, max_norm) as pilco_adam_update takes them, max_norm None -> 0 (no clipping); ValueError
    outside its ranges: lr > 0 finite, b1 and b2 in [0, 1), eps > 0, max_norm >= 0"""
    lr, eps = float(lr), float(eps)
    b1, b2 = (float(b) for b in betas)
    max_norm = 0.0 if max_norm is None else float(max_norm)
    for bad, what in ((not (0.0 < lr < float("inf")), "learning_rate must be finite and > 0"),
                      (not (0.0 <= b1 < 1.0 and 0.0 <= b2 < 1.0), "betas must be in [0, 1)"),
                      (not eps > 0.0, "eps must be > 0"), (not max_norm >= 0.0, "max_grad_norm must be >= 0")):
        if bad:
            raise ValueError("adam: %s (learning_rate=%r, betas=%r, eps=%r, max_grad_norm=%r)"
                             % (what, lr, tuple(betas), eps, max_norm))
    return lr, b1, b2, eps, max_norm


class AdamState:
    """Adam's state for R restarts of n flat parameters on the device (pilco_adam_update, DESIGN.md section 32): the
    moments ``m``, ``v`` [R,n], the step counts ``t`` [R], the running products ``b1t``, ``b2t`` [R], the iteration
    counter ``iter`` [1] (int64: ``normals`` reads it), and ``trace`` / ``ok`` [trace_rows,R], iteration k's -loss and
    whether it stepped.  ``step(theta, packed)`` enqueues one update of theta [R,>=n] from the rows packed [R,>=n+2] =
    [loss | status | gradient of loss], then advances the counter: no host synchronisation, graph-capturable.
    ``reset()`` restores the start (zero moments, counts and counter, unit products, a NaN trace).  Hyper-parameters
    out of range are a ValueError (``adam_hyperparameters``) raised before any allocation."""

    def __init__(self, R, n, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, max_norm=None, trace_rows=0):
        self.lr, self.b1, self.b2, self.eps, self.max_norm = adam_hyperparameters(lr, betas, eps, max_norm)
        self.R, self.n, self.trace_rows = int(R), int(n), int(trace_rows)
        if self.R < 1 or self.n < 1 or self.trace_rows < 0:
            raise ValueError("AdamState: needs R >= 1, n >= 1 and trace_rows >= 0 (R=%d, n=%d, trace_rows=%d)"
                             % (self.R, self.n, self.trace_rows))
        d, R, rows = device(), self.R, max(self.trace_rows, 1)
        mk = lambda *shape, dtype=F64: torch.zeros(shape, dtype=dtype, device=d)
        self.m, self.v, self.b1t, self.b2t, self.trace = mk(R, self.n), mk(R, self.n), mk(R), mk(R), mk(rows, R)
        self.t, self.iter, self.ok = mk(R, dtype=torch.int64), mk(1, dtype=torch.int64), mk(rows, R, dtype=torch.int32)
        self.reset()

    def reset(self):
        for z in (self.m, self.v, self.t, self.iter, self.ok):
            z.zero_()
        self.b1t.fill_(1.0)
        self.b2t.fill_(1.0)
        self.trace.fill_(float("nan"))

    def step(self, theta, packed):
        for a, w, what in ((theta, self.n, "theta"), (packed, self.n + 2, "packed")):
            if not isinstance(a, torch.Tensor) or a.dtype != F64 or not a.is_cuda or a.dim() != 2 or \
                    a.shape[0] != self.R or a.shape[1] < w or a.stride(1) != 1:
                raise ValueError("AdamState.step: %s must be an fp64 CUDA tensor [%d, >=%d] with unit column stride"
                                 % (what, self.R, w))
        a = _lib.Adam(self.R, self.n, self.lr, self.b1, self.b2, self.eps, self.max_norm, theta.data_ptr(),
                      theta.stride(0), packed.data_ptr(), packed.stride(0), self.m.data_ptr(), self.v.data_ptr(),
                      self.t.data_ptr(), self.b1t.data_ptr(), self.b2t.data_ptr(), self.iter.data_ptr(),
                      self.trace.data_ptr(), self.ok.data_ptr(), self.trace_rows)
        check(lib.pilco_adam_update(C.byref(a), stream_ptr()), "adam_update")


class PredictPlan:
    """``PILCO.predict(m, S, n)`` as ONE graph launch: host moments -> device, n-step cascade (R = 1), final
    moments + reward + status -> pinned host memory.  Built once per (model, policy, reward, n) state by
    ``PILCO`` and replayed for every call with new initial moments (pilco/models/pilco.py:118-136)."""

    def __init__(self, dyn, policy_spec, reward_terms, Ds, n, mult_mu=0.0, angles=None, measurement_noise=None,
                 schedule=False):
        """``Ds``: the state dimension (the dynamics GP's outputs); ``angles``, ``measurement_noise``, ``schedule``: as
        RolloutPlan."""
        _refuse_mlp(policy_spec, "PredictPlan")
        d = device()
        self.Ds, self.n = int(Ds), int(n)
        Ds = self.Ds
        self.h_in = torch.zeros(Ds + Ds * Ds, dtype=F64).pin_memory()
        self.h_out = torch.zeros(Ds + Ds * Ds + 2, dtype=F64).pin_memory()       # [m | S | reward | info]
        self.d_in = torch.zeros(Ds + Ds * Ds, dtype=F64, device=d)
        self.d_out = torch.zeros(Ds + Ds * Ds + 2, dtype=F64, device=d)
        self.plan = RolloutPlan(dyn, policy_spec, reward_terms, np.zeros(Ds), np.eye(Ds), self.n, R=1, mult_mu=mult_mu,
                                angles=angles, measurement_noise=measurement_noise, schedule=schedule)
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
        _refuse_mlp(policy_spec, "ActionPlan")
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
