/*
 * pilco_b200.h -- C ABI of the H100-native PILCO moment-matching rollout engine.
 *
 * The reference (nrontsis/PILCO) has no FFI: its hot path is TensorFlow ops composed in Python.
 * This ABI is therefore the boundary placed directly beneath the reference's Python class API;
 * each entry point names the reference function (file:line in nrontsis/PILCO) it replaces.
 *
 * Rules (all entry points):
 *   - every pointer is a DEVICE pointer to contiguous fp64 (or int32 for `info`), owned by the caller
 *     (PyTorch allocates them); the library never allocates or frees device memory;
 *   - work is only enqueued on the `stream` argument; no entry point synchronises the device
 *     (so every `*_forward/_backward/rollout` call is CUDA-graph capturable);
 *   - return value: 0 ok, <0 invalid argument (see pilco_status_string); numerical failures
 *     (non-PD matrices) are reported per batch element in the device `info` array
 *     (0 ok, bit0: input outside the moment match's domain -- see pilco_mm_forward --, bit1: non-PD Gram matrix);
 *   - batch dimension R = independent rollouts ("policy restarts", pilco/models/pilco.py:98-107);
 *   - matrices are row-major; `*_bs` arguments are batch strides in doubles (0 = one array shared
 *     by all R batch elements).
 */
#ifndef PILCO_B200_H
#define PILCO_B200_H

#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

#define PILCO_ABI_VERSION 3
#define PILCO_MAX_D 16          /* max GP input dimension (state+control) */
#define PILCO_MAX_E 16          /* max number of GP outputs */

typedef void* pilco_stream_t;   /* cudaStream_t */

/* ---- ABI / sizing ------------------------------------------------------------------------- */
int         pilco_version(void);
const char* pilco_status_string(int status);
/* rows/cols of every per-centre array are padded to a multiple of 64 */
int         pilco_pad_n(int n);
/* workspace bytes for pilco_mm_forward / pilco_mm_backward with these sizes */
size_t      pilco_mm_workspace_bytes(int n, int D, int E, int R);

/* ---- moment matching ------------------------------------------------------------------------
 * Replaces MGPR.predict_given_factorizations (pilco/models/mgpr.py:91-149; MATLAB gp0.m:63-104,
 * gp1.m:85-124, gp2.m:69-106): Gaussian input N(m,s) -> predictive mean M, covariance S and
 * V = inv(s) * input-output covariance, for E independent SE-ARD GPs over n centres.
 */
typedef struct pilco_gp_model {
    int n, D, E;
    int mode;               /* 0: GP with trace term, +sf2 on diag(S) (mgpr.py:143-147);
                               1: deterministic GP / RBF network: no trace term, +1e-6
                                  (controllers.py:116-117, gp2.m:96-99) */
    const double* X;    long long X_bs;     /* [n,D] centres (training inputs / inducing points / RBF centres) */
    const double* ell;  long long ell_bs;   /* [E,D] lengthscales */
    const double* sf2;  long long sf2_bs;   /* [E] signal variances */
    const double* beta; long long beta_bs;  /* [E,n] (K+sn2 I)^-1 y */
    const double* iK;   int ldk;            /* [E,ldk,ldk] (K+sn2 I)^-1, zero padded, ldk >= pilco_pad_n(n);
                                               NULL when mode==1.  Shared by the batch. */
} pilco_gp_model;

/* Moment match of N(m, s) through the GP.  Domain, checked on the device per batch element and reported as info bit0
 * (the outputs of a flagged element are not meaningful):
 *   - every length-scale lies in (0, inf): zero, negative, infinite and NaN length-scales are flagged (only ell^2
 *     enters the formulas, but a negative length-scale is taken for a caller's error, not for its absolute value);
 *   - s (its symmetric part is used) is positive semi-definite up to PILCO_MM_PSD_TOL: s = 0 and singular s are valid
 *     inputs; an eigenvalue below -PILCO_MM_PSD_TOL x max_i |s_ii| is flagged, as is a NaN;
 *   - s + diag(ell_a^2) and s + diag(1 / (ell_a^-2 + ell_b^-2)) are positive definite (implied by the above).
 * The same holds for pilco_mm_forward_taped and for the dynamics step of pilco_rollout.  pilco_mm_backward has no info
 * output: call it with inputs a forward call has accepted. */
#define PILCO_MM_PSD_TOL 1e-6
int pilco_mm_forward(const pilco_gp_model* gp, int R,
                     const double* m,       /* [R,D]   */
                     const double* s,       /* [R,D,D] */
                     double* M,             /* [R,E]   */
                     double* S,             /* [R,E,E] */
                     double* V,             /* [R,D,E] */
                     int* info,             /* [R] or NULL */
                     void* ws, size_t ws_bytes, pilco_stream_t stream);

/* VJP of pilco_mm_forward (the reference differentiates mgpr.py:91-149 with TensorFlow autodiff inside
 * gpflow.optimizers.Scipy, pilco/models/pilco.py:84-90).  Inputs: the forward inputs m, s, the forward output
 * M and the cotangents gM [R,E], gS [R,E,E], gV [R,D,E].  Outputs gm [R,D], gs [R,D,D] (symmetric part) and,
 * when all three pointers are non-NULL (trainable RBF policy), gX [R,n,D], gbeta [R,E,n], gell [R,E,D]. */
size_t pilco_mm_bwd_workspace_bytes(int n, int D, int E, int R, int need_param);
int pilco_mm_backward(const pilco_gp_model* gp, int R, const double* m, const double* s, const double* M,
                      const double* gM, const double* gS, const double* gV,
                      double* gm, double* gs, double* gX, double* gbeta, double* gell,
                      void* ws, size_t ws_bytes, pilco_stream_t stream);

/* Taped moment match: pilco_mm_forward that also leaves, per unordered output pair (a,b), the row sums, column sums
 * and the product (G_ab o L'_ab) Z of the N x N matrix it has in registers anyway (Z = centred inputs) on a tape;
 * pilco_mm_backward_taped turns the tape and the cotangents into gm, gs WITHOUT recomputing an exponential.
 * Only the cotangents of the input moments are produced (the dynamics GP of the policy objective, whose inputs
 * and hyper-parameters are constants, pilco/models/pilco.py:80-82); trainable centres need pilco_mm_backward. */
size_t pilco_mm_tape_bytes(int n, int D, int E, int R);          /* 0: shape not supported (n > 1024 for D <= 12, n > 704 beyond) */
size_t pilco_mm_tape_bwd_workspace_bytes(int D, int E, int R);
int pilco_mm_forward_taped(const pilco_gp_model* gp, int R, const double* m, const double* s,
                           double* M, double* S, double* V, int* info,
                           void* ws, size_t ws_bytes, void* tape, size_t tape_bytes, pilco_stream_t stream);
int pilco_mm_backward_taped(const pilco_gp_model* gp, int R, const double* m, const double* s, const double* M,
                            const double* gM, const double* gS, const double* gV,
                            const void* tape, size_t tape_bytes, double* gm, double* gs,
                            void* ws, size_t ws_bytes, pilco_stream_t stream);

/* ---- GP factorisation -----------------------------------------------------------------------
 * Replaces MGPR.calculate_factorizations (pilco/models/mgpr.py:81-89; gp0.m:46-61):
 * K_e = sf2_e exp(-0.5 |(x-x')/ell_e|^2); L = chol(K + sn2_e I); iK = (K+sn2 I)^-1; beta = iK y_e.
 * B batch elements (B=1 for the dynamics GP; B=R for per-restart RBF policies).
 * iK is written with leading dimension ldk (zero padded; pass NULL to get beta only).
 * ws: scratch of pilco_gp_factorize_workspace_bytes(n, E, B) bytes; on return its first
 * B*E*ldw*ldw doubles (ldw = pilco_pad_n(n)) hold the Cholesky factors L (lower triangles), which
 * pilco_rollout_backward needs for the RBF policy (pilco_rollout_grad.pol_L).
 */
size_t pilco_gp_factorize_workspace_bytes(int n, int E, int B);
int pilco_gp_factorize(int n, int D, int E, int B,
                       const double* X,   long long X_bs,    /* [n,D]  */
                       const double* Y,   long long Y_bs,    /* [n,E]  */
                       const double* ell, long long ell_bs,  /* [E,D]  */
                       const double* sf2, long long sf2_bs,  /* [E]    */
                       const double* sn2, long long sn2_bs,  /* [E]    */
                       double* iK, int ldk,                  /* [B,E,ldk,ldk] or NULL */
                       double* beta,                         /* [B,E,n] */
                       int* info,                            /* [B] or NULL */
                       void* ws, size_t ws_bytes, pilco_stream_t stream);

/* Incremental set_data (SURVEY section 8f-2): k rows appended to the data of a factorised model with UNCHANGED
 * hyper-parameters (pilco/models/mgpr.py:38-45; examples/inv_double_pendulum.py:102-103, swimmer.py:87-88 append the
 * rows of each new episode).  X [n0+k, D] and Y [n0+k, E] hold the old rows first; iK_old [E,ldk_old,ldk_old] is the
 * inverse pilco_gp_factorize / an earlier append produced.  Writes the new zero-padded inverse iK_new
 * [E,ldk_new,ldk_new] (ldk_new >= pilco_pad_n(n0+k), out of place) and beta_new [E,n0+k] by the block-inverse
 * (Schur complement) update: O(n^2 k) instead of O(n^3).  info[0] bit 1: Schur complement not positive definite. */
size_t pilco_gp_append_workspace_bytes(int n0, int k, int E);
int pilco_gp_append(int n0, int k, int D, int E,
                    const double* X, const double* Y,
                    const double* ell, const double* sf2, const double* sn2,
                    const double* iK_old, int ldk_old,
                    double* iK_new, int ldk_new, double* beta_new, int* info,
                    void* ws, size_t ws_bytes, pilco_stream_t stream);

/* GP training objective (SURVEY section 8f-1): nlml[b,e] = -log p(y_e | X, theta_be) and its gradient w.r.t. the
 * constrained hyper-parameters, batched over B hyper-parameter sets x E outputs.  Replaces
 * gpflow.models.GPR.training_loss + TF autodiff inside MGPR.optimize (pilco/models/mgpr.py:47-75); the Gamma priors
 * of mgpr.py:33-34 are added by the host.  Outputs nlml [B,E], g_ell [B,E,D], g_sf2 [B,E], g_sn2 [B,E]. */
size_t pilco_gp_nlml_workspace_bytes(int n, int E, int B);
int pilco_gp_nlml(int n, int D, int E, int B,
                  const double* X,   long long X_bs, const double* Y,   long long Y_bs,
                  const double* ell, long long ell_bs, const double* sf2, long long sf2_bs,
                  const double* sn2, long long sn2_bs,
                  double* nlml, double* g_ell, double* g_sf2, double* g_sn2, int* info,
                  void* ws, size_t ws_bytes, pilco_stream_t stream);

/* FITC training objective (SURVEY section 8f-1, sparse half): value and gradient of the collapsed FITC bound
 * (gpflow.models.GPRFITC.training_loss as SMGPR.optimize minimises it, pilco/models/smgpr.py:16-22 via
 * mgpr.py:47-75; no priors) w.r.t. the constrained hyper-parameters AND the inducing inputs, batched over B
 * parameter sets x E outputs -- every output trains its own Z [Mi,D].  X [N,D], Y [N,E] are shared by the batch;
 * Z [B,E,Mi,D], ell [B,E,D], sf2/sn2 [B,E].  Outputs nlml [B,E], g_ell [B,E,D], g_sf2, g_sn2 [B,E], g_Z [B,E,Mi,D].
 * info[b] bit 1: a Cholesky factorisation (Kuu + 1e-6 I, or I + V diag(1/nu) V') failed. */
size_t pilco_fitc_nlml_workspace_bytes(int N, int Mi, int D, int E, int B);
int pilco_fitc_nlml(int N, int Mi, int D, int E, int B,
                    const double* X, const double* Y, const double* Z,
                    const double* ell, const double* sf2, const double* sn2,
                    double* nlml, double* g_ell, double* g_sf2, double* g_sn2, double* g_Z, int* info,
                    void* ws, size_t ws_bytes, pilco_stream_t stream);

/* Replaces SMGPR.calculate_factorizations (pilco/models/smgpr.py:24-45; gp1.m:52-82): FITC over
 * Mi inducing points Z.  Outputs iK[E,ldk,ldk] (zero padded) and beta[E,Mi].
 * ws: scratch of pilco_fitc_workspace_bytes(N, Mi, E) bytes. */
size_t pilco_fitc_workspace_bytes(int N, int Mi, int E);
int pilco_fitc_factorize(int N, int Mi, int D, int E,
                         const double* X,   /* [N,D]  */
                         const double* Z,   /* [Mi,D] */
                         const double* Y,   /* [N,E]  */
                         const double* ell, const double* sf2, const double* sn2,
                         double* iK, int ldk, double* beta,
                         int* info, void* ws, size_t ws_bytes, pilco_stream_t stream);

/* ---- prediction at deterministic inputs -------------------------------------------------------
 * Stands in for gpflow GPR.predict_f / GPRFITC.predict_f, which the reference's users call on the output models of
 * MGPR / SMGPR (pilco/models/mgpr.py:28-36, smgpr.py:16-22) to check the learnt dynamics: the posterior of outputs
 * e0 .. e0+ne-1 of an unbatched mode-0 model with iK (pilco_gp_factorize, pilco_gp_append or pilco_fitc_factorize) at
 * T inputs Xs [T,D]:  mean = k*' beta_e,  var = sf2_e - k*' iK_e k*  (latent f; the caller adds sn2 for y), or with
 * full_cov the [ne,T,T] covariance K** - K* iK_e K*'.  A point's mean and variance do not depend on T, on its row in
 * Xs or on which outputs are requested (fixed-order reductions; diagonal path).  PILCO_ERR_UNSUPPORTED: mode != 0,
 * no iK, or a batched model; PILCO_ERR_ALIGN: iK or ws not 16-byte aligned, or ldk odd. */
size_t pilco_gp_predict_workspace_bytes(int n, int D, int E, int T, int full_cov);   /* 0: unsupported arguments */
int    pilco_gp_predict(const pilco_gp_model* gp, int e0, int ne, int T,
                        const double* Xs,      /* [T,D] deterministic inputs */
                        double* mean,          /* [T,ne] */
                        double* var,           /* full_cov ? [ne,T,T] : [T,ne] */
                        int full_cov, void* ws, size_t ws_bytes, pilco_stream_t stream);
/* Posterior function samples at the same inputs (gpflow GPModel.predict_f_samples), given the caller's standard normals:
 *   full_cov = 1:  samples[s,:,e] = mean_e + L_e eps[s,:,e],  L_e = chol(cov_e + jitter I)  (pilco_gp_predict's covariance)
 *   full_cov = 0:  samples[s,t,e] = mean[t,e] + sqrt(max(var[t,e], 0)) eps[s,t,e]           (jitter unused)
 * Same models, validation, status codes and T limits as pilco_gp_predict, plus PILCO_ERR_DIM for S < 1 or a negative
 * or non-finite jitter.  info[e] is set on the stream: nonzero where cov_e + jitter I is not positive definite (always 0
 * for full_cov = 0).  Workspace (0: unsupported sizes or size_t overflow):
 *   full_cov = 0:  pilco_gp_predict's (rounded up to 16 bytes) + 2 T ne doubles  -- O(T)
 *   full_cov = 1:  max(pilco_gp_predict's, 2 S T ne doubles) + ne T^2 + T ne doubles
 * No host synchronisation (graph-capturable).  The first S' samples do not depend on S. */
size_t pilco_gp_predict_samples_workspace_bytes(int n, int D, int E, int T, int S, int full_cov);
int    pilco_gp_predict_samples(const pilco_gp_model* gp, int e0, int ne, int T, int S,
                                const double* Xs,      /* [T,D]     */
                                const double* eps,     /* [S,T,ne]  standard normals */
                                double* samples,       /* [S,T,ne]  */
                                int full_cov, double jitter,
                                int* info,             /* [ne] */
                                void* ws, size_t ws_bytes, pilco_stream_t stream);
/* Vector-Jacobian product of the diagonal posterior of ALL E outputs at the inputs:
 *   gXs[t] = d/dXs[t] sum_e (gmean[t,e] mean_e(Xs[t]) + gvar[t,e] var_e(Xs[t]))
 * over the same models and with the same validation and limits as pilco_gp_predict (full_cov = 0).  A point's result
 * does not depend on T or on its row in Xs (fixed-order reductions). */
size_t pilco_gp_predict_vjp_workspace_bytes(int n, int D, int E, int T);             /* 0: unsupported arguments */
int    pilco_gp_predict_vjp(const pilco_gp_model* gp, int T,
                            const double* Xs,      /* [T,D] */
                            const double* gmean,   /* [T,E] */
                            const double* gvar,    /* [T,E] */
                            double* gXs,           /* [T,D] */
                            void* ws, size_t ws_bytes, pilco_stream_t stream);

/* ---- closed-form moments ---------------------------------------------------------------------
 * squash_sin (pilco/controllers.py:13-36; gSin.m:33-48), LinearController.compute_action
 * (controllers.py:46-58; conlin.m:50-62), ExponentialReward.compute_reward (rewards.py:19-51;
 * reward.m:35-57).  All batched over R.
 */
int pilco_squash_sin(int U, int R, const double* m /*[R,U]*/, const double* s /*[R,U,U]*/,
                     const double* max_action /*[U]*/,
                     double* M /*[R,U]*/, double* S /*[R,U,U]*/, double* C /*[R,U,U]*/,
                     pilco_stream_t stream);

int pilco_linear_action(int Ds, int U, int R,
                        const double* W, long long W_bs,   /* [U,Ds] */
                        const double* b, long long b_bs,   /* [U]    */
                        const double* m /*[R,Ds]*/, const double* s /*[R,Ds,Ds]*/,
                        double* M /*[R,U]*/, double* S /*[R,U,U]*/, double* V /*[R,Ds,U]*/,
                        pilco_stream_t stream);

/* Ds is the dimension of whatever Gaussian is handed in: the state's, or D = Ds + U for joint state-action moments
 * (the closed form of PILCO_REWARD_EXP_SA). */
int pilco_exp_reward(int Ds, int R, const double* W /*[Ds,Ds]*/, const double* t /*[Ds]*/,
                     const double* m /*[R,Ds]*/, const double* s /*[R,Ds,Ds]*/,
                     double* muR /*[R]*/, double* sR /*[R] or NULL*/, int* info,
                     pilco_stream_t stream);

/* Safe-PILCO risk rewards (safe_pilco_extension/rewards_safe.py:13-58: RiskOfCollision.compute_reward,
 * SingleConstraint.compute_reward): probability that the constrained state dimensions lie inside a box,
 * each dimension an independent univariate normal with loc m[d] and scale sfac*s[d,d] (as the reference
 * writes it).  prm (device, doubles) = [nd, inside, sfac, (dim_k, low_k, high_k) x nd]; a missing bound is
 * +-inf; inside = 0 returns the complement.  Optional d risk/d m [R,Ds] and d risk/d diag(s) [R,Ds]. */
int pilco_box_risk(int Ds, int R, const double* prm, const double* m /*[R,Ds]*/, const double* s /*[R,Ds,Ds]*/,
                   double* risk /*[R]*/, double* drisk_dm /*[R,Ds] or NULL*/, double* drisk_dv /*[R,Ds] or NULL*/,
                   pilco_stream_t stream);

/* ---- H-step rollout ---------------------------------------------------------------------------
 * Replaces PILCO.predict / PILCO.propagate (pilco/models/pilco.py:118-153; pred.m:29-39,
 * propagate.m:33-85): policy moments -> joint state/action Gaussian -> dynamics moment match ->
 * next state; the expected reward is accumulated at the pre-step state (pilco.py:130-134).
 */
#define PILCO_POLICY_LINEAR 0
#define PILCO_POLICY_RBF    1
#define PILCO_REWARD_EXP    0
#define PILCO_REWARD_LINEAR 1
#define PILCO_REWARD_BOX    2   /* pilco_box_risk; W = its prm block, t unused */
/* Terms on the joint Gaussian of the state and the APPLIED action, x~_t = [x_t, u_t] (D = Ds + U): term k at step t
 * (t = 0 .. H-1) is evaluated at the (m~, s~) handed to the dynamics moment match of step t, i.e. u_t after squash_sin
 * when pol.squash.  The final state x_H has no action and gets no joint term.  Control-effort costs live here.
 * Within a step the state terms are accumulated first, in order, then the joint terms, in order (every path). */
#define PILCO_REWARD_EXP_SA     3   /* exp(-1/2 (x~-t)' W (x~-t)) moments over the joint:  W [D,D], t [D] */
#define PILCO_REWARD_LINEAR_SA  4   /* x~' W:  W [D] */
/* accumulation channel of a reward term (safe_pilco_extension/safe_pilco.py:29-50, SafePILCO.predict):
 *   ADD : reward_add  += coef * value(x_t)                       (PILCO.predict, pilco.py:130-134)
 *   MULT: reward_mult *= 1 - sum_k coef_k * value_k(x_t)          (the terms of this channel form the risk)
 * and the rollout returns  reward = reward_add + mult_mu * (1 - reward_mult). */
#define PILCO_CHANNEL_ADD   0
#define PILCO_CHANNEL_MULT  1

typedef struct pilco_policy {
    int kind;                   /* PILCO_POLICY_* */
    int Ds, U;
    int squash;                 /* 1: squash_sin with max_action */
    const double* max_action;   /* [U] */
    /* linear (controllers.py:39-63) */
    const double* W; long long W_bs;   /* [U,Ds] */
    const double* b; long long b_bs;   /* [U]    */
    /* RBF (controllers.py:80-129): deterministic GP over bf centres; beta from pilco_gp_factorize */
    pilco_gp_model rbf;
} pilco_policy;

typedef struct pilco_reward_term {
    int kind;                   /* PILCO_REWARD_* */
    int channel;                /* PILCO_CHANNEL_* */
    double coef;                /* CombinedRewards weight (rewards.py:64-81) */
    const double* W;            /* exp: [Ds,Ds]; linear: [Ds]; box: prm block; exp_sa: [D,D]; linear_sa: [D] */
    const double* t;            /* exp: [Ds] target; exp_sa: [D] target; otherwise unused */
} pilco_reward_term;

typedef struct pilco_rollout {
    int R, H;
    pilco_gp_model dyn;         /* D = Ds+U, E = Ds */
    pilco_policy   pol;
    int n_rewards;
    pilco_reward_term rewards[8];
    const double* m0; long long m0_bs;   /* [Ds]    initial state mean  */
    const double* S0; long long S0_bs;   /* [Ds,Ds] initial state cov   */
    /* outputs */
    double* traj_m;             /* [R,H+1,Ds]    state means, t=0..H   */
    double* traj_S;             /* [R,H+1,Ds,Ds] state covariances      */
    double* reward;             /* [R] sum_{t<H} E[r(x_t)]  (+ mult_mu (1 - prod_t (1 - risk_t)))  */
    double* step_reward;        /* [R,H] or NULL                        */
    int* info;                  /* [R]                                   */
    void* ws; size_t ws_bytes;
    double mult_mu;             /* SafePILCO.mu (safe_pilco.py:26,49); ignored without MULT terms */
    double* step_risk;          /* [R,H] per-step risk of the MULT channel, or NULL */
    /* Tape of the dynamics moment match (pilco_rollout_tape_bytes, 16-byte aligned) or NULL.  With a tape the forward
     * cascade runs the TAPED tile pass (pilco_mm_forward_taped) at every step and pilco_rollout_backward consumes
     * the tape instead of recomputing any N x N exponential: forward+backward cost ~1.9 forward tile passes instead
     * of ~5.  Without it pilco_rollout_backward recomputes (memory-lean path, same results). */
    void* tape; size_t tape_bytes;
} pilco_rollout;

size_t pilco_rollout_workspace_bytes(const pilco_rollout* ro);
size_t pilco_rollout_tape_bytes(const pilco_rollout* ro);   /* 0: shape not supported by the taped pass (n > 1024 centres for D <= 12, > 704 beyond) */
int    pilco_rollout_forward(const pilco_rollout* ro, pilco_stream_t stream);

/* Reverse sweep: gradient of ro->reward[r] (= sum_t E[r(x_t)], the negative of PILCO.training_loss,
 * pilco/models/pilco.py:47-50) with respect to the policy parameters.  Must follow pilco_rollout_forward
 * with the same `ro` (the per-step joint Gaussians it saved in ro->ws are re-used).
 * Linear policy: gW [R,U,Ds], gb [R,U].  RBF policy: gXc [R,bf,Ds] centres, gYc [R,bf,U] targets,
 * gell [R,U,Ds] lengthscales (constrained), pol_L = Cholesky factors left by pilco_gp_factorize. */
typedef struct pilco_rollout_grad {
    double* gW; double* gb;
    double* gXc; double* gYc; double* gell;
    const double* pol_L;
    double* gm0; double* gS0;       /* optional: gradient w.r.t. the initial state moments [R,Ds],[R,Ds,Ds] */
    void* ws; size_t ws_bytes;
} pilco_rollout_grad;

size_t pilco_rollout_bwd_workspace_bytes(const pilco_rollout* ro);
int    pilco_rollout_backward(const pilco_rollout* ro, const pilco_rollout_grad* g, pilco_stream_t stream);

/* ---- particle rollout -------------------------------------------------------------------------
 * Monte Carlo check of the moment-matching cascade (nothing in the reference; the PILCO papers validate moment
 * matching against particle rollouts of the same model).  P particles follow the Markov chain whose Gaussian
 * marginals pilco_rollout_forward approximates, with the caller's standard normals eps:
 *   u_t = pi(x_t)  (linear: W x + b; RBF: sum_i beta_i k(x, c_i), the mean action at a point), squashed as
 *         squash_sin does at the policy's output variance (0 linear, 1e-6 RBF, as compute_action),
 *   x_{t+1} = x_t + mu(x~_t) + sqrt(max(var(x~_t), 0)) o eps_t,  x~_t = [x_t, u_t]  (latent posterior, no noise),
 *   step_reward / step_risk = the ADD / MULT terms at the point x_t (t < H), ret = sum_t step_reward
 *   (+ mult_mu (1 - prod_t (1 - step_risk)) with MULT terms).  Joint terms (PILCO_REWARD_*_SA) are evaluated at the
 *   point x~_t; within a step the state terms are accumulated first, in order, then the joint terms, in order.
 * H+1 step launches and H pilco_gp_predict calls on `stream`; every argument, the predict step's included, is
 * validated before anything is enqueued.  A particle's outputs do not depend on P or on its row.
 * PILCO_ERR_UNSUPPORTED: dyn not an unbatched mode-0 model with iK, a batched policy, an RBF policy not in mode 1,
 * unknown kinds or channels. */
typedef struct pilco_particles {
    int P, H;
    pilco_gp_model dyn;             /* mode 0 with iK, unbatched; D = Ds+U, E = Ds */
    pilco_policy   pol;             /* unbatched: every *_bs of the policy is 0 */
    int n_rewards; pilco_reward_term rewards[8]; double mult_mu;
    const double* x0;               /* [P,Ds]   initial particles (the caller samples them) */
    const double* eps;              /* [P,H,Ds] standard normals (the caller draws them) */
    double* traj;                   /* [P,H+1,Ds] */
    double* act;                    /* [P,H,U]  squashed actions */
    double* step_reward;            /* [P,H]    additive channel */
    double* step_risk;              /* [P,H]    MULT channel (zeros without MULT terms) */
    double* ret;                    /* [P] */
    void* ws; size_t ws_bytes;
} pilco_particles;
size_t pilco_particles_workspace_bytes(const pilco_particles* pr);   /* 0: unsupported sizes */
int    pilco_particles_rollout(const pilco_particles* pr, pilco_stream_t stream);

/* Pathwise (reparameterisation) gradient of the particle return: runs the particle rollout of `pr` (its outputs are
 * bitwise those of pilco_particles_rollout; pr->ws is not used, g->ws holds every buffer) and then a reverse sweep
 * with x0 and eps held fixed.  value[0] = (1/P) sum_p ret_p and the gradient of value w.r.t. the policy parameters:
 * linear gW [U,Ds], gb [U]; RBF gXc [bf,Ds] centres, gYc [bf,U] targets, gell [U,Ds] lengthscales (constrained),
 * through beta = (K + sn2 I)^-1 Yc with pol_L = the Cholesky factors pilco_gp_factorize leaves (as
 * pilco_rollout_grad).  A joint term adds a_kt d v_k / d u_t to the action cotangent and a_kt d v_k / d x_t to the
 * state cotangent of step t, a_kt the weight the step's state terms carry (step H-1 included).  Box terms are flat almost everywhere: they enter value but not the gradient, so for them the
 * estimator is biased as an estimate of d E[return].  Where a predicted variance is close to 0 the derivative of its
 * square root is large (exact, not clamped); where it is <= 0 it is taken as 0.  Every argument, the forward's
 * included, is validated before anything is enqueued; no host synchronisation (graph-capturable). */
typedef struct pilco_particles_grad {
    double* gW; double* gb;                             /* linear policy */
    double* gXc; double* gYc; double* gell;             /* RBF policy */
    const double* pol_L;
    double* value;                                      /* [1] */
    void* ws; size_t ws_bytes;
} pilco_particles_grad;
size_t pilco_particles_grad_workspace_bytes(const pilco_particles* pr);  /* 0: unsupported sizes */
int    pilco_particles_rollout_grad(const pilco_particles* pr, const pilco_particles_grad* g, pilco_stream_t stream);

/* The particle gradient of R policies at once (policy optimisation on the sampled return, random restarts in one call):
 * restart r runs the policy at r times the policy's batch strides (W_bs, b_bs, rbf.X_bs / ell_bs / sf2_bs / beta_bs;
 * a stride of 0 shares that array) over the SAME x0 [P,Ds] and eps [P,H,Ds] (common random numbers: the restarts are
 * compared on one sample), through the one unbatched dynamics model.  Outputs are restart-major: traj [R,P,H+1,Ds],
 * act [R,P,H,U], step_reward / step_risk [R,P,H], ret [R,P], value [R], gW [R,U,Ds], gb [R,U], gXc [R,bf,Ds],
 * gYc [R,bf,U], gell [R,U,Ds]; pol_L = the [R,U,ldw,ldw] Cholesky factors a batched pilco_gp_factorize leaves.
 * Restart r's outputs are bitwise those of pilco_particles_rollout_grad with policy r.  One predict / VJP call per
 * step at T = R P.  Validation as pilco_particles_rollout_grad, plus PILCO_ERR_DIM for R < 1, R > 65535,
 * R P > 65535 * 32 (the predict limit) or a negative stride; no host synchronisation (graph-capturable). */
size_t pilco_particles_batch_grad_workspace_bytes(const pilco_particles* pr, int R);   /* 0: unsupported sizes */
int    pilco_particles_rollout_batch_grad(const pilco_particles* pr, int R,
                                          const pilco_particles_grad* g, pilco_stream_t stream);

/* The particle rollout with ONE function drawn per particle from the latent posterior of each dynamics output, instead
 * of fresh noise at every step: f_t = mu(x~_t) + sum_{s<t} l_s eps_s + sqrt(max(d2, 0)) eps_t, where l and d2 come
 * from conditioning on the particle's own earlier inputs (k_post(a,b) = k(a,b) - k(a,C) iK k(C,b); forward
 * substitution in the particle's running Cholesky factor; a pivot d2 <= 1e-10 sf2_e leaves its column out of later
 * substitutions, so a revisited input reproduces its value).  Same description, outputs, validation and status codes
 * as pilco_particles_rollout, with pr->ws sized by pilco_particles_consistent_workspace_bytes: O(P H E n) (the K*
 * history) + O(P H^2 E).  Step 0 is bitwise pilco_particles_rollout's.  A particle's outputs do not depend on P or
 * on its row; no host synchronisation (graph-capturable). */
size_t pilco_particles_consistent_workspace_bytes(const pilco_particles* pr);   /* 0: unsupported sizes or overflow */
int    pilco_particles_rollout_consistent(const pilco_particles* pr, pilco_stream_t stream);

/* The consistent rollout of R policies and the pathwise gradient of each one's mean return (DESIGN.md section 15):
 * pilco_particles_rollout_batch_grad's contract (shared x0 and eps, the policy's batch strides honoured, 0 sharing an
 * array, restart-major outputs, the gradient in pilco_particles_grad) with the particles of
 * pilco_particles_rollout_consistent.  Its forward outputs are bitwise those of pilco_particles_rollout_consistent with
 * the same policy; R = 1 with an unbatched policy is the single-policy call.  Validation and status codes are those of
 * pilco_particles_rollout_batch_grad and pilco_particles_rollout_consistent; g->ws is sized by
 * pilco_particles_consistent_grad_workspace_bytes: the consistent forward's at R P particles + O(R P H^2 E).  Every
 * sum has a fixed order, so a restart's results are bitwise independent of R and reproducible run to run; a pivot the
 * forward declares degenerate holds its step's own noise constant.  No host synchronisation (graph-capturable). */
size_t pilco_particles_consistent_grad_workspace_bytes(const pilco_particles* pr, int R);  /* 0: unsupported / overflow */
int    pilco_particles_rollout_consistent_grad(const pilco_particles* pr, int R, const pilco_particles_grad* g,
                                               pilco_stream_t stream);

/* Score-function (likelihood-ratio) gradient of the particle return (DESIGN.md section 16): the contract of
 * pilco_particles_rollout_batch_grad (R policies through the batch strides, 0 sharing an array, shared x0 and eps,
 * restart-major outputs, R = 1 with an unbatched policy the single-policy call, the same validation and status codes,
 * all checked before anything is enqueued), with g->ws sized by pilco_particles_score_grad_workspace_bytes.  The
 * forward outputs and value are bitwise those of pilco_particles_rollout_batch_grad; the gradient, in the same layout,
 * is that of (1/P) sum_p sum_{t<H-1} w_pt log N(x_{t+1} - x_t; mu(x~_t), var(x~_t)) with x_t, x_{t+1} held fixed:
 *   d/d mu = eps / s,  d/d var = (eps^2 - 1) / (2 var)   (both 0 where var <= 0; not clamped near 0),
 *   w_pt = G_pt - (S_t - G_pt) / (P - 1), G_pt the part of particle p's return that transition t can affect
 *   (the step rewards after t, and mult_mu prod_{s<=t} (1 - risk_s) (1 - prod_{s>t} (1 - risk_s))), S_t = sum_q G_qt
 *   over the restart's particles (a leave-one-out baseline; P = 1: w = G).
 * With the states held fixed a joint term (PILCO_REWARD_*_SA) still depends on the parameters directly, through
 * u_t = pi(x_t), so the estimator adds (1/P) sum_p sum_{t<H} a_kt d v_k / d u_t d pi(x_pt) / d theta (a_kt = coef_k, or
 * coef_k mult_mu prod_{s != t} (1 - risk_s) in the MULT channel; t = H-1 included): without it the gradient would be
 * biased as soon as a joint term is present.  G_pt needs no change: the step rewards contain the joint terms.
 * Its expectation is d E[return] for every reward kind, box terms included; it differentiates no trajectory, and its
 * variance grows as 1/var where the model is confident.  H <= 1 gives a zero gradient (H = 1 with joint terms: the
 * direct term alone).  A restart's results are
 * bitwise independent of R and reproducible run to run; no host synchronisation (graph-capturable). */
size_t pilco_particles_score_grad_workspace_bytes(const pilco_particles* pr, int R);   /* 0: unsupported / overflow */
int    pilco_particles_rollout_score_grad(const pilco_particles* pr, int R, const pilco_particles_grad* g,
                                          pilco_stream_t stream);

/* ---- diagnostics ------------------------------------------------------------------------------
 * fp64 pipe microbenchmark used for the roofline denominators (DESIGN.md "Roofline"): which = 0 DFMA,
 * 1 DMMA m8n8k4, 2 both interleaved, 3 table exp, 4 libdevice exp, 5 DMMA m16n8k8, 6 DMMA m16n8k16;
 * 8 ops/thread/iteration (16 DMMA for which=1,2 counted as 8 pairs; 8 MMAs per warp for which=5,6).  Synchronises (it times itself with CUDA events) -- never call it in a
 * captured region. */
/* pilco_mm_forward with CUDA events around its three launches: ms_out[0..2] = setup, tile, finish.
 * Synchronises. */
int pilco_mm_forward_profile(const pilco_gp_model* gp, int R, const double* m, const double* s,
                             double* M, double* S, double* V, int* info,
                             void* ws, size_t ws_bytes, float* ms_out, pilco_stream_t stream);
int pilco_mm_forward_taped_profile(const pilco_gp_model* gp, int R, const double* m, const double* s,
                                   double* M, double* S, double* V, int* info,
                                   void* ws, size_t ws_bytes, void* tape, size_t tape_bytes,
                                   float* ms_out, pilco_stream_t stream);
int pilco_microbench_fp64(int which, int iters, int blocks, double* sink_dev, float* ms_out, pilco_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* PILCO_B200_H */
