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
 * pilco_rollout_backward needs for the RBF policy (pilco_rollout_grad.pol_L), and when iK is requested the next
 * B*E*ldw*ldw doubles hold R = L^-1 (zero above the diagonal and in the padding), which pilco_gp_append_tri extends.
 * n <= 28000 (the substitution for beta keeps a right-hand side in shared memory); info[b] bit 1: a pivot of
 * batch element b was not positive (its outputs are then meaningless, the other elements' are unaffected).
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
 * rows of each new episode).  X [n0+k, D] and Y [n0+k, E] hold the old rows first.  R_old [E,ldr_old,ldr_old] is the
 * lower-triangular inverse Cholesky factor L^-1 of the old model (zero above the diagonal and in the padding):
 * pilco_gp_factorize leaves it in its workspace right after the factors L (second B*E*ldw*ldw doubles), an earlier
 * append in its R_new.  iK_old [E,ldk_old,ldk_old] is the old inverse.  Writes R_new [E,ldr_new,ldr_new] (zero
 * padded), the new zero-padded inverse iK_new [E,ldk_new,ldk_new] (both leading dimensions >= pilco_pad_n(n0+k), out
 * of place) and beta_new [E,n0+k] by extending R with one block row: O(n^2 k) instead of O(n^3), as accurate as a
 * refactorisation after any number of appends.  info[0] bit 1: the new rows' Schur complement is not positive
 * definite. */
size_t pilco_gp_append_tri_workspace_bytes(int n0, int k, int E);
int pilco_gp_append_tri(int n0, int k, int D, int E,
                    const double* X, const double* Y,
                    const double* ell, const double* sf2, const double* sn2,
                    const double* R_old, int ldr_old, const double* iK_old, int ldk_old,
                    double* R_new, int ldr_new, double* iK_new, int ldk_new, double* beta_new, int* info,
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
 * e0 .. e0+ne-1 of an unbatched mode-0 model with iK (pilco_gp_factorize, pilco_gp_append_tri or pilco_fitc_factorize) at
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
#define PILCO_POLICY_MLP    2   /* tanh MLP, particle rollouts only: pilco_particles_mlp_* with a pilco_mlp */
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

/* ---- angular state dimensions -----------------------------------------------------------------
 * PILCO's trigonometric augmentation (gTrig in propagate.m): the angular state dimensions dims[0 .. A-1] of x [Ds]
 * reach the policy and the dynamics GP through the feature map
 *   phi(x) = [x_j for j not an angle, increasing j] ++ [sin x_a, cos x_a for a = dims[0], ..., dims[A-1]]   (Dh = Ds + A)
 * whose Gaussian moments are exact.  The state itself stays raw: m0, S0, traj_m, traj_S, gm0, gS0, the state reward
 * terms and the dynamics GP's outputs (deltas of x, angles unwrapped) are in Ds.  With angles, a pilco_rollout has
 * pol.Ds = Dh, dyn.D = Dh + U and dyn.E = Ds, and its joint state-action terms (PILCO_REWARD_*_SA) are evaluated at
 * the Gaussian the dynamics receive, [phi(x), u] (D = Dh + U).  Every call below with ang == NULL or ang->A == 0 is
 * the corresponding call without angles.  Validation before any work is enqueued: PILCO_ERR_DIM for a dimension out of
 * range or repeated, A > Ds or Dh + U > PILCO_MAX_D, otherwise the status codes of the call without angles. */
typedef struct pilco_angles {
    int A;                      /* number of angular dimensions, 0 .. Ds */
    int dims[PILCO_MAX_D];      /* their state indices, distinct */
} pilco_angles;

/* moments of phi(x) for x ~ N(m, s): M [R,Dh], S [R,Dh,Dh] and C = inv(s) cov(x, phi(x)) [R,Ds,Dh] (no inverse is
 * formed: s = 0 and singular s are valid).  With no angles: M = m, S = s, C = I. */
int pilco_trig_moments(int Ds, int R, const pilco_angles* ang, const double* m /*[R,Ds]*/, const double* s /*[R,Ds,Ds]*/,
                       double* M, double* S, double* C, pilco_stream_t stream);

size_t pilco_rollout_angles_workspace_bytes(const pilco_rollout* ro, const pilco_angles* ang);
size_t pilco_rollout_angles_tape_bytes(const pilco_rollout* ro, const pilco_angles* ang);
size_t pilco_rollout_angles_bwd_workspace_bytes(const pilco_rollout* ro, const pilco_angles* ang);
int    pilco_rollout_angles_forward(const pilco_rollout* ro, const pilco_angles* ang, pilco_stream_t stream);
/* policy gradients in the policy's (Dh) layout; gm0 [R,Ds] and gS0 [R,Ds,Ds] with respect to the raw initial moments,
 * gS0 symmetric when angles are present (the gradient with respect to a symmetric S0) */
int    pilco_rollout_angles_backward(const pilco_rollout* ro, const pilco_angles* ang, const pilco_rollout_grad* g,
                                     pilco_stream_t stream);

/* ---- exploration objective (the original PILCO's exploration parameter b; DESIGN.md section 21) -----------------
 * The rollout of pilco_rollout_angles_* (ang may be NULL) with, per step t = 0 .. H-1 of restart r,
 *   sigma_t^2 = sum_k c_k^2 Var[r_k]  over the ADD-channel terms (CombinedRewards.compute_reward's rule, covariances
 *               between terms ignored): state terms at (m_t, S_t), joint terms (PILCO_REWARD_*_SA) at step t's joint
 *               Gaussian; exponential: r_2 - r_1^2 (reward.m:52-56), linear: W^T S W.  MULT-channel terms do not enter.
 *   sigma_t   = sqrt(sigma_t^2) if sigma_t^2 > 1e-12, else 0 (with zero gradient)
 * and reward[r] = sum_t (E[r_t] + b sigma_t), summed in step order, plus the MULT channel's term.  b > 0 is optimistic
 * under model uncertainty (exploration), b < 0 risk-averse.  step_reward stays E[r_t].  The call is inactive when
 * ex == NULL or b == 0 with step_var == NULL: it is then the pilco_rollout_angles_* call, workspace sizes included; with
 * b == 0 every output and gradient is bitwise that call's.  The tape is pilco_rollout_angles_tape_bytes'.  Validation
 * before any work is enqueued: the status codes of the call without exploration, PILCO_ERR_DIM for a non-finite b,
 * PILCO_ERR_UNSUPPORTED for an ADD-channel PILCO_REWARD_BOX term (no variance closed form), PILCO_ERR_WORKSPACE when
 * ro->ws_bytes is below pilco_rollout_explore_workspace_bytes. */
typedef struct pilco_exploration {
    double  b;                  /* weight of sigma_t in the objective; finite */
    double* step_var;           /* [R,H] sigma_t^2, or NULL */
} pilco_exploration;

size_t pilco_rollout_explore_workspace_bytes(const pilco_rollout* ro, const pilco_angles* ang, const pilco_exploration* ex);
size_t pilco_rollout_explore_bwd_workspace_bytes(const pilco_rollout* ro, const pilco_angles* ang,
                                                 const pilco_exploration* ex);
int    pilco_rollout_explore_forward(const pilco_rollout* ro, const pilco_angles* ang, const pilco_exploration* ex,
                                     pilco_stream_t stream);
/* gradient of reward[r] (with the bonus) as pilco_rollout_angles_backward gives it.  Must follow
 * pilco_rollout_explore_forward with the same `ro`, `ang` and `ex` (it reads the sigma_t^2 that call saved in ro->ws). */
int    pilco_rollout_explore_backward(const pilco_rollout* ro, const pilco_angles* ang, const pilco_exploration* ex,
                                      const pilco_rollout_grad* g, pilco_stream_t stream);

/* ---- measurement noise at the policy's input (propagate.m's noisy state measurement; DESIGN.md section 22) --------
 * The rollout of pilco_rollout_explore_* (ang and ex may be NULL) whose policy sees a noisy measurement z = x + nu,
 * nu ~ N(0, diag(var[0 .. Ds-1])) independent of x (Ds = dyn.E, the raw state).  Per step t of restart r:
 *   the policy is moment-matched at the moments of phi(z) under N(m_t, S_t + diag(var)) (phi = identity without angles);
 *   the dynamics GP receives [phi(x), u] with phi's moments under N(m_t, S_t) and cov(phi(x), u) = S^_x V_u, V_u the
 *   policy's (squashed) input-output factor at the noisy input (propagate.m's q = S(j,i) C: the true S, the noisy C);
 *   the next-state glue uses cov(x, [phi(x), u]) = S_t C^_x [I, V_u];
 *   the reward terms are unchanged (state terms at (m_t, S_t), joint terms and sigma_t^2 at the joint above).
 * With nz == NULL every call is the pilco_rollout_explore_* call, workspace sizes included.  The tape is
 * pilco_rollout_tape_bytes'.  Validation before any work is enqueued: the status codes of the explore call's
 * description and exploration checks, then PILCO_ERR_DIM for a non-finite or negative var[i], i < Ds, then
 * PILCO_ERR_WORKSPACE when ro->ws_bytes is below pilco_rollout_noisy_workspace_bytes (g->ws_bytes below
 * pilco_rollout_noisy_bwd_workspace_bytes for the backward).  The backward gives no gradient with respect to var. */
typedef struct pilco_obs_noise {
    double var[PILCO_MAX_D];    /* measurement noise variance of each raw state dimension, >= 0; the first Ds are used */
} pilco_obs_noise;

size_t pilco_rollout_noisy_workspace_bytes(const pilco_rollout* ro, const pilco_angles* ang, const pilco_exploration* ex,
                                           const pilco_obs_noise* nz);
size_t pilco_rollout_noisy_bwd_workspace_bytes(const pilco_rollout* ro, const pilco_angles* ang,
                                               const pilco_exploration* ex, const pilco_obs_noise* nz);
int    pilco_rollout_noisy_forward(const pilco_rollout* ro, const pilco_angles* ang, const pilco_exploration* ex,
                                   const pilco_obs_noise* nz, pilco_stream_t stream);
/* must follow pilco_rollout_noisy_forward with the same arguments (it reads the per-step moments saved in ro->ws) */
int    pilco_rollout_noisy_backward(const pilco_rollout* ro, const pilco_angles* ang, const pilco_exploration* ex,
                                    const pilco_obs_noise* nz, const pilco_rollout_grad* g, pilco_stream_t stream);

/* ---- time-varying linear policy (probabilistic MPC's action sequences; DESIGN.md section 27) ---------------------
 * The rollout of pilco_rollout_noisy_* (ang, ex and nz may be NULL) whose linear policy is indexed by the step: restart r
 * at step t = 0 .. H-1 applies u_t = W_t x~ + b_t (squashed when pol.squash, x~ the policy's input as in the noisy call)
 * with
 *   W_t = pol.W + r pol.W_bs + t W_ts   [U, Dh],     b_t = pol.b + r pol.b_bs + t b_ts   [U].
 * W_t = 0 at every step is an open-loop action sequence.  The schedule is active when sch != NULL and W_ts or b_ts is
 * non-zero; an inactive call is the pilco_rollout_noisy_* call: outputs, gradients, workspace sizes and status codes.
 * With an active schedule the backward writes the cotangents per step, g->gW [R, H, U, Dh] and g->gb [R, H, U] (their
 * sum over t is the stationary policy's gradient), and needs the larger reverse workspace
 * pilco_rollout_scheduled_bwd_workspace_bytes reports; the forward workspace and the tape are the noisy call's.
 * Validation before any work is enqueued: the noisy call's status codes up to its workspace check, then PILCO_ERR_DIM
 * for a negative stride, then PILCO_ERR_UNSUPPORTED for an active schedule with an RBF policy, then the workspace's
 * codes.  A size query returns 0 for R < 1, H < 0 or a negative stride. */
typedef struct pilco_policy_schedule {
    long long W_ts;             /* step stride of pol.W in doubles (U * Dh for a dense [H, U, Dh] block), >= 0 */
    long long b_ts;             /* step stride of pol.b in doubles (U for a dense [H, U] block), >= 0 */
} pilco_policy_schedule;

size_t pilco_rollout_scheduled_workspace_bytes(const pilco_rollout* ro, const pilco_angles* ang,
                                               const pilco_exploration* ex, const pilco_obs_noise* nz,
                                               const pilco_policy_schedule* sch);
int    pilco_rollout_scheduled_forward(const pilco_rollout* ro, const pilco_angles* ang, const pilco_exploration* ex,
                                       const pilco_obs_noise* nz, const pilco_policy_schedule* sch,
                                       pilco_stream_t stream);
size_t pilco_rollout_scheduled_bwd_workspace_bytes(const pilco_rollout* ro, const pilco_angles* ang,
                                                   const pilco_exploration* ex, const pilco_obs_noise* nz,
                                                   const pilco_policy_schedule* sch);
/* must follow pilco_rollout_scheduled_forward with the same arguments */
int    pilco_rollout_scheduled_backward(const pilco_rollout* ro, const pilco_angles* ang, const pilco_exploration* ex,
                                        const pilco_obs_noise* nz, const pilco_policy_schedule* sch,
                                        const pilco_rollout_grad* g, pilco_stream_t stream);

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

/* The particle rollouts with angular state dimensions (pilco_angles above; DESIGN.md section 20).  Each call below is
 * the call of the same name without "_angles" with the feature map phi at every particle:
 *   u_t = squash(pi(phi(x_t))),  x~_t = [phi(x_t), u_t],  x_{t+1} = x_t + mu(x~_t) + sqrt(max(var(x~_t), 0)) o eps_t
 * (the consistent sampler conditions on the particle's earlier x~, which hold phi).  With E = dyn.E the raw state
 * dimension and A = ang->A: pol.Ds = Dh = E + A and dyn.D = Dh + U.  x0 [P,E], eps [P,H,E], traj [..,H+1,E] and the
 * GP's outputs (deltas of x, angles unwrapped) stay raw; the state reward terms (EXP, LINEAR, BOX; W, t and the box's
 * indices in E) are evaluated at the raw x_t, the joint terms (*_SA, D = Dh + U) at x~_t, so a periodic target such as
 * "pendulum up" is an EXP_SA term on (sin, cos) = (0, -1).  Policy gradients are in the policy's Dh layout.  sin and
 * cos are evaluated once per particle and step, and the reverse sweep reuses those values.
 * The workspaces are those of the calls without angles at the same description, plus, for the three gradients, the
 * phi history [R P,H+1,Dh] (the forward-only ones do not grow with H).  Every call with ang == NULL or ang->A == 0 is
 * the call without angles.  Validation before anything is enqueued: PILCO_ERR_DIM for a repeated or out-of-range
 * dimension, A > E, pol.Ds != E + A, dyn.D != pol.Ds + U, dyn.D > PILCO_MAX_D or an RBF policy with rbf.D != Dh;
 * otherwise the status codes of the call without angles (a workspace query returns 0 where its call would fail on
 * these).  batch_grad at R = 1 with an unbatched policy is the single-policy pathwise gradient. */
size_t pilco_particles_angles_workspace_bytes(const pilco_particles* pr, const pilco_angles* ang);
int    pilco_particles_angles_rollout(const pilco_particles* pr, const pilco_angles* ang, pilco_stream_t stream);
size_t pilco_particles_angles_consistent_workspace_bytes(const pilco_particles* pr, const pilco_angles* ang);
int    pilco_particles_angles_consistent_rollout(const pilco_particles* pr, const pilco_angles* ang,
                                                 pilco_stream_t stream);
size_t pilco_particles_angles_batch_grad_workspace_bytes(const pilco_particles* pr, const pilco_angles* ang, int R);
int    pilco_particles_angles_batch_grad_rollout(const pilco_particles* pr, const pilco_angles* ang, int R,
                                                 const pilco_particles_grad* g, pilco_stream_t stream);
size_t pilco_particles_angles_consistent_grad_workspace_bytes(const pilco_particles* pr, const pilco_angles* ang, int R);
int    pilco_particles_angles_consistent_grad_rollout(const pilco_particles* pr, const pilco_angles* ang, int R,
                                                      const pilco_particles_grad* g, pilco_stream_t stream);
size_t pilco_particles_angles_score_grad_workspace_bytes(const pilco_particles* pr, const pilco_angles* ang, int R);
int    pilco_particles_angles_score_grad_rollout(const pilco_particles* pr, const pilco_angles* ang, int R,
                                                 const pilco_particles_grad* g, pilco_stream_t stream);

/* The particle rollouts with measurement noise at the policy's input (propagate.m's noisy state measurement at every
 * particle; DESIGN.md section 23).  Each call below is the pilco_particles_angles_* call of the same name (ang may be
 * NULL) whose policy sees a noisy measurement of the state.  Per particle p, restart r and step t < H, with E = dyn.E:
 *   z_t = x_t + sqrt(v) o nu_t,  u_t = squash(pi(phi(z_t))),  x~_t = [phi(x_t), u_t],
 *   x_{t+1} = x_t + mu(x~_t) + sqrt(max(var(x~_t), 0)) o eps_t
 * (phi = identity without angles; the consistent sampler conditions on the particle's earlier x~, which hold phi(x)).
 * The state terms are evaluated at the raw x_t and the joint terms at x~_t, as before.  traj, act, step_reward,
 * step_risk, ret and value keep their layouts.  nu is an exogenous input like x0 and eps: each gradient is conditioned on
 * it and estimates the derivative of the return's expectation over (x0, eps, nu); none is taken with respect to v.
 * The forward-only workspaces are those of the angle calls; the three gradients' are those of the angle calls with
 * angles (the phi history [R P,H+1,Dh], with A = 0 too), then the phi(z) history [R P,H+1,Dh] and, for the pathwise and
 * consistent gradients, phi_bar_z [R P,Dh] (each slot rounded up to an even number of doubles).
 * With nz == NULL every call is the pilco_particles_angles_* call with the same arguments, workspace sizes included.
 * Validation before anything is enqueued: the angle call's status codes up to its workspace check, then PILCO_ERR_DIM
 * for a non-finite or negative v.var[i] (i < E), then PILCO_ERR_NULL for nu == NULL with H > 0, then the workspace's
 * codes (PILCO_ERR_WORKSPACE).  A workspace query returns 0 wherever its call would fail on these checks. */
typedef struct pilco_particles_noise {
    pilco_obs_noise v;          /* measurement variances of the raw state; the first dyn.E are used, finite, >= 0 */
    const double*   nu;         /* [P,H,E] standard normals of the measurement noise, shared by the R restarts */
} pilco_particles_noise;

size_t pilco_particles_noisy_workspace_bytes(const pilco_particles* pr, const pilco_angles* ang,
                                             const pilco_particles_noise* nz);
int    pilco_particles_noisy_rollout(const pilco_particles* pr, const pilco_angles* ang, const pilco_particles_noise* nz,
                                     pilco_stream_t stream);
size_t pilco_particles_noisy_consistent_workspace_bytes(const pilco_particles* pr, const pilco_angles* ang,
                                                        const pilco_particles_noise* nz);
int    pilco_particles_noisy_consistent_rollout(const pilco_particles* pr, const pilco_angles* ang,
                                                const pilco_particles_noise* nz, pilco_stream_t stream);
size_t pilco_particles_noisy_batch_grad_workspace_bytes(const pilco_particles* pr, const pilco_angles* ang,
                                                        const pilco_particles_noise* nz, int R);
int    pilco_particles_noisy_batch_grad_rollout(const pilco_particles* pr, const pilco_angles* ang,
                                                const pilco_particles_noise* nz, int R, const pilco_particles_grad* g,
                                                pilco_stream_t stream);
size_t pilco_particles_noisy_consistent_grad_workspace_bytes(const pilco_particles* pr, const pilco_angles* ang,
                                                             const pilco_particles_noise* nz, int R);
int    pilco_particles_noisy_consistent_grad_rollout(const pilco_particles* pr, const pilco_angles* ang,
                                                     const pilco_particles_noise* nz, int R,
                                                     const pilco_particles_grad* g, pilco_stream_t stream);
size_t pilco_particles_noisy_score_grad_workspace_bytes(const pilco_particles* pr, const pilco_angles* ang,
                                                        const pilco_particles_noise* nz, int R);
int    pilco_particles_noisy_score_grad_rollout(const pilco_particles* pr, const pilco_angles* ang,
                                                const pilco_particles_noise* nz, int R, const pilco_particles_grad* g,
                                                pilco_stream_t stream);

/* PILCO's exploration objective in the particle rollouts (pilco_exploration above; DESIGN.md section 24).  Each call is
 * the pilco_particles_noisy_* gradient of the same name (ang and nz may be NULL) whose value adds the sample spread of
 * each step's reward.  Per restart r, over its P particles, for each ADD-channel term k with coefficient c_k at step
 * t < H (state terms at the raw x_pt, joint terms at x~_pt = [phi(x_pt), u_pt]):
 *   rbar_kt = (1/P) sum_p r_kpt,  s_kt^2 = 1/(P-1) sum_p (r_kpt - rbar_kt)^2   (unbiased, two-pass, fixed order)
 *   sigma_t^2 = sum_k c_k^2 s_kt^2   (section 21's rule: covariances between terms ignored; MULT terms do not enter)
 *   sigma_t   = sqrt(sigma_t^2) if sigma_t^2 > 1e-12, else 0 (with zero gradient)
 *   value[r]  = (1/P) sum_p ret_p + b sum_t sigma_t   (the bonus summed in step order)
 * ex->step_var [R,H] receives sigma_t^2 when not NULL.  The gradient is pathwise: the bonus adds
 * a_kpt grad r_kpt, a_kpt = P b c_k^2 (r_kpt - rbar_kt) / ((P-1) sigma_t), to each particle's cotangent at each step.
 * traj, act, step_reward, step_risk and ret keep their meaning and bits.  sigma_t is the square root of an unbiased
 * variance, so it is biased low by O(1/P).  The call is inactive when ex == NULL or b == 0 with step_var == NULL: it is
 * then the pilco_particles_noisy_* call, workspace sizes included; with b == 0 every output and gradient is bitwise that
 * call's.  Validation before anything is enqueued: the noisy call's status codes up to its workspace check, then
 * PILCO_ERR_DIM for a non-finite b, PILCO_ERR_UNSUPPORTED for an ADD-channel PILCO_REWARD_BOX term, PILCO_ERR_DIM for
 * P < 2, then the workspace's codes.  The workspace is the noisy call's (with the angle layout when ang or nz is given)
 * followed by sigma_t [R,H] and a table [R,H,n_rewards,2] (each slot rounded up to an even number of doubles); a
 * workspace query returns 0 wherever its call would fail on the size or exploration checks. */
size_t pilco_particles_explore_batch_grad_workspace_bytes(const pilco_particles* pr, const pilco_angles* ang,
                                                          const pilco_particles_noise* nz, const pilco_exploration* ex,
                                                          int R);
int    pilco_particles_explore_batch_grad_rollout(const pilco_particles* pr, const pilco_angles* ang,
                                                  const pilco_particles_noise* nz, const pilco_exploration* ex, int R,
                                                  const pilco_particles_grad* g, pilco_stream_t stream);
size_t pilco_particles_explore_consistent_grad_workspace_bytes(const pilco_particles* pr, const pilco_angles* ang,
                                                               const pilco_particles_noise* nz,
                                                               const pilco_exploration* ex, int R);
int    pilco_particles_explore_consistent_grad_rollout(const pilco_particles* pr, const pilco_angles* ang,
                                                       const pilco_particles_noise* nz, const pilco_exploration* ex,
                                                       int R, const pilco_particles_grad* g, pilco_stream_t stream);

/* Score-function (likelihood-ratio) gradient over consistent function samples (DESIGN.md section 25): the contract of
 * pilco_particles_noisy_consistent_grad_rollout (ang and nz may be NULL; R policies through the batch strides, shared
 * x0, eps and nu, restart-major outputs, R = 1 with an unbatched policy the single-policy call; the same validation and
 * status codes in the same order, all checked before anything is enqueued), with g->ws sized by
 * pilco_particles_consistent_score_grad_workspace_bytes.  The forward outputs and value are bitwise those of the
 * consistent pathwise call; the gradient, in the same layout, is that of
 *   (1/P) sum_p sum_{t<H-1, piv_t>0} w_pt (-eps_t(theta)^2 / 2 - log piv_t(theta)),
 *   eps_t(theta) = (f_t - mean'_t(theta)) / piv_t(theta),  mean'_t = mu(x~_t) + sum_{s<t} l_ts eps_s(theta)
 * per output, with the increments f_t = x_{t+1} - x_t and the states x_t held fixed (theta enters through u_s = pi(x_s)
 * inside every x~_s, s <= t): the log-density of the particle's whole path under its function draw.  w_pt is section
 * 16's (return-to-go with the leave-one-out baseline, P = 1: w = G), and the joint terms' direct term is added as there.
 * Its expectation is d E[return] for every reward kind, box terms included, on rollouts whose pivots are all above the
 * forward's threshold: a step whose pivot is degenerate (d2 <= 1e-10 sf2) is deterministic given the particle's past, has
 * no likelihood ratio and is dropped, so the estimate is biased where such steps occur.  Near the threshold nothing is
 * clamped: 1/piv is large there and so is the variance.  H <= 1 gives a zero gradient (H = 1 with joint terms: the
 * direct term alone).  The workspace is the consistent gradient's layout (with the angle layout when ang or nz is
 * given, the noise slots when nz is) followed by G [H-1,R P], the sums [R,H], m_bar and v_bar [H-1,R P,E] and the x~_bar
 * history [H,R P,D] (each slot rounded up to an even number of doubles); the query returns 0 wherever the call would
 * fail on its sizes, and on size_t overflow.  A restart's results are bitwise independent of R and reproducible run to
 * run; no host synchronisation (graph-capturable). */
size_t pilco_particles_consistent_score_grad_workspace_bytes(const pilco_particles* pr, const pilco_angles* ang,
                                                             const pilco_particles_noise* nz, int R);
int    pilco_particles_consistent_score_grad_rollout(const pilco_particles* pr, const pilco_angles* ang,
                                                     const pilco_particles_noise* nz, int R,
                                                     const pilco_particles_grad* g, pilco_stream_t stream);

/* The per-step sample moments above over a forward that has already run: traj [R P,H+1,E] and act [R P,H,U] of R
 * restarts of P particles (any sampler, chunked or not).  step_mean [R,H] = sum_k c_k rbar_kt and step_var [R,H] =
 * sigma_t^2, each skipped when NULL.  Reads P, H, dyn.E, pol.Ds (= E + A), pol.U, the reward terms, traj and act of pr
 * and nothing else.  PILCO_ERR_DIM for P < 2, H < 0, R outside [1, 65535], a bad angle map or widths
 * (pol.Ds != E + A, E + A + U > PILCO_MAX_D), n_rewards outside [1, 8]; PILCO_ERR_NULL / PILCO_ERR_UNSUPPORTED for
 * the reward terms as the rollouts check them and PILCO_ERR_UNSUPPORTED for an ADD-channel box term; PILCO_ERR_NULL
 * for traj or act NULL with H > 0.  One launch (none at H = 0), no workspace. */
int    pilco_particles_reward_moments(const pilco_particles* pr, const pilco_angles* ang, int R, double* step_mean,
                                      double* step_var, pilco_stream_t stream);

/* Gaussian-resampled particle rollouts (Deep PILCO's refit; DESIGN.md section 26), step-wise sampler.  At every step
 * t >= 1 each restart's particles are refitted to a Gaussian and redrawn from it (no refit at t = 0):
 *   x'_pt = x_{p,t-1} + mu(x~_{p,t-1}) + sqrt(max(var, 0)) o eps_{p,t-1}     (pilco_particles_rollout's step)
 *   mu^_t = (1/P) sum_p x'_pt,  S^_t = 1/(P-1) sum_p (x'_pt - mu^_t)(x'_pt - mu^_t)'   (over the restart's particles)
 *   L^_t  = chol(S^_t) column by column; a column j whose pivot d_j <= 1e-12 S^_t,jj (or S^_t,jj <= 0) is zeroed
 *   x_pt  = mu^_t + L^_t xi_{p,t-1}
 * traj[:, t] holds x_t, at which the rewards, the policy and x~_t are evaluated as pilco_particles_rollout evaluates
 * them.  xi [P,H,Ds] are standard normals shared by the restarts.  step_mean [R,H+1,Ds] and step_cov [R,H+1,Ds,Ds]
 * receive mu^_t and S^_t (t = 0: the moments of x0), each skipped when NULL.  A restart's results do not depend on R.
 * pilco_particles_resampled_rollout: pilco_particles_rollout's description, outputs and contract (unbatched policy,
 * pr->ws).  pilco_particles_resampled_grad_rollout: pilco_particles_rollout_batch_grad's contract (R policies, shared
 * x0, eps and xi, g->ws) with the pathwise gradient of value = mean return through the refit, x0, eps and xi held
 * fixed (away from degenerate pivots a smooth function of the policy parameters).  At H <= 1 value and gradient are
 * bitwise the call without resampling.  Validation is the call without resampling's, then PILCO_ERR_NULL for rs NULL
 * or xi NULL with H > 0, then PILCO_ERR_DIM for P < 2, then the workspace; a size query returns 0 exactly where its
 * call fails on sizes.  The workspace is the call without resampling's followed by O(H R P Ds + H R Ds^2). */
typedef struct pilco_particles_resample {
    const double* xi;           /* [P,H,Ds] standard normals of the redraw */
    double* step_mean;          /* [R,H+1,Ds] or NULL */
    double* step_cov;           /* [R,H+1,Ds,Ds] or NULL */
} pilco_particles_resample;
size_t pilco_particles_resampled_workspace_bytes(const pilco_particles* pr, const pilco_particles_resample* rs);
int    pilco_particles_resampled_rollout(const pilco_particles* pr, const pilco_particles_resample* rs,
                                         pilco_stream_t stream);
size_t pilco_particles_resampled_grad_workspace_bytes(const pilco_particles* pr, const pilco_particles_resample* rs,
                                                      int R);
int    pilco_particles_resampled_grad_rollout(const pilco_particles* pr, const pilco_particles_resample* rs, int R,
                                              const pilco_particles_grad* g, pilco_stream_t stream);

/* Time-varying linear policies in the particle rollouts (DESIGN.md section 28): each call is the most general call of
 * its family (pilco_particles_noisy_*, _explore_*, _consistent_score_grad_*, _resampled_*) with a pilco_policy_schedule
 * (section 27's) added.  Restart r at step t = 0 .. H-1 applies u_t = W_t z + b_t (squashed when pol.squash, z the
 * policy's input as in the call without a schedule) with
 *   W_t = pol.W + r pol.W_bs + t W_ts   [U, Dh],     b_t = pol.b + r pol.b_bs + t b_ts   [U].
 * W_t = 0 at every step is an open-loop action sequence.  The schedule is active when sch != NULL and W_ts or b_ts is
 * non-zero; an inactive call is the call without it: outputs, gradients, workspace sizes and status codes.  With an
 * active schedule the gradients are per step, g->gW [R, H, U, Dh] and g->gb [R, H, U] (their sum over t is the
 * stationary policy's gradient); value and the workspace are the call's without a schedule.  Validation before any
 * work is enqueued: the call's status codes up to its workspace check, then PILCO_ERR_DIM for a negative stride, then
 * PILCO_ERR_UNSUPPORTED for an active schedule with an RBF policy, then the workspace's codes.  A size query returns 0
 * where the call's without a schedule does, and for a negative stride. */
size_t pilco_particles_scheduled_workspace_bytes(const pilco_particles* pr, const pilco_angles* ang,
                                                 const pilco_particles_noise* nz, const pilco_policy_schedule* sch);
int    pilco_particles_scheduled_rollout(const pilco_particles* pr, const pilco_angles* ang,
                                         const pilco_particles_noise* nz, const pilco_policy_schedule* sch,
                                         pilco_stream_t stream);
size_t pilco_particles_scheduled_consistent_workspace_bytes(const pilco_particles* pr, const pilco_angles* ang,
                                                            const pilco_particles_noise* nz,
                                                            const pilco_policy_schedule* sch);
int    pilco_particles_scheduled_consistent_rollout(const pilco_particles* pr, const pilco_angles* ang,
                                                    const pilco_particles_noise* nz, const pilco_policy_schedule* sch,
                                                    pilco_stream_t stream);
size_t pilco_particles_scheduled_batch_grad_workspace_bytes(const pilco_particles* pr, const pilco_angles* ang,
                                                            const pilco_particles_noise* nz,
                                                            const pilco_exploration* ex,
                                                            const pilco_policy_schedule* sch, int R);
int    pilco_particles_scheduled_batch_grad_rollout(const pilco_particles* pr, const pilco_angles* ang,
                                                    const pilco_particles_noise* nz, const pilco_exploration* ex,
                                                    const pilco_policy_schedule* sch, int R,
                                                    const pilco_particles_grad* g, pilco_stream_t stream);
size_t pilco_particles_scheduled_consistent_grad_workspace_bytes(const pilco_particles* pr, const pilco_angles* ang,
                                                                 const pilco_particles_noise* nz,
                                                                 const pilco_exploration* ex,
                                                                 const pilco_policy_schedule* sch, int R);
int    pilco_particles_scheduled_consistent_grad_rollout(const pilco_particles* pr, const pilco_angles* ang,
                                                         const pilco_particles_noise* nz, const pilco_exploration* ex,
                                                         const pilco_policy_schedule* sch, int R,
                                                         const pilco_particles_grad* g, pilco_stream_t stream);
size_t pilco_particles_scheduled_score_grad_workspace_bytes(const pilco_particles* pr, const pilco_angles* ang,
                                                            const pilco_particles_noise* nz,
                                                            const pilco_policy_schedule* sch, int R);
int    pilco_particles_scheduled_score_grad_rollout(const pilco_particles* pr, const pilco_angles* ang,
                                                    const pilco_particles_noise* nz, const pilco_policy_schedule* sch,
                                                    int R, const pilco_particles_grad* g, pilco_stream_t stream);
size_t pilco_particles_scheduled_consistent_score_grad_workspace_bytes(const pilco_particles* pr,
                                                                       const pilco_angles* ang,
                                                                       const pilco_particles_noise* nz,
                                                                       const pilco_policy_schedule* sch, int R);
int    pilco_particles_scheduled_consistent_score_grad_rollout(const pilco_particles* pr, const pilco_angles* ang,
                                                               const pilco_particles_noise* nz,
                                                               const pilco_policy_schedule* sch, int R,
                                                               const pilco_particles_grad* g, pilco_stream_t stream);
size_t pilco_particles_scheduled_resampled_workspace_bytes(const pilco_particles* pr,
                                                           const pilco_particles_resample* rs,
                                                           const pilco_policy_schedule* sch);
int    pilco_particles_scheduled_resampled_rollout(const pilco_particles* pr, const pilco_particles_resample* rs,
                                                   const pilco_policy_schedule* sch, pilco_stream_t stream);
size_t pilco_particles_scheduled_resampled_grad_workspace_bytes(const pilco_particles* pr,
                                                                const pilco_particles_resample* rs,
                                                                const pilco_policy_schedule* sch, int R);
int    pilco_particles_scheduled_resampled_grad_rollout(const pilco_particles* pr, const pilco_particles_resample* rs,
                                                        const pilco_policy_schedule* sch, int R,
                                                        const pilco_particles_grad* g, pilco_stream_t stream);

/* Tanh MLP policies in the particle rollouts (DESIGN.md section 29), the policy class Deep PILCO trains on sampled
 * returns.  pr->pol.kind = PILCO_POLICY_MLP, pol.Ds / U / squash / max_action as for a linear policy, the network in
 * *mlp with L = 1 or 2 hidden layers of width[l] in 1 .. 64 units:
 *   h_1 = tanh(A_1 [x; 1]),  h_2 = tanh(A_2 [h_1; 1])  (L = 2),  z = A_out [h_L; 1],  u = max_action o sin(z) (squash,
 *   at output variance 0 as the linear policy) or z
 * Each A is row-major [out, in + 1], its last column the bias; theta is A_1, (A_2,) A_out in that order:
 *   n_theta = width[0] (Ds + 1) + (L = 2: width[1] (width[0] + 1)) + U (width[L-1] + 1)
 * restart r's at theta + r theta_bs (the gradient calls; 0: shared).  Every other field of pr and every output has the
 * meaning it has for a linear policy.  The gradient calls write value [R] and gtheta [R, n_theta] = d value / d theta
 * (g's linear and RBF fields are ignored); ex may be NULL, as in pilco_particles_explore_*.  Each call is its
 * sampler's linear-policy call (pilco_particles_rollout, _rollout_consistent, _resampled_rollout,
 * _rollout_batch_grad / _explore_batch_grad, _explore_consistent_grad, _resampled_grad_rollout) with the MLP in place
 * of the policy: no angles, measurement noise, schedule or score estimator.  Deterministic; a restart's results do
 * not depend on R.  Validation before any work is enqueued: the linear call's status codes with its policy checks
 * replaced by PILCO_ERR_UNSUPPORTED for pol.kind != PILCO_POLICY_MLP, PILCO_ERR_NULL for mlp or theta NULL,
 * PILCO_ERR_DIM for L outside {1, 2}, a width outside 1 .. 64 or theta_bs < 0, PILCO_ERR_UNSUPPORTED for theta_bs != 0
 * in a forward call; PILCO_ERR_NULL for gtheta NULL (gradient calls) with the gradient's outputs; then the sampler's
 * own codes; then the workspace's.  A size query returns 0 exactly where its call fails on sizes (mlp NULL included).
 * The linear and RBF calls return PILCO_ERR_UNSUPPORTED for PILCO_POLICY_MLP. */
typedef struct pilco_mlp {
    int L, width[2];
    const double* theta; long long theta_bs;
    double* gtheta;             /* [R, n_theta], gradient calls only */
} pilco_mlp;
size_t pilco_particles_mlp_workspace_bytes(const pilco_particles* pr, const pilco_mlp* mlp);
int    pilco_particles_mlp_rollout(const pilco_particles* pr, const pilco_mlp* mlp, pilco_stream_t stream);
size_t pilco_particles_mlp_consistent_workspace_bytes(const pilco_particles* pr, const pilco_mlp* mlp);
int    pilco_particles_mlp_consistent_rollout(const pilco_particles* pr, const pilco_mlp* mlp, pilco_stream_t stream);
size_t pilco_particles_mlp_resampled_workspace_bytes(const pilco_particles* pr, const pilco_mlp* mlp,
                                                     const pilco_particles_resample* rs);
int    pilco_particles_mlp_resampled_rollout(const pilco_particles* pr, const pilco_mlp* mlp,
                                             const pilco_particles_resample* rs, pilco_stream_t stream);
size_t pilco_particles_mlp_batch_grad_workspace_bytes(const pilco_particles* pr, const pilco_mlp* mlp,
                                                      const pilco_exploration* ex, int R);
int    pilco_particles_mlp_batch_grad_rollout(const pilco_particles* pr, const pilco_mlp* mlp,
                                              const pilco_exploration* ex, int R, const pilco_particles_grad* g,
                                              pilco_stream_t stream);
size_t pilco_particles_mlp_consistent_grad_workspace_bytes(const pilco_particles* pr, const pilco_mlp* mlp,
                                                           const pilco_exploration* ex, int R);
int    pilco_particles_mlp_consistent_grad_rollout(const pilco_particles* pr, const pilco_mlp* mlp,
                                                   const pilco_exploration* ex, int R, const pilco_particles_grad* g,
                                                   pilco_stream_t stream);
size_t pilco_particles_mlp_resampled_grad_workspace_bytes(const pilco_particles* pr, const pilco_mlp* mlp,
                                                          const pilco_particles_resample* rs, int R);
int    pilco_particles_mlp_resampled_grad_rollout(const pilco_particles* pr, const pilco_mlp* mlp,
                                                  const pilco_particles_resample* rs, int R,
                                                  const pilco_particles_grad* g, pilco_stream_t stream);

/* ---- function samples from random-feature draws (DESIGN.md section 30) -----------------------------------------
 * The consistent sampler's process (one dynamics function per particle and output, x_{t+1} = x_t + f_p(x~_t)) with
 * each function drawn once as a random-feature prior plus an exact data update (Wilson et al. 2020):
 *   omega_ei = zeta_ei / ell_e,  phi_e(x) = sqrt(sf2_e / F) [cos(omega_e x); sin(omega_e x)]  (2F features)
 *   v_pe = beta_e - iK_e (Phi_e(X) w_pe + sqrt(sn2_e) eps_pe),  f_pe(x~) = phi_e(x~)' w_pe + k_e(x~, X) v_pe
 * Given the frequencies, the sample's covariance is the posterior's with the F-feature prior in place of k; its cost
 * per particle, output and step is O(F + n), and no buffer grows with the horizon beyond the outputs and the
 * gradient's x~ history.  dyn must be the exact GP pilco_gp_factorize leaves (iK = (K + sn2 I)^-1 and sn2 the noise
 * variances it was factorised with): the C layer cannot tell a FITC model apart, and for one the update is wrong.
 *
 * pilco_particles_features_draw: omega [E,F,D] and v [P,E,n] from the caller's standard normals zeta [E,F,D] (shared
 * by all particles), w [P,E,2F] and eps_y [P,E,n]; sn2 [E] on the device.  Once per set of normals, not per rollout.
 * A particle's v is bitwise independent of P.  PILCO_ERR_NULL for a NULL pointer (dyn, its arrays, sn2, zeta, w,
 * eps_y, omega, v), PILCO_ERR_UNSUPPORTED for a model that is not unbatched mode 0 with iK, PILCO_ERR_DIM for sizes
 * out of range (P, F in 1 .. PILCO_MAX_FEATURES, n, D, E, ldk), then the workspace's codes.
 *
 * The rollouts take the draws in place of pr->eps (not read; it may be NULL) and otherwise are the consistent calls
 * they mirror: pilco_particles_features_rollout as pilco_particles_noisy_consistent_rollout,
 * _features_grad_rollout as pilco_particles_explore_consistent_grad_rollout (R restarts share the draws; restart r
 * is bitwise the R = 1 call with policy r), and the _mlp_ calls as pilco_particles_mlp_consistent_rollout /
 * _mlp_consistent_grad_rollout.  Same outputs, angles, noise and exploration rules (ang, nz, ex NULL: without them).
 * Validation before any work is enqueued: the mirrored call's codes up to its workspace check (pr->eps excepted),
 * then PILCO_ERR_NULL for fd, omega, w or v NULL, PILCO_ERR_DIM for F outside 1 .. PILCO_MAX_FEATURES, then the
 * workspace's codes.  A size query returns 0 exactly where its call fails on sizes (fd NULL included).
 * Deterministic, no host synchronisation (graph-capturable); a particle's outputs depend neither on P nor on its row. */
#define PILCO_MAX_FEATURES 8192
typedef struct pilco_feature_draws {
    int F;                      /* 1 .. 8192 frequency pairs per output */
    const double* omega;        /* [E,F,D] written by the draw call */
    const double* w;            /* [P,E,2F] the caller's standard normals */
    const double* v;            /* [P,E,n]  written by the draw call */
} pilco_feature_draws;
size_t pilco_particles_features_draw_workspace_bytes(const pilco_gp_model* dyn, int P, int F);
int    pilco_particles_features_draw(const pilco_gp_model* dyn, const double* sn2, int P, int F, const double* zeta,
                                     const double* w, const double* eps_y, double* omega, double* v,
                                     void* ws, size_t ws_bytes, pilco_stream_t stream);
size_t pilco_particles_features_workspace_bytes(const pilco_particles* pr, const pilco_angles* ang,
                                                const pilco_particles_noise* nz, const pilco_feature_draws* fd);
int    pilco_particles_features_rollout(const pilco_particles* pr, const pilco_angles* ang,
                                        const pilco_particles_noise* nz, const pilco_feature_draws* fd,
                                        pilco_stream_t stream);
size_t pilco_particles_features_grad_workspace_bytes(const pilco_particles* pr, const pilco_angles* ang,
                                                     const pilco_particles_noise* nz, const pilco_exploration* ex,
                                                     const pilco_feature_draws* fd, int R);
int    pilco_particles_features_grad_rollout(const pilco_particles* pr, const pilco_angles* ang,
                                             const pilco_particles_noise* nz, const pilco_exploration* ex,
                                             const pilco_feature_draws* fd, int R, const pilco_particles_grad* g,
                                             pilco_stream_t stream);
size_t pilco_particles_mlp_features_workspace_bytes(const pilco_particles* pr, const pilco_mlp* mlp,
                                                    const pilco_feature_draws* fd);
int    pilco_particles_mlp_features_rollout(const pilco_particles* pr, const pilco_mlp* mlp,
                                            const pilco_feature_draws* fd, pilco_stream_t stream);
size_t pilco_particles_mlp_features_grad_workspace_bytes(const pilco_particles* pr, const pilco_mlp* mlp,
                                                         const pilco_exploration* ex, const pilco_feature_draws* fd,
                                                         int R);
int    pilco_particles_mlp_features_grad_rollout(const pilco_particles* pr, const pilco_mlp* mlp,
                                                 const pilco_exploration* ex, const pilco_feature_draws* fd, int R,
                                                 const pilco_particles_grad* g, pilco_stream_t stream);

/* ---- batched forward-only scheduled rollouts and the cross-entropy method (DESIGN.md section 31) ------------------
 * pilco_particles_scheduled_batch_rollout / _scheduled_consistent_batch_rollout: the forward of
 * pilco_particles_scheduled_batch_grad_rollout / _scheduled_consistent_grad_rollout (ex NULL) without the reverse sweep
 * or its histories.  R restarts share x0, eps (and nu); restart r runs the schedule at pol.W + r pol.W_bs + t W_ts and
 * pol.b + r pol.b_bs + t b_ts.  The outputs have a leading R as in the gradient calls, and value [R] is the fixed-order
 * mean return.  Outputs and value are bitwise the gradient call's; restart r is bitwise
 * pilco_particles_scheduled_rollout (_consistent_rollout) with restart r's schedule.  ang and nz may be NULL.  The
 * workspace is pr->ws.  Validation before any work is enqueued: the gradient call's codes with PILCO_ERR_NULL for value
 * NULL in place of its gradient-output checks, then the workspace's codes.  A size query returns 0 exactly where its
 * call fails on sizes.  Deterministic, no host synchronisation (graph-capturable).
 *
 * pilco_cem_update: one iteration of the cross-entropy method over K candidate sequences cand [K,H,U] scored value
 * [K] (a batched rollout's value with b = cand, b_bs = H U, b_ts = U), in this order:
 *   1. rank: value descending, NaN last, ties to the lower index; the elites are the first n_elite in rank order
 *   2. refit per (t, u): m_e, v_e the elites' mean and biased variance (two passes, summed in rank order);
 *      mean <- alpha mean + (1 - alpha) m_e, std <- sqrt(alpha std^2 + (1 - alpha) v_e)
 *   3. best so far: when the top value is strictly above *best_value, it and its candidate go to best_value and best
 *   4. next candidates (xi not NULL): row 0 = clip(mean, lo, hi), row k >= 1 = clip(mean + std o xi_k, lo, hi)
 *   5. trace (not NULL): trace[0] = the top value, trace[1] = the elites' mean value (rank-order sum / n_elite)
 * pilco_cem_draw: step 4 alone (the first candidates); it reads cand, xi, mean, std, K, H, U, lo and hi.
 * Validation before any work is enqueued: PILCO_ERR_NULL for c or a pointer the call uses (update: value, cand, mean,
 * std, best_value, best; draw: cand, xi, mean, std), then PILCO_ERR_DIM for K outside 1 .. 8192, H < 1, U < 1,
 * H U > 2^24, lo >= hi (or a NaN bound) and (update) n_elite outside 1 .. K or alpha outside [0, 1), then the
 * workspace's codes (NULL, PILCO_ERR_ALIGN below 16-byte alignment, PILCO_ERR_WORKSPACE).  The workspace query returns
 * 0 exactly for K outside 1 .. 8192.  Deterministic (no atomics), no host synchronisation (graph-capturable). */
size_t pilco_particles_scheduled_batch_workspace_bytes(const pilco_particles* pr, const pilco_angles* ang,
                                                       const pilco_particles_noise* nz,
                                                       const pilco_policy_schedule* sch, int R);
int    pilco_particles_scheduled_batch_rollout(const pilco_particles* pr, const pilco_angles* ang,
                                               const pilco_particles_noise* nz, const pilco_policy_schedule* sch,
                                               int R, double* value, pilco_stream_t stream);
size_t pilco_particles_scheduled_consistent_batch_workspace_bytes(const pilco_particles* pr, const pilco_angles* ang,
                                                                  const pilco_particles_noise* nz,
                                                                  const pilco_policy_schedule* sch, int R);
int    pilco_particles_scheduled_consistent_batch_rollout(const pilco_particles* pr, const pilco_angles* ang,
                                                          const pilco_particles_noise* nz,
                                                          const pilco_policy_schedule* sch, int R, double* value,
                                                          pilco_stream_t stream);
typedef struct pilco_cem {
    int K, H, U;                /* candidates, steps, action width */
    int n_elite;                /* 1 .. K */
    double alpha;               /* smoothing in [0, 1) */
    double lo, hi;              /* the candidates' bounds, lo < hi */
    const double* value;        /* [K] the candidates' values */
    double* cand;               /* [K,H,U] in: the scored candidates; out: the next ones */
    const double* xi;           /* [K,H,U] standard normals of the next candidates (row 0 unread); NULL: no draw */
    double* mean;               /* [H,U] the sampling mean, updated in place */
    double* std;                /* [H,U] the sampling standard deviation, updated in place */
    double* best_value;         /* [1] the best value so far (-inf before the first iteration) */
    double* best;               /* [H,U] its candidate */
    double* trace;              /* [2] this iteration's (top value, elites' mean value), or NULL */
} pilco_cem;
size_t pilco_cem_update_workspace_bytes(int K);
int    pilco_cem_update(const pilco_cem* c, void* ws, size_t ws_bytes, pilco_stream_t stream);
int    pilco_cem_draw(const pilco_cem* c, pilco_stream_t stream);

/* ---- batched forward-only rollouts of stationary policies (DESIGN.md section 33) ------------------------------------
 * pilco_particles_batch_rollout / _consistent_batch_rollout: the forward of pilco_particles_explore_batch_grad_rollout /
 * _explore_consistent_grad_rollout (ex NULL) without the reverse sweep or its histories, for a linear or RBF policy.
 * pilco_particles_mlp_batch_rollout / _mlp_consistent_batch_rollout: the same of pilco_particles_mlp_batch_grad_rollout
 * / _mlp_consistent_grad_rollout (ex NULL) for a tanh MLP policy (no angles or noise, as every MLP call).  R restarts
 * share x0, eps (and nu); restart r reads its policy at the batch strides (linear W_bs, b_bs; RBF the batched policy
 * model's strides; MLP theta_bs).  The outputs have a leading R as in the gradient calls, and value [R] is the
 * fixed-order mean return of the gradient calls' value CTA.  Outputs and value are bitwise the gradient call's; restart
 * r is bitwise the single forward call (pilco_particles_noisy_rollout / _noisy_consistent_rollout,
 * pilco_particles_mlp_rollout / _mlp_consistent_rollout) with restart r's policy.  ang and nz may be NULL.  The
 * workspace is pr->ws; the step-wise sampler's does not grow with H.  Validation before any work is enqueued: the
 * gradient call's codes with PILCO_ERR_NULL for value NULL in place of its gradient-output checks, then the workspace's
 * codes.  A size query returns 0 exactly where its call fails on sizes.  Deterministic, no host synchronisation
 * (graph-capturable). */
size_t pilco_particles_batch_workspace_bytes(const pilco_particles* pr, const pilco_angles* ang,
                                             const pilco_particles_noise* nz, int R);
int    pilco_particles_batch_rollout(const pilco_particles* pr, const pilco_angles* ang,
                                     const pilco_particles_noise* nz, int R, double* value, pilco_stream_t stream);
size_t pilco_particles_consistent_batch_workspace_bytes(const pilco_particles* pr, const pilco_angles* ang,
                                                        const pilco_particles_noise* nz, int R);
int    pilco_particles_consistent_batch_rollout(const pilco_particles* pr, const pilco_angles* ang,
                                                const pilco_particles_noise* nz, int R, double* value,
                                                pilco_stream_t stream);
size_t pilco_particles_mlp_batch_workspace_bytes(const pilco_particles* pr, const pilco_mlp* mlp, int R);
int    pilco_particles_mlp_batch_rollout(const pilco_particles* pr, const pilco_mlp* mlp, int R, double* value,
                                         pilco_stream_t stream);
size_t pilco_particles_mlp_consistent_batch_workspace_bytes(const pilco_particles* pr, const pilco_mlp* mlp, int R);
int    pilco_particles_mlp_consistent_batch_rollout(const pilco_particles* pr, const pilco_mlp* mlp, int R,
                                                    double* value, pilco_stream_t stream);

/* ---- counter-based normals and the Adam step (DESIGN.md section 32) -----------------------------------------------
 * pilco_normals: out[0 .. n) standard normals.  Normal i is a pure function of (seed, stream_id, *iter, i): Philox4x32-10
 * (curand's Philox4_32_10) of the counter (j low 32 bits, j high 32 bits, stream_id, low 32 bits of *iter), j = i / 2,
 * under the key (seed low 32 bits, seed high 32 bits) gives x0..x3; u1 = (((x0 << 32 | x1) >> 11) + 0.5) 2^-53 and u2
 * likewise from (x2, x3), both in (0, 1); r = sqrt(-2 log u1), element 2j = r cospi(2 u2), element 2j + 1 =
 * r sinpi(2 u2).  *iter is read on the device when the kernel runs, so a captured graph draws new normals at every
 * replay after something advances it (pilco_adam_update does).  The bits depend neither on the grid nor on n (a call's
 * first n elements are the n call's).  Validation before any work is enqueued: PILCO_ERR_NULL for iter or out NULL,
 * PILCO_ERR_DIM for n < 0; n = 0 enqueues nothing.  Deterministic, no host synchronisation (graph-capturable).
 *
 * pilco_adam_update: one Adam step of R restarts' flat parameters theta [R, n] (row stride ld_theta) from the packed rows
 * [loss | status | gradient of loss [n]] (row stride ld_packed, read only), then *iter += 1.  For each restart r:
 *   ok_r = status_r == 0, loss_r finite and every gradient entry finite
 *   if ok_r:  max_norm > 0 and ||g_r|| > max_norm: g_r <- g_r (max_norm / ||g_r||)   (||.||^2 summed in a fixed order)
 *             t_r += 1, b1t_r <- b1t_r b1, b2t_r <- b2t_r b2                           (running products b^t, no pow)
 *             m_r <- b1 m_r + (1 - b1) g_r,  v_r <- b2 v_r + (1 - b2) g_r o g_r
 *             theta_r <- theta_r - lr (m_r / (1 - b1t_r)) / (sqrt(v_r / (1 - b2t_r)) + eps)
 *   k = *iter (read before the increment): when 0 <= k < trace_rows, trace[k, r] = -loss_r and ok[k, r] = ok_r
 * A restart that is not ok keeps theta, m, v, t and its running products; no restart reads another's row.  Every
 * product, sum, quotient and square root is rounded once (no fma), so a host build of sgd_math.cuh gives the same bits.
 * Start a run with m = v = 0, t = 0, b1t = b2t = 1.  Validation before any work is enqueued: PILCO_ERR_NULL for a NULL
 * a, theta, packed, m, v, t, b1t, b2t or iter (trace and ok too when trace_rows > 0), then PILCO_ERR_DIM for R < 1,
 * n < 1, ld_theta < n, ld_packed < n + 2, trace_rows < 0, lr <= 0 or not finite, b1 or b2 outside [0, 1), eps <= 0
 * (or NaN) and max_norm < 0 (or NaN).  Deterministic (no atomics), no host synchronisation (graph-capturable). */
int pilco_normals(unsigned long long seed, unsigned stream_id, const long long* iter, long long n, double* out,
                  pilco_stream_t stream);
typedef struct pilco_adam {
    int R, n;                   /* restarts, parameters per restart */
    double lr, b1, b2, eps;     /* step size > 0, moment decays in [0, 1), eps > 0 */
    double max_norm;            /* clip ||g|| to it when > 0; 0: no clipping */
    double* theta;              /* [R, ld_theta] the parameters, updated in place */
    int ld_theta;               /* >= n */
    const double* packed;       /* [R, ld_packed] rows [loss | status | gradient of loss] */
    int ld_packed;              /* >= n + 2 */
    double* m;                  /* [R, n] first moments */
    double* v;                  /* [R, n] second moments */
    long long* t;               /* [R] steps taken */
    double* b1t;                /* [R] b1^t */
    double* b2t;                /* [R] b2^t */
    long long* iter;            /* [1] the iteration counter k */
    double* trace;              /* [trace_rows, R] -loss of iteration k */
    int* ok;                    /* [trace_rows, R] whether iteration k stepped */
    int trace_rows;             /* >= 0 */
} pilco_adam;
int pilco_adam_update(const pilco_adam* a, pilco_stream_t stream);

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
