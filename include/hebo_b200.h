/*
 * hebo_b200.h -- C ABI of libhebo_b200.so: the H100 (sm_90a) implementation of HEBO's
 * exact-GP fit + batched posterior/MACE hot path.
 *
 * This is the drop-in boundary a HEBO maintainer binds with ctypes (see INTEGRATION.md).
 * Every entry point cites the reference code it replaces (paths relative to the reference
 * checkout, HEBO/hebo/...).  The arithmetic the reference delegates to gpytorch
 * (Gram / Cholesky / solves / log-det / predictive variance; requirements.txt:6) is restated
 * in SURVEY.md Appendix A and implemented here from scratch.
 *
 * Conventions
 *   - extern "C", plain pointers and sizes; no torch / C++ types cross the boundary.
 *   - Unless marked HOST, every pointer is a DEVICE pointer (tensor.data_ptr()).
 *   - fp32, row-major.  Square work matrices use the padded order NP = hb_padded_n(n)
 *     (next multiple of 128) with leading dimension NP; the pad is an identity block.
 *   - `stream` is a cudaStream_t passed as void* (torch.cuda.current_stream().cuda_stream).
 *   - The caller owns all memory, keeps it alive until the stream work completes; the
 *     library retains nothing between calls except lazily-built per-device state (kernel
 *     attributes, device-resident tile tables of the tensor-core fit stages, one capture stream).
 *   - Threading: like the reference (every call comes from the Python main thread,
 *     optimizers/hebo.py:143-186), one in-flight call per process and device; the lazily-built
 *     state is not guarded by locks.  hb_cholesky / hb_fit use a cooperative launch whose CTAs
 *     synchronise through flags in the caller's workspace: give concurrent calls distinct
 *     workspaces.
 *   - Return value: HB_OK, or an error below.  Never throws / aborts across the ABI.
 *     "Not positive definite" is reported through the device word `info` (LAPACK style:
 *     0 = ok, j>0 = leading minor j not PD) so the caller can reproduce the reference's
 *     jitter escalation (models/gp/gp.py:104-126, 140-157) without a CUDA error.
 *
 * Hyper-parameter vectors (P = d + 3 floats, gpytorch registration order, SURVEY Appendix A):
 *   raw[0] = raw_noise, raw[1] = mean constant, raw[2] = raw_outputscale, raw[3..3+d) = raw_lengthscale
 *   hyp[0] = sigma_n^2 = softplus(raw_noise)+noise_lb, hyp[1] = c, hyp[2] = s = softplus(raw_os),
 *   hyp[3..3+d) = lengthscale = softplus(raw_ls)
 *
 * Mixed numeric + categorical models and ard_kernel=False (the `_ex` entry points, hb_model_spec_t): the reference's
 * EmbTransform (models/layers.py:14-34: one nn.Embedding(num_uniq_c, emb_size_c) per categorical column, outputs
 * concatenated) feeds  ScaleKernel(Matern(ARD, numeric dims) * Matern-3/2(one lengthscale, embedding dims))
 * (models/gp/gp_util.py:39-59); the tables are trained inside the MLL.  Parameter order = module registration order:
 *   raw = (raw_noise, table_0 [num_uniq_0, emb_0] row-major, table_1, ..., [warp: raw_a[d], raw_b[d]], mean,
 *          raw_outputscale, raw_lengthscale[d if ard else 1] (absent when d = 0), raw_emb_lengthscale (when num_enum > 0))
 *   hyp = (sigma_n^2, c, s, lengthscale per numeric dim [d] (the shared one repeated when ard = 0), emb lengthscale,
 *          [warp: a[d], b[d] = 0.01 + 9.99 sigmoid(raw)])
 * With a warp the numeric features are z = (2 w(u) - 1) / l,  u = clamp((x~ + 1) / 2, 1e-6, 1 - 1e-6),  w = 1 - (1 - u^a)^b
 * (x~ = MinMax(-1,1)-scaled input); training rows are warped once per epoch (O(n d)), candidates inside the K* load stage.
 * hb_num_params() gives P.  Categories travel as int32 [rows, num_enum].
 */
#ifndef HEBO_B200_H
#define HEBO_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define HB_OK              0
#define HB_ERR_INVALID     1   /* bad argument (null pointer, size, unknown kernel id) */
#define HB_ERR_NOT_PD      2   /* host-visible "not positive definite" (hb_fit only)   */
#define HB_ERR_CUDA        3   /* CUDA runtime error; see hb_last_error()               */

#define HB_KERN_MATERN32   0   /* reference default: models/gp/gp_util.py:46 (nu = 1.5) */
#define HB_KERN_MATERN52   1   /* conf['kern'] injection, models/gp/gp.py:201            */
#define HB_KERN_RBF        2
#define HB_KERN_MATERN12   4   /* gpytorch MaternKernel(nu=0.5), through conf['kern'], models/gp/gp.py:201.
                                  Ids 3 and 5-7 are not kernels: every entry point that takes kern rejects them. */

/* Largest feature count d + De (numeric dims plus the summed embedding widths of the categorical columns) a model may
 * have.  Every entry point that takes a model description returns HB_ERR_INVALID above it (hb_num_params and the
 * workspace queries return -1).  The kernels stream features in 32-wide chunks, so shared memory does not grow with it. */
#define HB_MAX_FEATURES    4096

/* Most outputs one batched fit (hb_fit_multi_ex) trains together. */
#define HB_MAX_OUTPUTS     32

/* Most objectives the k-objective survival (hb_nsga2_survive_k) and front (hb_pareto_front_k) take. */
#define HB_MAX_OBJ         8

/* Model description beyond the numeric ARD default (HOST struct; NULL = numeric-only, ard_kernel=True). */
typedef struct {
  int32_t        ard_kernel;  /* conf['ard_kernel'] (models/gp/gp.py:47, gp_util.py:45): 0 = one shared numeric lengthscale */
  int32_t        num_enum;    /* categorical columns e (0 = none)                                                          */
  const int32_t *num_uniqs;   /* HOST [e] categories per column (conf['num_uniqs'], optimizers/hebo.py:99-100)            */
  const int32_t *emb_sizes;   /* HOST [e] embedding widths (models/layers.py:19 default min(50, 1 + num_uniq // 2))       */
  int32_t        warp;        /* Kumaraswamy input warp of the numeric dims (BASELINE config 3; KumarWarp,
                                 models/nn/mono_layers/layers.py:85-117): 0 none, 1 exponents a, b LEARNED inside the MLL
                                 (2 d more parameters), 2 exponents fixed at the values in raw (never updated)             */
} hb_model_spec_t;

/* ---- library info (HOST) -------------------------------------------------------------- */
int32_t     hb_version(void);
const char *hb_last_error(void);                    /* last CUDA error string of this thread */
int64_t     hb_padded_n(int64_t n);                 /* NP: next multiple of 128               */
int32_t     hb_vnorm_operand_kind(void);            /* layout of hb_fit_state_t.Linv_hi/lo: 0 = two-level fp16 split (the only one built) */
/* Measurement hooks used by bench.py (HOST): number of kernels this library launched since the last reset, and
 * CUDA-event timing of the dominant kernel (the posterior variance contraction) on its launching stream. */
int64_t     hb_launch_count(int32_t reset);
int32_t     hb_profile_enable(int32_t on);
int32_t     hb_profile_collect(double *total_ms, int32_t *n_launches);
/* rows_flagged[0] = candidate rows that went through the tensor path since the last reset, [1] = how many of them the
 * precision guard re-contracted on the FP32 pipe (synchronises the device; current device only). */
int32_t     hb_guard_stats(uint64_t *rows_flagged, int32_t reset);
/* Workspace sizes in BYTES for the fused calls below. */
int64_t     hb_fit_workspace_bytes(int64_t n, int64_t d);
int64_t     hb_fit_workspace_bytes_ex(int64_t n, int64_t d, const hb_model_spec_t *spec);
int64_t     hb_num_params(int64_t d, const hb_model_spec_t *spec);      /* P: length of raw / grad / a Langevin row */
int64_t     hb_posterior_workspace_bytes(int64_t n, int64_t d, int64_t m_chunk);
int64_t     hb_pareto_workspace_bytes(int64_t m);

/* ---- hyper-parameter transform ---------------------------------------------------------
 * gpytorch Positive()/GreaterThan() constraints used at models/gp/gp.py:86 and
 * models/gp/gp_util.py:46,57: hyp = softplus(raw) (+ noise_lb for the noise). */
int32_t hb_transform_hypers(const float *raw, int64_t d, float noise_lb, float *hyp, void *stream);

/* ---- lengthscale initialisation  (models/gp/gp_util.py:47-52: per-dimension median of the pairwise |dx| over
 * <= 1000 rows, clamp >= 0.02) ------------------------------------------------------------------------------
 * Xt [d, NP] transposed scaled inputs; idx [d, k] int32 row subsets (np.random.choice per dimension) or NULL = rows
 * 0..k-1; k <= 1024.  out[d] = max(lower median of the k(k-1)/2 differences, clamp_min)  (torch.median semantics). */
int32_t hb_median_pdist(const float *Xt, int64_t n, int64_t d, const int32_t *idx, int64_t k, float clamp_min,
                        float *out, void *stream);

/* ---- Gram matrix  (replaces GPyTorchModel.forward -> self.cov(x_all), models/gp/gp.py:203-207,
 * kernel built at models/gp/gp_util.py:39-59) -----------------------------------------------
 * Xt       [d, NP] TRANSPOSED MinMax-scaled training inputs (column i = point i; pad columns ignored).  The same holds
 *          for the Xt of hb_mll_grad, hb_fit, hb_fit_ex, hb_fit_multi_ex, hb_mll_fwd_bwd, hb_factorize and
 *          hb_factorize_ex: the pad columns may hold anything, NaN and Inf included, and no result depends on them or on
 *          what the workspace held before the call.
 * K        [NP, NP] out: lower triangle (incl. diagonal) of s*k(X,X) + (sigma_n^2 + jitter [+ noise_diag_i]) I;
 *          pad block = identity.  The strict upper triangle of off-diagonal tiles is not written.
 * noise_diag  [n] or NULL: per-row extra noise (BASELINE config 4 "heteroscedastic"; no reference). */
int32_t hb_gram(const float *Xt, int64_t n, int64_t d, const float *hyp, int32_t kern,
                const float *noise_diag, float jitter, float *K, void *stream);

/* ---- Cholesky  (replaces gpytorch psd_safe_cholesky inside ExactMarginalLogLikelihood /
 * the prediction strategy; call sites models/gp/gp.py:112-113, 148) ---------------------------
 * A [NP, NP] in/out, lower triangle; blocked right-looking, in place.  ws: >= 128*128*4 bytes.
 * info: device int32, set to j>0 if the leading minor j is not PD (left 0 otherwise; caller zeroes). */
int32_t hb_cholesky(float *A, int64_t np, float *ws, int32_t *info, void *stream);

/* ---- Triangular inverse and K^-1 (the n^3-class part of autograd's backward through the MLL,
 * models/gp/gp.py:115 loss.backward()) ---------------------------------------------------------
 * Linv = L^-1 (lower, strict upper zero-filled); tmp: [NP, NP] scratch.
 * Kinv = Linv^T Linv: lower tiles only. */
int32_t hb_tri_inverse(const float *L, int64_t np, float *Linv, float *tmp, void *stream);
int32_t hb_kinv(const float *Linv, int64_t np, float *Kinv, void *stream);

/* ---- Tensor-core twins of hb_cholesky / hb_tri_inverse / hb_kinv: the stages every pSGLD epoch of hb_fit* runs, with
 * their O(NP^3) GEMMs on the 3xTF32 tensor cores (each fp32 operand split hi + lo, products hi*hi + hi*lo + lo*hi).
 * tc_ws: device workspace of >= hb_tc_workspace_bytes(np) bytes (tc_ws_bytes = its size), laid out like the fit
 * workspace's own tensor-core block: the hi/lo copies of L, L^-1, U = L^-T, the doubling products and the Cholesky panel.
 * NP > 0 and a multiple of 128, no NULL pointer and a large enough tc_ws, otherwise HB_ERR_INVALID before any launch.
 * hb_cholesky_tc     as hb_cholesky; the trailing update right of each 512-column outer block on the tensor cores.
 * hb_tri_inverse_tc  Linv = L^-1 (lower; Linv and the strict upper triangles of the hi/lo copies are zero-filled first).
 *                    128 x 128 diagonal blocks on the FP32 pipe, the doubling levels on the tensor cores; also leaves
 *                    the split of U = Linv^T in tc_ws.
 * hb_kinv_tc         Kinv = U U^T from the U that the last hb_tri_inverse_tc left in the same tc_ws: every lower 128-tile,
 *                    and an upper tile only where a 256-column output tile of its tile row overhangs the diagonal
 *                    (columns < min(NP, round_up(r0 + 128, 256)) of tile row r0); nothing else is written. */
int64_t hb_tc_workspace_bytes(int64_t np);
int32_t hb_cholesky_tc(float *A, int64_t np, float *ws, int32_t *info, void *tc_ws, int64_t tc_ws_bytes, void *stream);
int32_t hb_tri_inverse_tc(const float *L, int64_t np, float *Linv, void *tc_ws, int64_t tc_ws_bytes, void *stream);
int32_t hb_kinv_tc(int64_t np, float *Kinv, void *tc_ws, int64_t tc_ws_bytes, void *stream);

/* ---- alpha, quadratic form, log-det  (the data term of ExactMarginalLogLikelihood,
 * models/gp/gp.py:102,113; alpha is also the prediction-strategy mean cache, gp.py:148) --------
 * r = y - c (pad = 0).  alpha = Khat^-1 r, quad = r^T Khat^-1 r, logdet = 2 sum log L_ii.
 * scal[0] = quad, scal[1] = logdet (device, fp64 accumulated, stored as double[2]).
 * 1 <= n <= NP, otherwise HB_ERR_INVALID before any launch.
 * ws: >= (1 + NP/64)*NP*sizeof(double). */
int32_t hb_solve_logdet(const float *L, const float *Linv, const float *y, int64_t n, int64_t np,
                        const float *hyp, float *alpha, double *scal, void *ws, void *stream);

/* ---- MLL gradient (closed form of SURVEY Appendix A; replaces loss.backward(), gp.py:115) ----
 * grad[P] = d(-mll/n)/d raw,  loss[0] = -mll/n including the Gamma(.5,.5) outputscale prior
 * (gp_util.py:57) and LogNormal(ln noise_guess, .5) noise prior (gp.py:87). */
int32_t hb_mll_grad(const float *Xt, int64_t n, int64_t d, const float *raw, const float *hyp,
                    int32_t kern, const float *Kinv, const float *alpha, const double *scal,
                    float noise_guess, float *grad, float *loss, void *ws, void *stream);

/* ---- pSGLD update  (models/nn/sgld.py:49-70 on torch.optim.RMSprop) --------------------------
 * xi: [P] N(0,1) draws or NULL (= pretrain phase, no Langevin noise).  Per element, each operation rounded on its own
 * (no FMA), a = rms_alpha:  v = sq a + (1 - a) (g g);  avg = sqrt(v) + eps;  raw += ((-lr) g) / avg;
 * then raw += (factor sqrt((2 lr) / avg)) xi;  square_avg = v. */
int32_t hb_psgld_step(float *raw, const float *grad, float *square_avg, int64_t p, float lr,
                      float rms_alpha, float rms_eps, float factor, const float *xi, void *stream);

/* ---- the whole fit loop  (GP.fit, models/gp/gp.py:96-135, optimizer='psgld') -----------------
 * Runs num_epochs x { transform, gram, cholesky, inverse, alpha/logdet, gradient, pSGLD } on
 * `stream` with one status read-back per epoch; on a not-PD epoch it retries with jitter x10 from
 * 1e-6 (fp32 value of gp.py:104-110) and gives up above 10 like gp.py:120-126.
 * langevin   [num_epochs, P] N(0,1) draws in registration order, or NULL for deterministic RMSprop.
 * losses     HOST [num_epochs] out (loss evaluated before each step), may be NULL.
 * After the loop it factorises at the final hypers and leaves in the workspace what predict needs;
 * hb_fit_state() returns the device pointers.  Returns HB_ERR_NOT_PD if the final factorisation fails. */
int32_t hb_fit(const float *Xt, const float *y, int64_t n, int64_t d, float *raw, int32_t kern,
               const float *noise_diag, float noise_lb, float noise_guess, float lr, int32_t num_epochs,
               const float *langevin, float *losses, void *ws, int64_t ws_bytes, void *stream);

/* Factorise at the hypers in `raw` and fill the predict state (used by hb_fit and by callers that
 * set hypers directly).  jitter_used HOST out (may be NULL). */
int32_t hb_factorize(const float *Xt, const float *y, int64_t n, int64_t d, const float *raw, int32_t kern,
                     const float *noise_diag, float noise_lb, float *jitter_used,
                     void *ws, int64_t ws_bytes, void *stream);

/* The general forms (mixed numeric + categorical inputs, ard_kernel=False; spec = NULL reduces to the calls above).
 * Xe DEVICE int32 [n, num_enum] training categories (NULL when num_enum = 0); Xt may be NULL when d = 0; raw [P] in the
 * order given at the top of this file; langevin [num_epochs, P]. */
int32_t hb_fit_ex(const float *Xt, const int32_t *Xe, const float *y, int64_t n, int64_t d, const hb_model_spec_t *spec,
                  float *raw, int32_t kern, const float *noise_diag, float noise_lb, float noise_guess, float lr,
                  int32_t num_epochs, const float *langevin, float *losses, void *ws, int64_t ws_bytes, void *stream);
int32_t hb_factorize_ex(const float *Xt, const int32_t *Xe, const float *y, int64_t n, int64_t d, const hb_model_spec_t *spec,
                        const float *raw, int32_t kern, const float *noise_diag, float noise_lb, float *jitter_used,
                        void *ws, int64_t ws_bytes, void *stream);
/* ---- batched fit of several outputs that share one training set (MultiTaskModel) -----------------------------------
 * Trains num_out (1 .. HB_MAX_OUTPUTS) independent single-output GPs on the same inputs Xt / Xe in one launch chain per
 * epoch.  The workspace is num_out consecutive single-output workspaces: slice b starts at ws + b * stride with
 * stride = hb_fit_workspace_bytes_ex(n, d, spec) and is, after the call, exactly what hb_fit_ex leaves in a workspace of
 * its own -- hb_fit_state_ex, the posterior / sample / gradient calls and hb_factorize_ex work on it unchanged.
 * Y [num_out, n] DEVICE targets; raw [num_out, P] DEVICE in/out; langevin [num_out, num_epochs, P] or NULL;
 * losses HOST [num_out, num_epochs] out (may be NULL); status HOST [num_out] out: HB_OK or HB_ERR_NOT_PD (final
 * factorisation of that output failed).  Each output runs the loop of hb_fit_ex on its own -- own epoch counter, own
 * jitter ladder, own give-up -- and its results equal those of hb_fit_ex on its slice bit for bit.  noise_diag [n] is
 * shared.  Returns HB_OK unless an argument is invalid or CUDA fails.  hb_fit_ex is the num_out = 1 case. */
int64_t hb_fit_multi_workspace_bytes(int64_t n, int64_t d, const hb_model_spec_t *spec, int64_t num_out);
int32_t hb_fit_multi_ex(const float *Xt, const int32_t *Xe, const float *Y, int64_t n, int64_t d, const hb_model_spec_t *spec,
                        int64_t num_out, float *raw, int32_t kern, const float *noise_diag, float noise_lb, float noise_guess,
                        float lr, int32_t num_epochs, const float *langevin, float *losses, int32_t *status, void *ws,
                        int64_t ws_bytes, void *stream);
/* One MLL forward + backward at `raw` (closure of models/gp/gp.py:111-116: loss = -mll(gp(X)) ; loss.backward()):
 * grad [P], loss [1], info [1] (Cholesky status, LAPACK style) are DEVICE outputs; jitter is added to the diagonal. */
int32_t hb_mll_fwd_bwd(const float *Xt, const int32_t *Xe, const float *y, int64_t n, int64_t d, const hb_model_spec_t *spec,
                       const float *raw, int32_t kern, const float *noise_diag, float noise_lb, float noise_guess, float jitter,
                       float *grad, float *loss, int32_t *info, void *ws, int64_t ws_bytes, void *stream);

typedef struct {
  float  *hyp;     /* [H]        constrained hypers                       */
  float  *L;       /* [NP, NP]   Cholesky factor (lower)                   */
  float  *Linv;    /* [NP, NP]   L^-1 (lower)                              */
  float  *alpha;   /* [NP]       Khat^-1 (y - c), pad = 0                  */
  float  *Zt;      /* [d + De, NP] Xt / lengthscale (transposed), then the embedding features / their lengthscale */
  double *scal;    /* [2]        quad, logdet                              */
  float  *Linv_hi; /* [NP, NP] floats of storage: OPAQUE tensor-path operands of Linv.  Default (fp16 two-level split):  */
  float  *Linv_lo; /* h0 = rn_fp16(Linv*2^k) as NP*NP halfs in Linv_hi; h1 = rn_fp16((Linv*2^k - h0)*2048) as NP*NP halfs  */
                   /* in Linv_lo, followed by the float scale 2^k.  (hb_vnorm_operand_kind() == 0)                         */
  float  *tab_s;   /* [T] embedding tables / embedding lengthscale (mixed models; candidate side of the posterior)        */
  int32_t *emb_meta; /* OPAQUE categorical layout arrays (mixed models)                                                    */
  float  *grad;    /* [P] gradient of the last MLL evaluation             */
  float  *loss;    /* [1] loss of the last MLL evaluation                 */
} hb_fit_state_t;
int32_t hb_fit_state(void *ws, int64_t n, int64_t d, hb_fit_state_t *out);     /* HOST */
int32_t hb_fit_state_ex(void *ws, int64_t n, int64_t d, const hb_model_spec_t *spec, hb_fit_state_t *out);     /* HOST */

/* ---- fused posterior + MACE  (GP.predict, models/gp/gp.py:137-164, and MACE.eval,
 * acquisitions/acq.py:146-171; Mean/Sigma acq.py:66-82 read mu/var) ----------------------------
 * Xs        [m, d] RAW candidates; x_mul/x_add [d]: MinMax scale_/min_ (models/scalers.py:86-87)
 * Zt, alpha, Linv, hyp: from hb_fit_state.  Linv_hi/Linv_lo: from hb_fit_state -> variance contraction on the
 *           wgmma tensor cores (error-compensated fp16 two-level split); both NULL -> FP32 SIMT contraction.
 * y_mean,y_std: TorchStandardScaler (models/scalers.py:56-60).  pred_likeli: gp.py:158-159.
 * tau,kappa,eps: MACE(best_y, kappa, eps).  xi1, xi2 [m]: the two torch.randn draws of acq.py:154-155
 *           (NULL -> Philox N(0,1) from `seed`, independent streams per row).
 * F [m,3] out (LCB, -logEI, -logPI) or NULL; mu [m], var [m] out or NULL (original y units).
 * ws: hb_posterior_workspace_bytes(n, d, m_chunk); candidates are processed in chunks of m_chunk. */
int32_t hb_posterior_mace(const float *Xs, int64_t m, int64_t n, int64_t d,
                          const float *x_mul, const float *x_add,
                          const float *Zt, const float *alpha, const float *Linv,
                          const float *Linv_hi, const float *Linv_lo, const float *hyp, int32_t kern, float y_mean, float y_std, int32_t pred_likeli,
                          float tau, float kappa, float eps, const float *xi1, const float *xi2,
                          uint64_t seed, float *F, float *mu, float *var,
                          void *ws, int64_t ws_bytes, int64_t m_chunk, void *stream);

/* General form: Xe_s DEVICE int32 [m, num_enum] candidate categories, emb_meta / tab_s from hb_fit_state_ex
 * (all three NULL when num_enum = 0); Zt has d + De rows.  rng_offset: position of row 0 in the Philox stream (row r
 * draws the normals of stream position rng_offset + r), so a batch scored in several calls -- e.g. chunk by chunk while
 * the next chunk's host->device copy is in flight -- gets the same draws as one call over the whole batch. */
int32_t hb_posterior_mace_ex(const float *Xs, const int32_t *Xe_s, int64_t m, int64_t rng_offset, int64_t n, int64_t d,
                             const hb_model_spec_t *spec,
                             const int32_t *emb_meta, const float *tab_s, const float *x_mul, const float *x_add,
                             const float *Zt, const float *alpha, const float *Linv, const float *Linv_hi,
                             const float *Linv_lo, const float *hyp, int32_t kern, float y_mean, float y_std, int32_t pred_likeli,
                             float tau, float kappa, float eps, const float *xi1, const float *xi2, uint64_t seed, float *F,
                             float *mu, float *var, void *ws, int64_t ws_bytes, int64_t m_chunk, void *stream);

/* ---- GP.predict with gradients  (the `support_grad` contract: models/base_model.py:27-29 and
 * test/test_base_model.py:94-108 require predict() to be differentiable in Xc; gpytorch autograd through
 * models/gp/gp.py:137-164) -------------------------------------------------------------------------------------
 * Same inputs as hb_posterior_mace (FP32 SIMT contraction; Linv only).  mu, var [m] as above;
 * dmu, dvar [m, d] = d mu / d Xs, d var / d Xs (closed form; zero where a variance floor is active, like clamp_min).
 * ws: hb_posterior_workspace_bytes(n, d, m_chunk).
 * No input warp: hb_posterior_grad_ex returns HB_ERR_INVALID for spec->warp != 0.  A warped model's caller applies the
 * Kumaraswamy warp in front, as hebo_b200.GP._predict_autograd does -- Xs = the warped MinMax-scaled rows, x_mul = 1,
 * x_add = 0, spec->warp = 0 -- and chains dw/dx onto dmu / dvar itself. */
int32_t hb_posterior_grad(const float *Xs, int64_t m, int64_t n, int64_t d,
                          const float *x_mul, const float *x_add,
                          const float *Zt, const float *alpha, const float *Linv, const float *hyp, int32_t kern,
                          float y_mean, float y_std, int32_t pred_likeli,
                          float *mu, float *var, float *dmu, float *dvar,
                          void *ws, int64_t ws_bytes, int64_t m_chunk, void *stream);

int32_t hb_posterior_grad_ex(const float *Xs, const int32_t *Xe_s, int64_t m, int64_t n, int64_t d, const hb_model_spec_t *spec,
                             const int32_t *emb_meta, const float *tab_s, const float *x_mul, const float *x_add,
                             const float *Zt, const float *alpha, const float *Linv, const float *hyp, int32_t kern, float y_mean,
                             float y_std, int32_t pred_likeli, float *mu, float *var, float *dmu, float *dvar, void *ws,
                             int64_t ws_bytes, int64_t m_chunk, void *stream);

/* ---- joint posterior samples  (GP.sample_y, models/gp/gp.py:166-177: pred.rsample(n_samples) of the [likelihood-]predictive
 * MultivariateNormal; used by NoisyAcq / GeneralBO, optimizers/general.py:131) ------------------------------------------
 * z [n_samples, m] N(0,1) draws (the caller's torch.randn, so the random stream stays the caller's); out [n_samples, m] in
 * original y units = (mu~ + R z) y_std + y_mean with R the Cholesky root of K** - V V^T (+ sigma_n^2 I with pred_likeli)
 * + jitter I, jitter from 1e-6 x10 per failed attempt (gpytorch psd_safe_cholesky, fp32); m <= 8192.  hyp_host: HOST copy of
 * hyp (noise / outputscale feed launch parameters).  Everything -- K*, K**, the rank-n update, the factorisation -- runs in
 * this library's kernels; the call synchronises once per factorisation attempt. */
int64_t hb_sample_workspace_bytes(int64_t n, int64_t d, const hb_model_spec_t *spec, int64_t m);
int32_t hb_sample_y(const float *Xs, const int32_t *Xe_s, int64_t m, int64_t n, int64_t d, const hb_model_spec_t *spec,
                    const int32_t *emb_meta, const float *tab_s, const float *x_mul, const float *x_add, const float *Zt,
                    const float *alpha, const float *Linv, const float *hyp, const float *hyp_host, int32_t kern, float y_mean,
                    float y_std, int32_t pred_likeli, const float *z, int32_t n_samples, float *out, float *jitter_used, void *ws,
                    int64_t ws_bytes, void *stream);

/* ---- one joint sample of a GA batch on the device  (NoisyAcq.eval, acquisitions/acq.py:173-190: model.sample_y(x, xe),
 * one correlated draw per generation; GP.sample_y, models/gp/gp.py:166-177) ------------------------------------------
 * The fitted state and inputs of hb_sample_y (no host copy of hyp: sigma_n^2 and s are read from hyp on the device), with
 * 1 <= m <= 256 rows and ws_bytes >= hb_sample_workspace_bytes(n, d, spec, m).
 *   z [m] device N(0,1) draws by batch row, or NULL: in-kernel Philox4x32-10 + Box-Muller draws keyed by (seed, counter),
 *     e.g. counter = the generation index; the same (seed, counter) gives the same f bit for bit.
 *   f [m] device out: f = (mu~ + R z) y_std + y_mean, as hb_sample_y, over the DISTINCT rows.  A row equal to an earlier
 *     row of the batch (the duplicate predicate of hb_ga_survive: |a - b| <= 1e-16 in every numeric column, equal
 *     categories) is left out of the joint covariance, so that it cannot make it singular, and gets f = +inf; a distinct
 *     row's f is what the de-duplicated batch gives it.  R is a right-looking fp32 Cholesky of the distinct rows'
 *     covariance in one CTA, so f differs from hb_sample_y's (tile-DAG Cholesky) by the rounding of the factorisation.
 *   jitter [1] device out: the jitter of the accepted factorisation (ladder 1e-6 x10 per failed attempt, as hb_sample_y,
 *     run on the device); on give-up the last one tried.
 *   status [1] device int32: set to HB_ERR_NOT_PD when the ladder gives up (then f = NaN in every row), otherwise left
 *     unchanged, so one word zeroed by the caller collects the outcome of many calls.
 * No host read and no synchronisation: the call can be captured in a CUDA graph.  Six launches and one memset. */
int32_t hb_sample_y_batch(const float *Xs, const int32_t *Xe_s, int64_t m, int64_t n, int64_t d, const hb_model_spec_t *spec,
                          const int32_t *emb_meta, const float *tab_s, const float *x_mul, const float *x_add, const float *Zt,
                          const float *alpha, const float *Linv, const float *hyp, int32_t kern, float y_mean, float y_std,
                          int32_t pred_likeli, const float *z, uint64_t seed, uint64_t counter, float *f, float *jitter,
                          int32_t *status, void *ws, int64_t ws_bytes, void *stream);

/* ---- MACE epilogue alone  (MACE.eval, acquisitions/acq.py:151-171, over any model's predict output) ----
 * mu, var [m] in original y units (device); noise_var = model.noise (gp.py:182-184); xi1/xi2 as above.
 * F [m,3] out = (LCB, -logEI, -logPI). */
int32_t hb_mace_epilogue(const float *mu, const float *var, int64_t m, float noise_var, float tau, float kappa,
                         float eps, const float *xi1, const float *xi2, uint64_t seed, float *F, void *stream);

/* ---- single-objective acquisitions  (LCB / Mean / Sigma.eval, acquisitions/acq.py:55-82, and AbsEtaDifference.eval,
 * optimizers/nomr.py:25-34, over the mu / var that hb_posterior_mace_ex writes with F = NULL) ----
 * mu, var [m] device; f [m] out, one launch.  Each mode is the reference's torch expression in fp32 (py = mu, ps2 = var):
 *   HB_ACQ1_LCB      py - kappa * ps2.sqrt()
 *   HB_ACQ1_MEAN     py
 *   HB_ACQ1_SIGMA    -1 * ps2.sqrt()
 *   HB_ACQ1_ABS_ETA  abs(py - eta) - kappa * ps2.sqrt()
 * with correctly rounded sqrt, products and differences and no FMA contraction: bit-identical to the IEEE fp32 evaluation
 * of the same expression on the same mu / var.  torch's CPU sqrt (MKL VML, < 1 ulp) is not always correctly rounded, so the
 * reference's CPU eval may differ from it by one ulp.  kappa / eta are ignored by the modes that do not use them.  m >= 1. */
#define HB_ACQ1_LCB        0
#define HB_ACQ1_MEAN       1
#define HB_ACQ1_SIGMA      2
#define HB_ACQ1_ABS_ETA    3
int32_t hb_acq1_epilogue(const float *mu, const float *var, int64_t m, int32_t mode, float kappa, float eta, float *f,
                         void *stream);

/* ---- GeneralAcq epilogue  (GeneralAcq.eval, acquisitions/acq.py:211-242: LCB of every objective and constraint of a
 * multi-output model, used by GeneralBO, optimizers/general.py:65-158) ----
 * mu, var [K, m] device, output-major (row b = output b, as K single-output posterior calls with F = NULL write them),
 * K = num_obj + num_constr, 1 <= num_obj, 0 <= num_constr, K <= HB_MAX_OUTPUTS.  With py = mu, ps2 = var (per column b):
 *   ps = sqrt(ps2).clamp(min = FLT_EPSILON)         (NaN stays NaN)
 *   py = py + noise_sd[b] * xi                        only when noise_sd [K] != NULL (use_noise; noise_sd = model.noise.sqrt())
 *   Fo [m, num_obj]    = py - kappa * ps              objectives
 *   Fc [m, num_constr] = py - c_kappa * ps            constraints (may be NULL)
 *   cv [m]             = sum_j max(0, Fc[:, j])       constraint violation, fp32, columns ascending (may be NULL; a NaN
 *                                                     constraint gives cv = NaN, which the survivals treat as +inf)
 * Correctly rounded operations, no FMA contraction: each column is bit-identical to the IEEE fp32 evaluation of the
 * reference's torch expression on the same mu / var / draws.  xi [m, K] device draws (the reference's torch.randn(py.shape))
 * or NULL: Philox4x32-10 + Box-Muller keyed by (seed, counter); element q = r K + b takes half q % 2 of pair q / 2, and the
 * same (seed, counter) replays the same bits.  cv is pymoo's constraint violation as recalled from pymoo 0.6 (a sum of the
 * positive parts), not checked against pymoo; feasibility (cv <= 0 exactly when every constraint is <= 0) and the order of
 * the infeasible rows do not depend on the aggregation, so a sum and a mean give the same survivors.  One launch. */
int32_t hb_general_acq_epilogue(const float *mu, const float *var, int64_t m, int64_t num_obj, int64_t num_constr, float kappa,
                                float c_kappa, const float *noise_sd, const float *xi, uint64_t seed, uint64_t counter, float *Fo,
                                float *Fc, float *cv, void *stream);

/* ---- MOMeanSigmaLCB epilogue  (MOMeanSigmaLCB.eval, acquisitions/acq.py:99-129: minimise (py, -ps) subject to
 * LCB < best_y; the acquisition HEBO takes as acq_cls, optimizers/hebo.py:162) ----
 * mu, var [m] device, in original y units (as hb_posterior_mace_ex writes them with F = NULL), m >= 1.  noise_sd =
 * sqrt(model.noise), computed by the caller.  With py = mu, ps2 = var:
 *   py = py + noise_sd * xi
 *   ps = sqrt(ps2)                                    no clamp: a NaN or negative ps2 gives NaN, as torch.sqrt does
 *   F [m, 2] = (py, -1 * ps)                          objectives; -1 * ps is an exact negation, so ps = 0 gives -0
 *   G [m]    = (py - kappa * ps) - best_y             the constraint, feasible iff G <= 0 (a NaN G is infeasible)
 * Correctly rounded operations, no FMA contraction: each column is bit-identical to the IEEE fp32 evaluation of the
 * reference's torch expression on the same mu / var / draws.  xi [m] device draws (the reference's torch.randn(py.shape))
 * or NULL: Philox4x32-10 + Box-Muller keyed by (seed, counter); row r takes half r % 2 of pair r / 2, which is
 * hb_general_acq_epilogue's layout with K = 1, and the same (seed, counter) replays the same bits.  One launch, no host
 * synchronisation. */
int32_t hb_mo_lcb_epilogue(const float *mu, const float *var, int64_t m, float noise_sd, float best_y, float kappa,
                           const float *xi, uint64_t seed, uint64_t counter, float *F, float *G, void *stream);

/* ---- 3-objective non-dominated filter  (the rank-0 set NSGA-II returns as res.X,
 * acq_optimizers/evolution_optimizer.py:141-149) ----------------------------------------------
 * F [m,3]; idx_out [m] int32 ascending indices of the non-dominated rows; count device int32.
 * Rows with a NaN objective are excluded (they can neither dominate nor be dominated, and must never be recommended). */
int32_t hb_pareto_front3(const float *F, int64_t m, int32_t *idx_out, int32_t *count,
                         void *ws, int64_t ws_bytes, void *stream);
/* The same filter over F [m, num_obj], 1 <= num_obj <= HB_MAX_OBJ, same workspace (hb_pareto_workspace_bytes(m)) and rules;
 * hb_pareto_front3 is num_obj = 3. */
int32_t hb_pareto_front_k(const float *F, int64_t m, int64_t num_obj, int32_t *idx_out, int32_t *count,
                          void *ws, int64_t ws_bytes, void *stream);

/* ---- device NSGA-II  (acq_optimizers/evolution_optimizer.py:107-160: pymoo NSGA2 with MixedVariableMating over the MACE
 * objectives; variable typing :26-41).  The population lives on the device: X [pop, D] fp32 rows in the optimisation space
 * (d numeric columns, then D - d categorical indices), kind [D] (0 Real, 1 Integer, 2 Choice), lb / ub [D],
 * fixed [D] (NaN = free; otherwise the value of a fix_input column, :97-101).  Every call also emits the rows split into
 * the model's inputs Xc [pop, d] fp32 / Xe [pop, D - d] int32.  One generation = hb_nsga2_mate -> hb_posterior_mace_ex on
 * the offspring -> hb_nsga2_survive_ex (rank + crowding of the 2 pop merged rows, duplicates and non-finite objectives
 * never survive); nothing synchronises with the host.  Philox streams keyed by (seed, generation).
 * hb_nsga2_survive_ex: 1 <= pop <= 16384, one launch per call.  pop <= 256 runs the single-CTA kernel (ws may be NULL);
 *   larger populations run a cooperative multi-CTA kernel and need ws_bytes >= hb_nsga2_workspace_bytes(pop, D).
 *   Both give the same survivors, bit for bit, and are deterministic.
 * hb_nsga2_workspace_bytes: host only; < 0 if pop < 1, pop > 16384 or D < 1.
 * hb_nsga2_survive: the workspace-free entry, pop <= 256.
 * hb_nsga2_survive_cv: the same survival with one constraint column (pymoo's survival with infeasible filtering, as
 *   EvolutionOpt uses it with n_constr = 1: evolution_optimizer.py:82,105,135-140; the rule is recalled, not checked
 *   against pymoo).  G [pop] / GC [pop] the population's / offspring's constraint, G_next [pop] out.  A row is feasible
 *   iff G <= 0; a non-finite G and a duplicate child count as G = +inf.  With at least pop feasible merged rows only
 *   those enter the rank-and-crowding survival; otherwise every feasible row survives and the remaining slots go to the
 *   infeasible rows in ascending G, ties by the lower merged index.  Survivors keep ascending merged-row order.  Same
 *   sizes, workspace, kernels and determinism as hb_nsga2_survive_ex; G = GC = 0 gives its result, except when the cut
 *   front is the front of all-+inf rows and holds a duplicate child (which is infeasible here). */
int32_t hb_nsga2_init(float *X, int64_t pop, int64_t D, int64_t d, const int32_t *kind, const float *lb, const float *ub,
                      const float *fixed, const float *init, int64_t n_init, uint64_t seed, float *Xc, int32_t *Xe, void *stream);
int32_t hb_nsga2_mate(const float *X, int64_t pop, int64_t D, int64_t d, const int32_t *kind, const float *lb, const float *ub,
                      const float *fixed, uint64_t seed, int32_t generation, float *C, float *Cc, int32_t *Ce, void *stream);
int32_t hb_nsga2_survive(const float *X, const float *F, const float *C, const float *FC, int64_t pop, int64_t D, int64_t d,
                         float *X_next, float *F_next, float *Xc_next, int32_t *Xe_next, void *stream);
int64_t hb_nsga2_workspace_bytes(int64_t pop, int64_t D);
int32_t hb_nsga2_survive_ex(const float *X, const float *F, const float *C, const float *FC, int64_t pop, int64_t D,
                            int64_t d, float *X_next, float *F_next, float *Xc_next, int32_t *Xe_next,
                            void *ws, int64_t ws_bytes, void *stream);
int32_t hb_nsga2_survive_cv(const float *X, const float *F, const float *G, const float *C, const float *FC, const float *GC,
                            int64_t pop, int64_t D, int64_t d, float *X_next, float *F_next, float *G_next, float *Xc_next,
                            int32_t *Xe_next, void *ws, int64_t ws_bytes, void *stream);
/* hb_ga_survive: the survival of the single-objective GA (pymoo MixedVariableGA's FitnessSurvival, which EvolutionOpt runs
 *   when the acquisition has one objective: evolution_optimizer.py:123-124,132-133; the order np.lexsort([F, cv]) then
 *   pop[S[:n_survive]] is recalled from pymoo 0.6, not checked against it).  Mating is unchanged: hb_nsga2_init /
 *   hb_nsga2_mate.  F [pop] / FC [pop] one objective per merged row (population rows 0..pop-1, offspring pop..2 pop-1).
 *   A non-finite f counts as +inf; a duplicate child (the predicate of hb_nsga2_survive_ex) gets f = +inf.  The survivors
 *   are the pop merged rows first in ascending (f, merged index) order, written in that order (row 0 is the best);
 *   F_next [pop] holds their sanitised f, Xc_next / Xe_next the split rows.  Same sizes and workspace as
 *   hb_nsga2_survive_ex (ws may be NULL when pop <= 256); both kernels give the same bytes, deterministic, one launch. */
int32_t hb_ga_survive(const float *X, const float *F, const float *C, const float *FC, int64_t pop, int64_t D, int64_t d,
                      float *X_next, float *F_next, float *Xc_next, int32_t *Xe_next, void *ws, int64_t ws_bytes, void *stream);
/* hb_ga_survive_cv: the same survival with one constraint column (FitnessSurvival with constraints, np.lexsort([F, cv]),
 *   which EvolutionOpt runs for a constrained one-objective acquisition, evolution_optimizer.py:132-133; recalled from
 *   pymoo 0.6, not checked against it).  G [pop] / GC [pop]: the constraint of the population / offspring; cv = max(G, 0),
 *   a non-finite G counts as +inf, a duplicate child gets cv = f = +inf.  The survivors are the pop merged rows first in
 *   ascending (cv, f, merged index) order, best first, so row 0 is the best feasible row or, without one, the least
 *   infeasible row (pymoo's filter_optimum).  G_next [pop] out: their cv.  Same sizes, workspace and determinism as
 *   hb_ga_survive; G = GC = 0 gives its bytes except among the f = +inf rows when one of them is a duplicate child. */
int32_t hb_ga_survive_cv(const float *X, const float *F, const float *G, const float *C, const float *FC, const float *GC, int64_t pop,
                         int64_t D, int64_t d, float *X_next, float *F_next, float *G_next, float *Xc_next, int32_t *Xe_next, void *ws,
                         int64_t ws_bytes, void *stream);
/* hb_nsga2_survive_k: the rank-and-crowding survival of hb_nsga2_survive_ex / _cv over num_obj objectives,
 *   2 <= num_obj <= HB_MAX_OBJ: F / FC [pop, num_obj], F_next [pop, num_obj]; crowding adds the num_obj objectives in
 *   column order, each normalised by its own range.  G / GC / G_next all NULL: the unconstrained survival; all three given:
 *   the constrained one.  ws_bytes >= hb_nsga2_workspace_bytes_k(pop, D, num_obj) when pop > 256.  hb_nsga2_survive_ex and
 *   hb_nsga2_survive_cv are the num_obj = 3 instances (same kernels, same bytes), and hb_nsga2_workspace_bytes(pop, D) =
 *   hb_nsga2_workspace_bytes_k(pop, D, 3). */
int64_t hb_nsga2_workspace_bytes_k(int64_t pop, int64_t D, int64_t num_obj);
int32_t hb_nsga2_survive_k(const float *X, const float *F, const float *G, const float *C, const float *FC, const float *GC,
                           int64_t pop, int64_t D, int64_t d, int64_t num_obj, float *X_next, float *F_next, float *G_next,
                           float *Xc_next, int32_t *Xe_next, void *ws, int64_t ws_bytes, void *stream);

/* ---- bound violation of a random embedding  (MACE_Embedding.eval, optimizers/hebo_embedding.py:85-90, clip = False)
 * Y [m, e] candidates in the embedding, B [e, D] projection matrix, both row-major fp32 on the device; G [m] out:
 *   G[i] = sum_j max(|sum_k Y[i,k] B[k,j]| - 1, 0)   (hebo_embedding.py:88-89)
 * without forming Y B.  Each projected coordinate is an fp32 sum over k ascending; the sums over j are reduced in fp64 in
 * a fixed order (no float atomics), so G is bit-identical from run to run.  A NaN coordinate gives G = NaN (torch.clamp
 * keeps NaN), which hb_nsga2_survive_cv and the feasible front treat as +inf, i.e. infeasible.  1 <= m, 1 <= e <= HB_MAX_FEATURES, 1 <= D.
 * hb_embed_violation_workspace_bytes: host only; < 0 on bad sizes.  Two launches, no host synchronisation. */
int64_t hb_embed_violation_workspace_bytes(int64_t m, int64_t e, int64_t D);
int32_t hb_embed_violation(const float *Y, int64_t m, int64_t e, const float *B, int64_t D, float *G, void *ws,
                           int64_t ws_bytes, void *stream);

/* ---- multi-GPU front exchange  (candidate-sharded scoring, BASELINE config 5: every rank filters its shard, ONE
 * all-gather of fixed-capacity front buffers, every rank merges; no reference counterpart -- the reference is one process,
 * optimizers/hebo.py:119-194) ------------------------------------------------------------------------------------
 * Buffer layout [(capacity + 1), 8] fp32: row 0 = (count, overflow flag, 0...); row 1 + j = (F0, F1, F2, mu, sigma,
 * id_lo, id_hi, 0) with the global candidate id = id_lo + 2^24 id_hi; unused rows hold +inf objectives.
 * hb_front_pack : F [m,3], mu / var [m] (or NULL), idx / count from hb_pareto_front3, row_offset = first global id of
 *                 this shard -> out.  A front larger than `capacity` sets the overflow flag (never silently truncated).
 * hb_front_merge: all_buf [world][capacity + 1][8] (the all-gathered buffers) -> out [(world * capacity + 1), 8]: the
 *                 non-dominated rows of the union in ascending global-id order.  No host synchronisation in either call. */
int64_t hb_front_merge_workspace_bytes(int64_t world, int64_t capacity);
int32_t hb_front_pack(const float *F, const float *mu, const float *var, const int32_t *idx, const int32_t *count,
                      int64_t row_offset, int64_t capacity, float *out, void *stream);
int32_t hb_front_merge(const float *all_buf, int64_t world, int64_t capacity, float *out, void *ws, int64_t ws_bytes,
                       void *stream);

/* ---- deep-ensemble surrogate (models/nn/deep_ensemble.py: DeepEnsemble :29-181, BaseNet :183-238) -------------------
 * E members, each BaseNet: inputs [numeric (MinMax-scaled) | embedding or one-hot of each categorical column]
 * -> (Linear -> ReLU) x num_layers -> heads mu [num_out] (+ prior_net(inputs), not differentiated) and, with output_noise,
 * sigma2 = noise_lb + softplus(Linear) [num_out].  One member's raw parameters are P = hb_de_num_params(spec) floats in
 * BaseNet's registration order with torch's [out, in] weight layout, so a state_dict maps to them without permutation:
 *   enum_layer.emb.{c}.weight [u_c, min(50, 1 + u_c / 2)] (embedding only; models/layers.py:19),
 *   hidden.{2l}.weight [H, in_l], hidden.{2l}.bias [H] (l < num_layers), mu.weight [O, H], mu.bias [O],
 *   sigma2.0.weight [O, H], sigma2.0.bias [O] (output_noise), prior_net.{2l}.weight / bias, prior_net.prior_net_out.weight
 *   [O, H] / bias [O] (rand_prior).
 * Envelope (HB_ERR_INVALID outside it, hb_de_num_params / hb_de_fit_workspace_bytes return -1): */
#define HB_DE_MAX_LAYERS   3      /* num_layers                                                                      */
#define HB_DE_MAX_HIDDEN   256    /* num_hiddens                                                                     */
#define HB_DE_MAX_OUT      8      /* num_out                                                                         */
#define HB_DE_MAX_IN       256    /* input width num_cont + sum of embedding (or one-hot) widths                     */
#define HB_DE_MAX_MEMBERS  32     /* ensemble members E                                                              */
/* A fit keeps one minibatch's activations on chip: rows B = min(n, batch_size) must satisfy
 * B * (in_ld + (num_layers + 2) * hid_ld + 5 * num_out + 1) <= HB_DE_MAX_BATCH_FLOATS, with in_ld = in | 1 and
 * hid_ld = max(num_hiddens, in) | 1 (odd leading dimensions).  BaseNet's defaults (batch 32) fit with room to spare at every
 * layer / width / output count above.  The feature-gated ensemble (hb_fe_fit) adds 2 * B * in_ld to the left side; the
 * Gumbel ensemble (hb_gumbel_fit) takes in_ld and hid_ld of the SELECTED width r + enum width and adds B * (num_cont | 1)
 * for the minibatch's numeric rows when num_cont > 0. */
#define HB_DE_MAX_BATCH_FLOATS 56000

#define HB_DE_EMBEDDING    0      /* conf['enum_trans'] = 'embedding' (deep_ensemble.py:199-201) */
#define HB_DE_ONEHOT       1      /* conf['enum_trans'] = 'onehot'    (deep_ensemble.py:202-203) */

typedef struct {                  /* HOST struct */
  int32_t        num_cont;        /* numeric columns                                                   */
  int32_t        num_enum;        /* categorical columns                                               */
  const int32_t *num_uniqs;       /* HOST [num_enum] categories per column (conf['num_uniqs'])         */
  int32_t        enum_trans;      /* HB_DE_EMBEDDING | HB_DE_ONEHOT                                     */
  int32_t        num_layers;      /* conf['num_layers'] (default 1)                                    */
  int32_t        num_hiddens;     /* conf['num_hiddens'] (default 128)                                 */
  int32_t        num_out;         /* outputs                                                           */
  int32_t        output_noise;    /* conf['output_noise'] (default 1): sigma2 head and NLL loss, else MSE */
  int32_t        rand_prior;      /* conf['rand_prior'] (default 0): fixed random prior network         */
  float          noise_lb;        /* conf['noise_lb'] (default 1e-4)                                   */
} hb_de_spec_t;

/* P of one member, or -1 outside the envelope (HOST). */
int64_t hb_de_num_params(const hb_de_spec_t *spec);
/* Workspace of hb_de_fit: 3 E P floats laid out as Adam's exp_avg [E, P], exp_avg_sq [E, P] and the gradient of the last
 * step [E, P] (data term + L1 term), all readable after the call.  -1 outside the envelope (HOST). */
int64_t hb_de_fit_workspace_bytes(const hb_de_spec_t *spec, int64_t E);
/* DeepEnsemble.fit's member loop (deep_ensemble.py:81-85) and fit_one (:151-181) for all E members in ONE launch, one CTA
 * per member, with no host round trip: per epoch a permutation of the n rows, minibatches of batch_size rows (the last
 * partial batch dropped iff n > batch_size; n <= batch_size gives one batch of n rows), per step forward, the data loss
 * (NLL 0.5 (t - mu)^2 / sigma2 + 0.5 log sigma2, or MSE, over the finite entries of y), its backward, the L1 term
 * l1 sum|p| / (n num_out) over all parameters, and torch.optim.Adam (0.9, 0.999, eps 1e-8; fresh moments; lr a double as
 * torch keeps it, its bias corrections computed in double per step and rounded to fp32 where torch rounds them).
 *   Xc [n, num_cont] MinMax-scaled (NULL iff num_cont = 0), Xe [n, num_enum] int32 (NULL iff num_enum = 0), y [n, num_out]
 *   standardised (non-finite entries are masked out of the loss; every row needs one finite entry).
 *   params [E, P] in/out.  perm: NULL, or [E, num_epochs, n] int32 rows of each member's epoch in order, for tests that
 *   replay a given order; every row must be a permutation of 0..n-1, which the library does not check (the caller must:
 *   hebo_b200.DeepEnsemble.fit does).  Categories outside 0 .. num_uniqs[c] - 1 load NaN (never a read outside a table).  With perm = NULL the order is a keyed Philox bijection of (seed, member, epoch): positions are
 *   mapped through a 4-round Feistel network on 2h bits (2^(2h) >= n, round r keyed by word 0 of the Philox4x32-10 block
 *   of counter (half, epoch, member, 0x44450000 + r) under `seed`) and cycle-walked into 0..n-1.
 *   losses [E, num_epochs]: epoch_loss / n as the reference prints it (:176-179).
 * Every reduction runs in a fixed order, so the result is bit-identical from run to run.  No host synchronisation. */
int32_t hb_de_fit(const float *Xc, const int32_t *Xe, const float *y, int64_t n, const hb_de_spec_t *spec, int64_t E,
                  float *params, double lr, float l1, int64_t batch_size, int64_t num_epochs, const int32_t *perm,
                  uint64_t seed, float *losses, void *ws, int64_t ws_bytes, void *stream);
/* DeepEnsemble.predict (deep_ensemble.py:95-106) of m candidates: Xs [m, num_cont] raw inputs scaled in the load as
 * x * x_mul + x_add (the MinMax scaler's transform), Xe [m, num_enum] int32.  Members combine in index order:
 *   output_noise: py = mean(mu), ps2 = var(mu, unbiased=False) + mean(sigma2); else py = mean(mu), ps2 = 1e-8 + var(mu)
 * then py * y_std + y_mean, ps2 * y_std^2 (y_mean / y_std [num_out] device arrays).  mu / var [m, num_out].
 * member >= 0: member's own mu, un-scaled, alone (sample_f, :108-116; var may be NULL).  A category outside
 * 0 .. num_uniqs[c] - 1 gives that row NaN outputs.  No host synchronisation. */
int32_t hb_de_predict(const float *Xs, const int32_t *Xe, int64_t m, const hb_de_spec_t *spec, int64_t E,
                      const float *params, const float *x_mul, const float *x_add, const float *y_mean, const float *y_std,
                      int32_t member, float *mu, float *var, void *stream);
/* hb_de_predict (member = -1) and its input gradients dmu, dvar [m, num_out, num_cont] with respect to the raw numeric
 * inputs, through the ReLU masks of every member (prior_net's output is a constant, as under the reference's no_grad).
 * num_cont >= 1.  No host synchronisation. */
int32_t hb_de_predict_grad(const float *Xs, const int32_t *Xe, int64_t m, const hb_de_spec_t *spec, int64_t E,
                           const float *params, const float *x_mul, const float *x_add, const float *y_mean,
                           const float *y_std, float *mu, float *var, float *dmu, float *dvar, void *stream);
/* hb_de_fit for B ensembles of one spec in ONE launch (a MultiTaskModel of K single-output ensembles, model_factory.py:60-92),
 * 1 <= B <= HB_MAX_OUTPUTS, grid B E CTAs: CTA (b, member) runs hb_de_fit's member on ensemble b.  B E > 132 takes more
 * than one wave on a 132-SM H100.
 *   off HOST [B + 1] int64: ensemble b trains on rows off[b] .. off[b + 1] - 1 (n_b >= 1 of them) of the concatenated
 *   Xc [., num_cont], Xe [., num_enum] and y [., num_out], each slice filtered and scaled by its own ensemble.
 *   seeds HOST [B]: ensemble b's Philox key; the minibatch order is always the keyed bijection of hb_de_fit (no perm).
 *   params [B, E, P] in/out; losses [B, E, num_epochs]; L1 coefficient l1 / (n_b num_out) per ensemble; lr, l1,
 *   batch_size and num_epochs shared.  The minibatch of min(n_b, batch_size) rows obeys HB_DE_MAX_BATCH_FLOATS for every b.
 *   ws: ws_bytes >= B * hb_de_fit_workspace_bytes(spec, E); slice b (3 E P floats from ws + 3 b E P) is laid out as
 *   hb_de_fit's workspace.
 * Ensemble b's params, Adam moments, last gradient and losses are bit-identical to hb_de_fit on its slice alone with
 * seed seeds[b].  No host synchronisation. */
int32_t hb_de_fit_batch(const float *Xc, const int32_t *Xe, const float *y, const int64_t *off, int64_t B,
                        const hb_de_spec_t *spec, int64_t E, float *params, double lr, float l1, int64_t batch_size,
                        int64_t num_epochs, const uint64_t *seeds, float *losses, void *ws, int64_t ws_bytes, void *stream);
/* hb_de_predict (member = -1) of B ensembles of one spec over one candidate batch, 1 <= B <= HB_MAX_OUTPUTS: params
 * [B, E, P], x_mul / x_add [B, num_cont], y_mean / y_std [B, num_out].  mu / var [B num_out, m] OUTPUT-MAJOR (row
 * b num_out + o is output o of ensemble b), the layout hb_general_acq_epilogue reads; each row is bit-identical to the
 * matching column of hb_de_predict on ensemble b.
 * n_samples > 0: the same launch also writes y_samp [n_samples, m, B num_out] = py + sqrt(ps2) * xi (BaseModel.sample_y,
 * base_model.py:78-84: independent draws) with py / ps2 the mu / var above, correctly rounded fp32 without FMA
 * contraction, so bit-identical to torch's fp32 expression on the same draws.  xi [n_samples, m, B num_out] device, or
 * NULL: Philox4x32-10 + Box-Muller keyed by (seed, counter), element q (flat index of y_samp) takes half q % 2 of pair
 * q / 2 (hb_general_acq_epilogue's convention); the same (seed, counter) replays the same bits.  No host synchronisation. */
int32_t hb_de_predict_batch(const float *Xs, const int32_t *Xe, int64_t m, const hb_de_spec_t *spec, int64_t B, int64_t E,
                            const float *params, const float *x_mul, const float *x_add, const float *y_mean,
                            const float *y_std, float *mu, float *var, int64_t n_samples, const float *xi, uint64_t seed,
                            uint64_t counter, float *y_samp, void *stream);

/* ---- feature-selecting deep ensemble (models/nn/fe_deep_ensemble.py: FeNet, FeDeepEnsemble; fe_layers.py) ---------------
 * The deep ensemble above whose members multiply their input row x [din] (numeric columns, then the embedding or one-hot
 * columns) by a learned gate mask before the first hidden layer.  The prior net, when rand_prior is set, is built and takes
 * the L1 term but is not evaluated (FeNet.forward).  One member's raw parameters are P_fe = hb_fe_num_params(spec) =
 * hb_de_num_params(spec) + din floats: BaseNet's layout, then the gate's feature_select.mu (stg) or feature_select.logits
 * (concrete layers) [din] LAST, so a FeNet state_dict maps to them without permutation.  Masks of parameter theta, draw r
 * and temperature T, in IEEE fp32 without FMA contraction:
 *   HB_FE_STG            clamp((T r + theta) + 0.5, 0, 1),                     r ~ N(0, 1)
 *   HB_FE_CONCRETE       sigmoid((theta + log(u / (1 - u))) / T),              u = clamp(r, eps, 1 - eps), r ~ U(0, 1]
 *   HB_FE_HARD_CONCRETE  clamp(concrete * 1.2 + (-0.1), 0, 1)                  (stretched to [-0.1, 1.1])
 * eps = FLT_EPSILON; the clamps pass the gradient at both bounds inclusive, as torch.clamp does. */
#define HB_FE_STG            0    /* conf['fe_layer'] = 'stg' (the default)  */
#define HB_FE_CONCRETE       1    /* conf['fe_layer'] = 'concrete'           */
#define HB_FE_HARD_CONCRETE  2    /* conf['fe_layer'] = 'hard_concrete'      */

typedef struct {                  /* HOST struct */
  int32_t kind;                   /* HB_FE_*                                                                            */
  float   temperature;            /* > 0.  stg: its T in fit and predict (conf['temperature'], default 1.0).  Concrete
                                     layers: predict's T, the last epoch's of the fit's schedule (the constructor's,
                                     default 0.1, before any epoch)                                                      */
  double  start_temp;             /* concrete layers: epoch e of a fit uses T = fp32(max(start_temp anneal_base^e,      */
  double  end_temp;               /*   end_temp)), computed in double and rounded once, as torch.tensor(.).clamp(.)     */
  double  anneal_base;            /*   rounds it (defaults 1.0, 0.1, 0.99); unused by stg                               */
  float   mask_reg;               /* conf['mask_reg'] (default 0.1)                                                      */
} hb_fe_gate_t;

/* P_fe of one gated member, or -1 outside the deep ensemble's envelope (HOST). */
int64_t hb_fe_num_params(const hb_de_spec_t *spec);
/* Workspace of hb_fe_fit: 3 E P_fe floats, laid out as hb_de_fit's (Adam's exp_avg, exp_avg_sq, last gradient). */
int64_t hb_fe_fit_workspace_bytes(const hb_de_spec_t *spec, int64_t E);
/* hb_de_fit of FeDeepEnsemble (fe_deep_ensemble.py:46-75) in ONE launch, one CTA per member: hb_de_fit's minibatches,
 * data loss and Adam, with
 *   - the training mask drawn per minibatch row and input column, applied after the inputs are loaded; the backward
 *     carries the input delta through the mask into the gate (rows summed in order) and into the embedding tables;
 *   - the L1 term l1 sum|w| / (n num_out) over the WEIGHTS only (parameters whose name contains 'weight': embedding
 *     tables, hidden / heads / prior-net weights), not biases or the gate;
 *   - mask_loss = mask_reg mask_norm / (n num_out) when num_cont > 0 (none otherwise), mask_norm = sum Phi((mu + 0.5) / T)
 *     (stg) or sum sigmoid(logits) (concrete layers);
 *   - the concrete layers' temperature set at the start of every epoch (see hb_fe_gate_t).
 * The rows B = min(n, batch_size) must satisfy, on top of hb_de_fit's formula, the unmasked inputs and gate states:
 *   B * (in_ld + (num_layers + 2) * hid_ld + 5 * num_out + 1) + 2 * B * in_ld <= HB_DE_MAX_BATCH_FLOATS.
 *   params [E, P_fe] in/out; perm as hb_de_fit.  draws: NULL, or [E, num_epochs, nb, B, din] raw draws r (nb minibatches
 *   per epoch) for tests that replay given draws.  With draws = NULL, element q = ((epoch nb + step) B + row) din + column
 *   of member e's fit takes half q % 2 of the Philox4x32-10 block of counter (q / 2 as 64 bits, member, 0x46454654) under
 *   `seed` (words 0-1, 2, 3), as a Box-Muller normal (stg, hb_de_predict_batch's pair convention) or the word as a uniform
 *   (concrete layers); the minibatch order's counters end in 0x44450000 + r, so the two streams never share a block.
 * Bit-identical from run to run.  No host synchronisation. */
int32_t hb_fe_fit(const float *Xc, const int32_t *Xe, const float *y, int64_t n, const hb_de_spec_t *spec,
                  const hb_fe_gate_t *gate, int64_t E, float *params, double lr, float l1, int64_t batch_size,
                  int64_t num_epochs, const int32_t *perm, const float *draws, uint64_t seed, float *losses, void *ws,
                  int64_t ws_bytes, void *stream);
/* hb_de_predict over gated members (member = -1: the ensemble; member >= 0: sample_f's one member, var may be NULL).  Each
 * member's eval mask is one draw per input column, shared by every candidate row: draws [E, din] device raw draws, or
 * NULL: column k of member e takes half k % 2 of the Philox4x32-10 block of counter (counter as 64 bits,
 * (e << 16) | (k / 2), 0x46454556) under `seed`.  A new counter (a GA generation) gives fresh masks, as the reference
 * redraws them on every call; the same (seed, counter) replays the same bits.  No input gradients.  No host
 * synchronisation. */
int32_t hb_fe_predict(const float *Xs, const int32_t *Xe, int64_t m, const hb_de_spec_t *spec, const hb_fe_gate_t *gate,
                      int64_t E, const float *params, const float *x_mul, const float *x_add, const float *y_mean,
                      const float *y_std, int32_t member, const float *draws, uint64_t seed, uint64_t counter, float *mu,
                      float *var, void *stream);

/* ---- Gumbel feature-selection deep ensemble (models/nn/gumbel_linear.py: GumbelNet, GumbelDeepEnsemble) ----------------
 * The deep ensemble above whose members first map their num_cont numeric inputs to r = reduced_dim selected ones,
 * x_sel = x_num W^T, W [r, num_cont] = RelaxedOneHotCategorical(T, logits).rsample() (softmax over the numeric columns),
 * ONE W per forward shared by every row.  The member's input row is [x_sel | embedding or one-hot]; with num_cont = 0
 * nothing is drawn and the member is a BaseNet.  One member's raw parameters are P_gb = hb_gumbel_num_params(spec, r)
 * floats: BaseNet's layout for spec with num_cont replaced by r (when num_cont > 0), then feature_select.logits
 * [r, num_cont] LAST (GumbelNet's state_dict order).  W from logits theta, uniforms u and temperature T, in fp32:
 *   L = theta - lse(theta),  g = -log(-log(clamp(u, eps, 1 - eps))),  s = (L + g) / T,  W = exp(s - lse(s))
 * with lse(v) = log(sum exp(v - max v)) + max v over the row, eps = FLT_EPSILON, and (L + g) / T one IEEE fp32 division by
 * fp32(T), as torch divides an fp32 tensor by a Python float.
 * Envelope, on top of the deep ensemble's: num_cont <= HB_DE_MAX_IN, 1 <= r, r + embedding / one-hot width <= HB_DE_MAX_IN;
 * rand_prior needs r = num_cont or num_cont = 0 (the prior net keeps the unselected width).  The numeric rows of the
 * minibatch stay on chip next to BaseNet's buffers of the selected width (in_ld, hid_ld of r + enum width):
 *   B * (in_ld + (num_layers + 2) * hid_ld + 5 * num_out + 1) + B * (num_cont | 1) <= HB_DE_MAX_BATCH_FLOATS
 * (the last term only when num_cont > 0).  W and d loss / d W live in global memory (the fit's workspace).  Outside the
 * envelope: HB_ERR_INVALID before any launch, and -1 from the two queries. */
int64_t hb_gumbel_num_params(const hb_de_spec_t *spec, int64_t reduced_dim);
/* Workspace of hb_gumbel_fit: 3 E P_gb floats laid out as hb_de_fit's (exp_avg, exp_avg_sq, last gradient), then each
 * member's W of its last step [E, r, num_cont]. */
int64_t hb_gumbel_fit_workspace_bytes(const hb_de_spec_t *spec, int64_t reduced_dim, int64_t E);
/* GumbelDeepEnsemble.fit_one (gumbel_linear.py:69-100) for all E members in ONE launch, one CTA per member: hb_de_fit's
 * minibatch order, data loss and Adam, with
 *   - NO drop_last: ceil(n / batch_size) steps per epoch, the last one of the remaining rows; each step's loss is the mean
 *     over its own minibatch, the L1 divisor stays n num_out;
 *   - per step a fresh W from uniforms, x_sel = x_num W^T, and the backward through W, the softmax and the logits'
 *     normalisation into the logits (d loss / d W sums the minibatch rows in order);
 *   - the L1 term over the WEIGHTS only (embedding tables, hidden / heads / prior-net weights), not biases or logits;
 *   - the random prior net (rand_prior) evaluated without gradient; its weights take the L1 term, its biases do not move;
 *   - T = fp32(0.8^epoch + 0.1) (the double rounded once) throughout epoch `epoch`.
 *   perm as hb_de_fit (rows of each epoch in order).  draws: NULL, or [E, num_epochs, nb, r, num_cont] uniforms, nb the
 *   steps per epoch, for tests that replay given draws.  With draws = NULL, element q = ((epoch nb + step) r + j) num_cont
 *   + k of member e's fit takes the word q % 2 of the Philox4x32-10 block of counter (q / 2 as 64 bits, e, 0x47424654)
 *   under `seed`, as the uniform (w + 0.5) 2^-32; the minibatch order's counters end in 0x44450000 + r and the fe
 *   ensemble's in 0x4645..., so no two streams share a block.
 * Bit-identical from run to run.  No host synchronisation. */
int32_t hb_gumbel_fit(const float *Xc, const int32_t *Xe, const float *y, int64_t n, const hb_de_spec_t *spec,
                      int64_t reduced_dim, int64_t E, float *params, double lr, float l1, int64_t batch_size,
                      int64_t num_epochs, const int32_t *perm, const float *draws, uint64_t seed, float *losses, void *ws,
                      int64_t ws_bytes, void *stream);
/* hb_de_predict over GumbelNet members (member = -1: the ensemble; member >= 0: sample_f's one member, var may be NULL) at
 * temperature T = `temperature` (the last trained epoch's; 0.1 before any epoch).  Each member's W is built ONCE per call
 * into ws (ws_bytes >= 4 E r num_cont; unused when num_cont = 0) and shared by every candidate tile: draws [E, r, num_cont]
 * device uniforms, or NULL: element q = j num_cont + k of member e takes the word q % 2 of the Philox4x32-10 block of
 * counter (counter as 64 bits, (e << 16) | (q / 2), 0x47424556) under `seed`.  A new counter (a GA generation) gives a
 * fresh W, as the reference redraws it on every forward; the same (seed, counter) replays the same bits, so a call split
 * over candidate rows equals the whole call.  No input gradients.  Two launches, no host synchronisation. */
int32_t hb_gumbel_predict(const float *Xs, const int32_t *Xe, int64_t m, const hb_de_spec_t *spec, int64_t reduced_dim,
                          float temperature, int64_t E, const float *params, const float *x_mul, const float *x_add,
                          const float *y_mean, const float *y_std, int32_t member, const float *draws, uint64_t seed,
                          uint64_t counter, float *mu, float *var, void *ws, int64_t ws_bytes, void *stream);

/* ---- random-forest surrogate (models/rf/rf.py: RF :19-56 over sklearn's RandomForestRegressor defaults) ------------------
 * T regression trees per output, each exact CART (squared error, every feature, min_samples_split 2, min_samples_leaf 1,
 * unlimited depth) grown on bootstrap weights.  Tree inputs are NOT scaled: [Xc | one_hot(Xe)] (rf.py:27-35, layers.py:36),
 * width = num_cont + sum(num_uniqs); one-hot column num_cont + j is category u of column c in column-major category order
 * (c = 0 first).  Envelope (HB_ERR_INVALID before any launch outside it; the size queries return -1): */
#define HB_RF_MAX_ROWS   8192     /* training rows n                                                                 */
#define HB_RF_MAX_WIDTH  4096     /* num_cont + sum(num_uniqs) (= HB_MAX_FEATURES)                                  */
#define HB_RF_MAX_TREES  1024     /* trees per output T (conf['n_estimators'])                                       */
#define HB_RF_NAN_LEFT   (1 << 30) /* flag of an internal node's feature word: NaN inputs go left (missing_go_to_left)    */
/* and 1 <= B <= HB_MAX_OUTPUTS outputs per fit.
 *
 * Forest (device bytes, hb_rf_forest_bytes): a 256-byte header {cap, B, T, woh, num_enum, 0, 0, 0} (int32; cap = node
 * capacity per tree), then, each block 256-byte aligned: the decode tables int32 [num_enum] (categories per column) and
 * [woh] ((c << 12) | u of one-hot column j); node counts int32 [B, T]; nodes int4 [B, T, cap]; thresholds double
 * [B, T, cap]; node values double [B, T, cap].  Tree (b, t) is entry b T + t.  A node replaces one entry of sklearn's
 * tree_ arrays (_tree.pyx): internal {feature | HB_RF_NAN_LEFT if missing_go_to_left, RD32(threshold) as fp32 bits, left,
 * right}, leaf
 * {-2, 0, value as the low and high words of its double}; the thresholds hold sklearn's fp64 threshold (-2 for a leaf) and the values
 * tree_.value = sum(w y) / sum(w) of every node.  For fp32 x, x <= t exactly when x <= RD32(t) (t rounded toward -inf), so
 * the fp32 traversal takes the fp64 decision of DecisionTreeRegressor.predict.  A NaN input goes left exactly where
 * missing_go_to_left is set; sklearn sets it, for trees trained without NaN, where the split leaves more distinct in-bag
 * rows left than right, and a fit here sets it so.  +inf goes right and -inf left, as any comparison takes them.  A
 * fitted tree is numbered breadth first:
 * the split nodes of a level, in index order, append their left then right child. */
typedef struct {                  /* HOST struct */
  int32_t        num_cont;        /* numeric columns                                                   */
  int32_t        num_enum;        /* categorical columns                                               */
  const int32_t *num_uniqs;       /* HOST [num_enum] categories per column (conf['num_uniqs'])         */
} hb_rf_spec_t;

/* Workspace of hb_rf_fit (HOST). */
int64_t hb_rf_fit_workspace_bytes(int64_t n, const hb_rf_spec_t *spec, int64_t B, int64_t T);
/* Bytes of a forest of B outputs x T trees with max_nodes node slots per tree (a fit of n rows: max_nodes = 2 n - 1)
 * (HOST). */
int64_t hb_rf_forest_bytes(const hb_rf_spec_t *spec, int64_t max_nodes, int64_t B, int64_t T);
/* RF.fit (rf.py:37-43) of B outputs over one X, every tree of every output in one grow launch.
 *   Xc [n, num_cont] fp32 (finite), Xe [n, num_enum] int32 in range, y [n, B] fp32: output b uses the rows with finite
 *   y[:, b] (filter_nan(..., 'all') per column).
 *   counts: NULL, or [B, T, n] int32 bootstrap counts (rows with non-finite y and negative counts weigh 0).  With NULL,
 *   tree (b, t) draws n_b = #finite rows indices with replacement from output b's finite rows in row order: draw j is
 *   row kept[umulhi(word j % 4 of Philox4x32-10 block (j / 4, t, b, 0x52460000) under `seed`, n_b)].
 *   Growth: a node with fewer than 2 distinct in-bag rows, or impurity sum(w y^2)/W - (sum(w y)/W)^2 <= DBL_EPSILON, is a
 *   leaf.  Each feature's in-bag rows are taken in the stable (value, row) order; a cut lies between sorted values
 *   v[p-1] < v[p] with v[p] > v[p-1] + 1e-7 (fp64); the split maximises S_L^2/W_L + S_R^2/W_R (fp64), ties to the lowest
 *   feature, then the lowest cut; threshold v[p-1]/2 + v[p]/2, or v[p-1] when that equals v[p] or is infinite; rows with
 *   x <= threshold go left.  No feature with a cut: leaf.  Sums: the root's in row order; a node's left prefix
 *   sums W_L, S_L = sum(w y), Q_L = sum((w y) y) sequentially in that sorted order; a child's totals are the split's left
 *   sums and total - left for the right child.  Leaf value S / W.
 *   forest: hb_rf_forest_bytes(spec, 2 n - 1, B, T) bytes; noise [B] fp32: est_noise = fp32(np.mean((forest mean -
 *   y)^2)) over output b's finite rows, with the forest mean summed sequentially in tree order over fp64 leaf values, / T,
 *   and numpy's pairwise sum.  Bit-identical from run to run.  Copies the spec's tables from the host and synchronises
 *   the stream once before the launches. */
int32_t hb_rf_fit(const float *Xc, const int32_t *Xe, const float *y, int64_t n, const hb_rf_spec_t *spec, int64_t B,
                  int64_t T, const int32_t *counts, uint64_t seed, void *forest, float *noise, void *ws, int64_t ws_bytes,
                  void *stream);
/* RF.predict (rf.py:49-56) of m candidates over a forest of B outputs x T trees: mean / var [m, B] with
 *   mean = fp32(sum_t v_t / T), the sum sequential in tree order (RandomForestRegressor.predict);
 *   var = fp32(np.var(v)) + noise[b] in fp32, np.var's mean and squared deviations both summed pairwise as numpy does.
 * Bit-identical to the reference's fp32 outputs for the same trees.  A category outside 0 .. num_uniqs[c] - 1, or a forest
 * whose header disagrees with (B, T, num_enum), gives NaN outputs.  n_samples > 0: samples [n_samples, m, B] =
 * mean + sqrt(var) * xi, correctly rounded fp32, xi Philox4x32-10 + Box-Muller keyed by (seed, counter), element q (flat
 * index of samples) takes half q % 2 of pair q / 2.  No host synchronisation. */
int32_t hb_rf_predict(const float *Xc, const int32_t *Xe, int64_t m, const hb_rf_spec_t *spec, const void *forest,
                      int64_t B, int64_t T, const float *noise, float *mean, float *var, int64_t n_samples, uint64_t seed,
                      uint64_t counter, float *samples, void *stream);
/* A one-output forest (B = 1) of T trees from device arrays [T, max_nodes] in sklearn's tree_ layout: children_left,
 * children_right (-1 at a leaf), feature, threshold (fp64), value (fp64); node_counts [T] device int32.  An internal
 * node's feature may carry HB_RF_NAN_LEFT (sklearn's tree_.missing_go_to_left): NaN inputs go left there, right at every
 * node without it.  For scoring a forest grown elsewhere.  Synchronises the stream once (header copy). */
int32_t hb_rf_load(const int32_t *left, const int32_t *right, const int32_t *feature, const double *threshold,
                   const double *value, const int32_t *node_counts, const hb_rf_spec_t *spec, int64_t T,
                   int64_t max_nodes, void *forest, void *stream);

/* ---- Monte-Carlo expected hypervolume improvement  (GeneralBO's ref_point selection, optimizers/general.py:116-140) ----
 * One selection round, bit for bit with the host's exact hypervolume (hebo_b200.general.hypervolume, minimisation):
 *   base_hv  = hypervolume(front, ref)
 *   ehvi[j]  = (sum_k (hypervolume(vstack([front, samples[k, j]]), ref) - base_hv)) / n_mc,  the sum from 0.0, k ascending
 * front [n, K], samples [n_mc, m, K], ref [K], base_hv [1], ehvi [m]: fp64 on the device.  A hypervolume keeps the rows
 * strictly below ref in every coordinate (NaN rows drop out), sorts them stably by the last coordinate (a sample after the
 * front rows it ties), and adds, over the slices with hi > y in ascending order, hv(nondominated(prefix[:, :-1]),
 * ref[:-1]) * (hi - y) with base case ref[0] - min; every operation is one rounded fp64 operation (no FMA), so +-inf
 * samples take the host's IEEE path.  Cost is exponential in K, as on the host.  2 <= K <= HB_MAX_OBJ, 0 <= n < 2^31 - 2,
 * m >= 0, n_mc >= 1; front may be NULL when n == 0.  m == 0 launches nothing and leaves base_hv unwritten.
 * hb_ehvi_workspace_bytes: host only, < 0 on bad sizes; non-decreasing in every argument.  No host synchronisation. */
int64_t hb_ehvi_workspace_bytes(int64_t n, int64_t K, int64_t m, int64_t n_mc);
int32_t hb_ehvi(const double *front, int64_t n, int64_t K, const double *samples, int64_t m, int64_t n_mc, const double *ref,
                double *base_hv, double *ehvi, void *ws, int64_t ws_bytes, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* HEBO_B200_H */
