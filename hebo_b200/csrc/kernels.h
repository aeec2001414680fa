// Internal launcher declarations (C++ linkage); the C ABI lives in api.cu / include/hebo_b200.h.
#pragma once
#include <cuda_fp16.h>
#include "common.cuh"

namespace hb {

// hi/lo (3xTF32) companion buffers of the fit's tensor-core path (fit_tc.cu); all [NP, NP] except P [NP, 512]
struct TcBuffers {
  float *L_hi, *L_lo, *Linv_hi, *Linv_lo, *U_hi, *U_lo, *T_hi, *T_lo, *P_hi, *P_lo;
};

// Parameter layout of the (optionally mixed numeric + categorical) exact GP, in the reference's registration order
// (likelihood.raw_noise, embedding tables, mean constant, raw_outputscale, numeric raw_lengthscale[s], embedding
// raw_lengthscale: HEBO/hebo/models/gp/gp.py:86-103, gp_util.py:22-59, layers.py:14-34).  With e == 0 and ard == 1 this is
// the numeric-only layout raw = (noise, mean, outputscale, lengthscale[d]).
//   raw : [P]  P = 3 + T + 2 d [warp] + n_ls + (e > 0):  noise, tables, warp a / b (feature-extractor parameters), mean,
//              outputscale, numeric lengthscale(s), embedding lengthscale
//   hyp : [H]  H = 3 + d + (e > 0) + 2 d [warp]:  sigma_n^2, c, s, lengthscale per numeric dim (expanded when ard == 0),
//              emb lengthscale, Kumaraswamy exponents a[d], b[d]
struct ModelSpec {
  int d = 0;      // numeric dims (0 allowed when e > 0)
  int ard = 1;    // conf['ard_kernel'] (gp.py:47)
  int e = 0;      // categorical columns
  int De = 0;     // total embedding width  sum_c emb_size_c
  int T = 0;      // total table entries    sum_c num_uniq_c * emb_size_c
  int warp = 0;   // Kumaraswamy input warp of the numeric dims: 0 none, 1 learned exponents a, b (2 d parameters), 2 frozen
  // device int32 arrays living in the fit workspace (nullptr when e == 0)
  const int32_t *q_col = nullptr, *q_loc = nullptr;               // [De] categorical column / coordinate inside it
  const int32_t *tab_off = nullptr, *emb_size = nullptr;          // [e]  offset of table c inside the T block, its width
  const int32_t *ent_col = nullptr, *ent_u = nullptr, *ent_q = nullptr;   // [T] (column, category, coordinate) of entry t
  const int32_t *Xe = nullptr;                                    // [n, e] training categories
  __host__ __device__ int n_ls() const { return d == 0 ? 0 : (ard ? d : 1); }
  __host__ __device__ int i_tab() const { return 1; }
  __host__ __device__ int n_w() const { return warp ? 2 * d : 0; }       // raw warp parameters (a[d], b[d]) after the tables
  __host__ __device__ int i_wa() const { return 1 + T; }
  __host__ __device__ int i_wb() const { return 1 + T + d; }
  __host__ __device__ int i_mean() const { return 1 + T + n_w(); }
  __host__ __device__ int i_os() const { return 2 + T + n_w(); }
  __host__ __device__ int i_ls() const { return 3 + T + n_w(); }
  __host__ __device__ int i_le() const { return 3 + T + n_w() + n_ls(); }
  __host__ __device__ int P() const { return 3 + T + n_w() + n_ls() + (e > 0 ? 1 : 0); }
  __host__ __device__ int h_wa() const { return 3 + d + (e > 0 ? 1 : 0); }        // hyp: a[d], b[d] after the lengthscales
  __host__ __device__ int h_wb() const { return h_wa() + d; }
  __host__ __device__ int H() const { return 3 + d + (e > 0 ? 1 : 0) + n_w(); }
  __host__ __device__ int dtot() const { return d + De; }
};

// What candidate scoring reads of a fitted GP (GP.state_tensors() on the Python side), validated and bound once per entry
// point (open_fitted, api.cu).  The launchers take it whole; kernels keep their __restrict__ pointer lists, unpacked where
// the <<<...>>> is written.
struct Fitted {
  ModelSpec sp;                 // layout arrays bound (bind_meta)
  int64_t n, np;                // training rows, np = round_up(n, TILE)
  int kern;
  const float *Zt, *alpha, *Linv, *hyp, *tab_s, *x_mul, *x_add;
  float y_mean, y_std;
  int pred_likeli;
};

// Consecutive float blocks of a workspace.  With base == nullptr it only counts, which is how a size query runs the same
// carve as its launcher.
struct Carver {
  float *base;
  int64_t used = 0;
  float *take(int64_t count) {
    used += count;
    return base ? base + used - count : nullptr;
  }
};

// ---- output dimension of the fit-loop kernels (DESIGN §3).  A batch of `nout` outputs that share one training set is
// `nout` consecutive single-output workspaces `ws` bytes apart; output b reads its raw row at raw + b * P and its targets at
// y + b * n, and shares the training inputs Xt / Xe.  Element-wise and tile kernels take b from blockIdx.z, the persistent
// and cooperative ones from their work item.  nout = 1 is the single-output fit.
struct Batch {
  int nout = 1;
  int64_t ws = 0;   // workspace slice stride in bytes (256-byte aligned)
};
template <class T>
__host__ __device__ __forceinline__ T *slice(T *p, int64_t stride_bytes, int b) {
  return p ? reinterpret_cast<T *>(reinterpret_cast<uintptr_t>(p) + (uintptr_t)(stride_bytes * b)) : p;
}
// memset of `bytes` at p in every slice of the batch
inline cudaError_t memset_slices(void *p, int value, size_t bytes, const Batch &bt, cudaStream_t st) {
  if (bt.nout == 1) return cudaMemsetAsync(p, value, bytes, st);
  return cudaMemset2DAsync(p, (size_t)bt.ws, value, bytes, (size_t)bt.nout, st);
}

// ---- candidate feature map (DESIGN §5).  Every kernel that scales candidate rows goes through these two functions, and
// the training rows take the same operations in the same order (scale_zt_kernel, emb_gather_kernel), so that a candidate
// duplicating a training row has r = 0 exactly.
// Index into the embedding tables of embedding coordinate q of row `row` of the categories Xe [rows, e]
// (EmbTransform.forward, layers.py:33-34).
__device__ __forceinline__ int emb_entry(const ModelSpec &sp, const int32_t *Xe, int64_t row, int q) {
  const int c = sp.q_col[q];
  return sp.tab_off[c] + Xe[row * sp.e + c] * sp.emb_size[c] + sp.q_loc[q];
}
// Numeric coordinate k of a candidate x_k: MinMax scale (TorchMinMaxScaler.transform, scalers.py:86-87), the Kumaraswamy
// warp when `warp`, then the reciprocal of the lengthscale times the result.
__device__ __forceinline__ float cand_feature(const ModelSpec &sp, bool warp, float x, int k, const float *x_mul,
                                              const float *x_add, const float *hyp) {
  float xt = __fadd_rn(__fmul_rn(x_mul[k], x), x_add[k]);
  if (warp) xt = kumar_warp(xt, hyp[sp.h_wa() + k], hyp[sp.h_wb() + k]);
  const float *ls = hyp + 3;
  return xt * (1.0f / ls[k]);
}

// cholesky.cu / linalg.cu   (tc: outer update on the tensor cores, the gradient epochs; nullptr -> FP32 SIMT)
int launch_cholesky(float *A, int64_t np, float *ws, int32_t *info, cudaStream_t st, const TcBuffers *tc = nullptr,
                    const Batch &bt = Batch());
int launch_triinv_base2(const float *L, int64_t np, float *Linv, float *Linv_hi, float *Linv_lo, float *U_hi, float *U_lo,
                        cudaStream_t st, const Batch &bt = Batch());
// fit_tc.cu
int launch_chol_outer_update_tc(float *A, int64_t np, int64_t cb, int64_t ce, const TcBuffers &tc, cudaStream_t st,
                                const Batch &bt);
int launch_tri_inverse_tc(const float *L, int64_t np, float *Linv, const TcBuffers &tc, bool zero_fill, cudaStream_t st,
                          const Batch &bt);
int launch_kinv_tc(int64_t np, float *Kinv, const TcBuffers &tc, cudaStream_t st, const Batch &bt);
int launch_tri_inverse(const float *L, int64_t np, float *Linv, float *tmp, cudaStream_t st);
int launch_kinv(const float *Linv, int64_t np, float *Kinv, cudaStream_t st);
int launch_linv_refine(float *L, float *Linv, int64_t np, float *R, float *out, cudaStream_t st);
int launch_solve_logdet(const float *L, const float *Linv, const float *y, int64_t n, int64_t np,
                        const float *hyp, float *alpha, double *scal, void *ws, cudaStream_t st, const Batch &bt = Batch());
size_t solve_ws_bytes(int64_t np);

// pairwise.cu
int launch_transform_hypers(const float *raw, const ModelSpec &sp, float noise_lb, float *hyp, cudaStream_t st,
                            const Batch &bt = Batch());
int launch_gram(const float *Xt, const float *Ets, int64_t n, int64_t np, const ModelSpec &sp, const float *hyp, int kern,
                const float *noise_diag, float jitter, float *K, cudaStream_t st, const Batch &bt = Batch());
int launch_mll_grad(const float *Xt, const float *Ets, int64_t n, int64_t np, const ModelSpec &sp, const float *raw,
                    const float *hyp, int kern, const float *Kinv, const float *alpha, const double *scal, float noise_guess,
                    float *grad, float *loss, void *ws, cudaStream_t st, const float *dZa = nullptr, const float *dZb = nullptr,
                    const Batch &bt = Batch());
size_t grad_ws_bytes(int64_t np, const ModelSpec &sp);
int launch_emb_gather(const float *tables, const ModelSpec &sp, int64_t n, int64_t np, const float *hyp, float *Ets, float *tab_s,
                      cudaStream_t st, const Batch &bt = Batch());
int launch_psgld(float *raw, const float *grad, float *sq, int64_t p, float lr, float a, float eps,
                 float factor, const float *xi, cudaStream_t st);
int launch_scale_zt(const float *Xt, int64_t np, const ModelSpec &sp, const float *hyp, float *Zt, float *dZa, float *dZb,
                    cudaStream_t st, const Batch &bt = Batch());

// init.cu
int launch_median_pdist(const float *Xt, int64_t np, int64_t d, const int32_t *idx, int64_t k, float clamp_min,
                        float *out, cudaStream_t st);

// posterior.cu
int launch_posterior_mace(const Fitted &gp, const float *Xs, const int32_t *Xe_s, int64_t m, int64_t rng_offset,
                          const float *Linv_hi, const float *Linv_lo, float tau, float kappa, float eps, const float *xi1,
                          const float *xi2, uint64_t seed, float *F, float *mu, float *var, void *ws, int64_t ws_bytes,
                          int64_t m_chunk, cudaStream_t st);
// The posterior workspace of one chunk of at most m_chunk candidates, rows padded to mc_pad = round_up(m_chunk, CHUNK_ROWS).
// KS: fp32 K* rows (SIMT and guard passes); KS2[b]: the fp16 two-level split h0 | h1 of the tensor path, or (KS2[0]) the V
// panel of the gradient path, which then overwrites KS with W; mupart[b] [groups, mc_pad]; vpart / vfix [np / GT, mc_pad];
// the guard lists.  KS2 and mupart come twice so that the tensor path can build the K* of chunk i + 1 into one buffer while
// chunk i is still contracted from the other (launch_posterior_mace).
struct PostWs {
  float *KS, *KS2[2], *mupart[2], *vpart, *vfix;
  int32_t *fixmap, *fixlist, *fixcount;
  int64_t mc_pad;
  size_t bytes;
};
PostWs carve_posterior_ws(void *ws, int64_t np, int64_t m_chunk);   // ws == nullptr: only .bytes, the size query
int guard_stats(unsigned long long *out, int reset);
int launch_mace_only(const float *mu, const float *var, int64_t m, float noise_var, float tau, float kappa, float eps,
                     const float *xi1, const float *xi2, uint64_t seed, float *F, cudaStream_t st);
// f[m] of a single-objective acquisition (mode HB_ACQ1_*) over (mu, var)
int launch_acq1(const float *mu, const float *var, int64_t m, int mode, float kappa, float eta, float *f, cudaStream_t st);
int launch_general_acq(const float *mu, const float *var, int64_t m, int64_t num_obj, int64_t num_constr, float kappa,
                       float c_kappa, const float *noise_sd, const float *xi, uint64_t seed, uint64_t counter, float *Fo,
                       float *Fc, float *cv, cudaStream_t st);
// F [m, 2] and G [m] of MOMeanSigmaLCB over (mu, var)
int launch_mo_lcb(const float *mu, const float *var, int64_t m, float noise_sd, float best_y, float kappa, const float *xi,
                  uint64_t seed, uint64_t counter, float *F, float *G, cudaStream_t st);
int kstar_groups(int64_t np);
int launch_kstar(const Fitted &gp, const float *xs, const int32_t *xe, int64_t mc, float *KS, float *KS_h16, float *mupart,
                 int64_t mc_pad, const int32_t *fixlist, const int32_t *fixcount, cudaStream_t st);

// posterior_grad.cu
int launch_posterior_grad(const Fitted &gp, const float *Xs, const int32_t *Xe_s, int64_t m, float *mu, float *var, float *dmu,
                          float *dvar, void *ws, int64_t ws_bytes, int64_t m_chunk, cudaStream_t st);

// fp16 two-level split tensor path of the posterior (vnorm_h16.cu: wgmma / TMA / mbarrier)
int launch_split_h16(const float *x, int64_t count, __half *h0, __half *h1, float *scale_slot, cudaStream_t st);
int launch_vnorm_h16(const __half *ks_h0, const __half *ks_h1, int64_t ks_rows, const __half *linv_h0, const __half *linv_h1,
                     const float *scale_b, const float *hyp, int64_t np, int64_t mc_pad, int64_t vpart_stride, float *vpart,
                     cudaStream_t st);

// pareto.cu
int launch_pareto_k(const float *F, int64_t m, int64_t K, int32_t *idx_out, int32_t *count, void *ws, int64_t ws_bytes,
                    cudaStream_t st);
size_t pareto_ws_bytes(int64_t m);
int launch_front_pack(const float *F, const float *mu, const float *var, const int32_t *idx, const int32_t *count,
                      int64_t row_offset, int64_t capacity, float *out, cudaStream_t st);
size_t front_merge_ws_bytes(int64_t world, int64_t capacity);
int launch_front_merge(const float *all, int64_t world, int64_t capacity, float *out, void *ws, int64_t ws_bytes,
                       cudaStream_t st);

size_t sample_ws_bytes(int64_t np, int64_t dtot, int64_t m);
int launch_sample_y(const Fitted &gp, const float *Xs, const int32_t *Xe_s, int64_t m, const float *hyp_host, const float *z,
                    int n_samples, float *out, float *jitter_used, void *ws, int64_t ws_bytes, cudaStream_t st);
// one joint draw f [m] over m <= 256 rows, duplicates dropped, jitter ladder on the device (hb_sample_y_batch)
int launch_sample_y_batch(const Fitted &gp, const float *Xs, const int32_t *Xe_s, int64_t m, const float *z, uint64_t seed,
                          uint64_t counter, float *f, float *jitter_out, int32_t *status, void *ws, int64_t ws_bytes,
                          cudaStream_t st);
// nsga.cu
int launch_nsga_init(float *X, int64_t P, int64_t D, int64_t d, const int32_t *kind, const float *lb, const float *ub,
                     const float *fixed, const float *init, int64_t n_init, uint64_t seed, float *Xc, int32_t *Xe, cudaStream_t st);
int launch_nsga_mate(const float *X, int64_t P, int64_t D, int64_t d, const int32_t *kind, const float *lb, const float *ub,
                     const float *fixed, uint64_t seed, int gen, float *C, float *Cc, int32_t *Ce, cudaStream_t st);
// survival of the 2P merged rows with K objectives (2 <= K <= HB_MAX_OBJ): one CTA for 2P <= 512 (ws may be NULL), the
// cooperative multi-CTA kernel up to P = 16384 (ws_bytes >= nsga_survive_ws_query(P, D, K)).  G / GC / Gn: constraint of
// the population / offspring / survivors (all three NULL: unconstrained).
int64_t nsga_survive_ws_query(int64_t P, int64_t D, int64_t K);
int launch_nsga_survive(const float *X, const float *F, const float *G, const float *C, const float *FC, const float *GC,
                        int64_t P, int64_t D, int64_t d, int64_t K, float *Xn, float *Fn, float *Gn, float *Xcn, int32_t *Xen,
                        void *ws, int64_t ws_bytes, cudaStream_t st);
// single-objective survival: the P best merged rows by (f, index) -- (cv, f, index) with G / GC / Gn -- best first; the
// workspace of the K = 3 survival
int launch_ga_survive(const float *X, const float *F, const float *G, const float *C, const float *FC, const float *GC, int64_t P,
                      int64_t D, int64_t d, float *Xn, float *Fn, float *Gn, float *Xcn, int32_t *Xen, void *ws, int64_t ws_bytes,
                      cudaStream_t st);
// embed.cu: G[i] = sum_j max(|sum_k Y[i,k] B[k,j]| - 1, 0)
int64_t embed_violation_ws_query(int64_t m, int64_t e, int64_t D);
int launch_embed_violation(const float *Y, int64_t m, int64_t e, const float *B, int64_t D, float *G, void *ws, int64_t ws_bytes,
                           cudaStream_t st);
// ensemble.cu: the deep ensembles' fit (one CTA per member) and predict / input gradients (dmu == nullptr: none).  The
// variant: DeepEnsemble's BaseNet members (DeVariant{}), FeDeepEnsemble's gated ones (GATED, the gate) or
// GumbelDeepEnsemble's (GUMBEL, r = reduced_dim and T = predict's temperature); draws, seed / counter and ws are the
// selection layer's (NULL / 0 for BaseNet)
struct DeVariant {
  enum Kind { BASE, GATED, GUMBEL } kind;
  const hb_fe_gate_t *gate;
  int64_t r;
  float T;
};
int64_t de_num_params(const hb_de_spec_t *spec, const DeVariant &v);
int64_t de_fit_ws_query(const hb_de_spec_t *spec, const DeVariant &v, int64_t E);
int launch_de_fit(const float *Xc, const int32_t *Xe, const float *y, int64_t n, const hb_de_spec_t *spec, const DeVariant &v,
                  int64_t E, float *params, double lr, float l1, int64_t batch_size, int64_t num_epochs, const int32_t *perm,
                  const float *draws, uint64_t seed, float *losses, void *ws, int64_t ws_bytes, cudaStream_t st);
int launch_de_predict(const float *Xs, const int32_t *Xe, int64_t m, const hb_de_spec_t *spec, const DeVariant &v, int64_t E,
                      const float *params, const float *x_mul, const float *x_add, const float *y_mean, const float *y_std,
                      int32_t member, const float *draws, uint64_t seed, uint64_t counter, float *mu, float *var,
                      float *dmu, float *dvar, void *ws, int64_t ws_bytes, cudaStream_t st);
// nens ensembles of one spec: the fit (one CTA per (ensemble, member)) and predict (mu / var output-major, optional draws)
int launch_de_fit_batch(const float *Xc, const int32_t *Xe, const float *y, const int64_t *off, int64_t nens,
                        const hb_de_spec_t *spec, int64_t E, float *params, double lr, float l1, int64_t batch_size,
                        int64_t num_epochs, const uint64_t *seeds, float *losses, void *ws, int64_t ws_bytes, cudaStream_t st);
int launch_de_predict_batch(const float *Xs, const int32_t *Xe, int64_t m, const hb_de_spec_t *spec, int64_t nens, int64_t E,
                            const float *params, const float *x_mul, const float *x_add, const float *y_mean,
                            const float *y_std, float *mu, float *var, int64_t n_samples, const float *xi, uint64_t seed,
                            uint64_t counter, float *y_samp, cudaStream_t st);

// hypervolume.cu: GeneralBO's Monte-Carlo EHVI selection round, bit for bit with general.hypervolume
int64_t ehvi_ws_query(int64_t n, int64_t K, int64_t m, int64_t n_mc);
int launch_ehvi(const double *front, int64_t n, int64_t K, const double *samples, int64_t m, int64_t n_mc, const double *ref,
                double *base_hv, double *ehvi, void *ws, int64_t ws_bytes, cudaStream_t st);
// random-forest surrogate (forest.cu)
int64_t rf_forest_bytes(const hb_rf_spec_t *spec, int64_t max_nodes, int64_t B, int64_t T);
int64_t rf_fit_ws_query(int64_t n, const hb_rf_spec_t *spec, int64_t B, int64_t T);
int launch_rf_fit(const float *Xc, const int32_t *Xe, const float *y, int64_t n, const hb_rf_spec_t *spec, int64_t B,
                  int64_t T, const int32_t *counts, uint64_t seed, void *forest, float *noise, void *ws, int64_t ws_bytes,
                  cudaStream_t st);
int launch_rf_predict(const float *Xc, const int32_t *Xe, int64_t m, const hb_rf_spec_t *spec, const void *forest,
                      int64_t B, int64_t T, const float *noise, float *mean, float *var, int64_t n_samples, uint64_t seed,
                      uint64_t counter, float *samples, cudaStream_t st);
int launch_rf_load(const int32_t *left, const int32_t *right, const int32_t *feature, const double *thr,
                   const double *value, const int32_t *node_counts, const hb_rf_spec_t *spec, int64_t T, int64_t max_nodes,
                   void *forest, cudaStream_t st);

}  // namespace hb
