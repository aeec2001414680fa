// Posterior mean / variance WITH their gradients w.r.t. the candidates -- the `support_grad` contract of the reference
// model (HEBO/hebo/models/base_model.py:27-29, test/test_base_model.py:94-108: predict() must be differentiable in Xc),
// which gpytorch provides through autograd (HEBO/hebo/models/gp/gp.py:137-164).  Closed form, FP32 SIMT:
//
//   k*_i   = s phi(r_i^2),  r_i^2 = sum_k (z*_k - z_ik)^2,  z = (x_mul x + x_add) / l          (kstar_kernel)
//   V      = K* Linv^T      (v = L^-1 k*),     W = V Linv   (w = K^-1 k*)                      (rows_gemm_kernel x 2)
//   mu~    = c + k*.alpha ;  sigma~^2 = s - |v|^2
//   d k*_i / d x_k    = -s h_i (z*_k - z_ik) x_mul_k / l_k         (h: kern_eval_grad, phi' = -h/2)
//   d mu~ / d x_k     =      sum_i alpha_i dk*_i/dx_k
//   d sigma~^2 / d x_k = -2  sum_i w_i     dk*_i/dx_k                                            (post_grad_kernel)
// followed by the same floors / un-scaling as the value path (the gradient of a clamped variance is zero, as autograd's).
// Meant for gradient-based acquisition refinement on small batches; the throughput path is posterior.cu.
#include "gemm_core.cuh"
#include "kernels.h"

namespace hb {

// C[rt, J] (128 x 128 tiles, row-major ld) = sum_{k in [kbeg(J), kend(J))} A[row][k] * Bop(col, k)
//   MODE 0:  V = KS Linv^T : Bop(c, k) = Linv[c][k] (K-major), k in [0, (J+1) 128)
//   MODE 1:  W = V  Linv   : Bop(c, k) = Linv[k][c],           k in [J 128, np)
template <int MODE>
__global__ void __launch_bounds__(GTHREADS, 2) rows_gemm_kernel(const float *__restrict__ A, const float *__restrict__ Linv,
                                                                int64_t np, float *__restrict__ C) {
  __shared__ GemmSmem sm;
  const int J = blockIdx.x;
  const int64_t rt = blockIdx.y;
  float acc[8][8];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[i][j] = 0.0f;
  if (MODE == 0)
    gemm_mainloop<true, true>(A + rt * GT * np, np, Linv + (int64_t)J * GT * np, np, 0, (J + 1) * GT, acc, sm);
  else
    gemm_mainloop<true, false>(A + rt * GT * np, np, Linv + (int64_t)J * GT, np, J * GT, (int)np, acc, sm);
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int jh = 0; jh < 2; ++jh)
      *reinterpret_cast<float4 *>(C + (rt * GT + gemm_row(i)) * np + (int64_t)J * GT + gemm_col(jh * 4)) =
          make_float4(acc[i][jh * 4 + 0], acc[i][jh * 4 + 1], acc[i][jh * 4 + 2], acc[i][jh * 4 + 3]);
}

// one CTA per candidate.  V row / W row are overwritten by the per-training-point coefficients of the two sums.
// EMB (mixed model): k* carries the extra factor Matern32(r over the embedding rows); gradients are w.r.t. the numeric
// inputs only (the categories are not differentiable).
template <int KERN, bool EMB>
__global__ void __launch_bounds__(256) post_grad_kernel(const float *__restrict__ Xs, int d, const float *__restrict__ x_mul,
                                                        const float *__restrict__ x_add, const float *__restrict__ Zt,
                                                        const float *__restrict__ alpha, const float *__restrict__ hyp,
                                                        int64_t n, int64_t np, float *__restrict__ V, float *__restrict__ W,
                                                        const float *__restrict__ mupart, int ncg, int64_t mc_pad,
                                                        int64_t row_offset, float y_mean, float y_std, int pred_likeli,
                                                        float *__restrict__ mu_out, float *__restrict__ var_out,
                                                        float *__restrict__ dmu, float *__restrict__ dvar,
                                                        const int32_t *__restrict__ Xe_s, const float *__restrict__ tab_s,
                                                        ModelSpec sp) {
  extern __shared__ float zs[];   // [d] scaled candidate, [d] x_mul / l, [De] scaled embedding features
  __shared__ float red[8];
  __shared__ float s_vsq;
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
  const int64_t r = blockIdx.x;                 // row inside the chunk
  const int64_t gr = row_offset + r;            // global candidate index
  // no warp here: the caller applies it in front of this kernel, so that the Jacobian row is x_mul / l
  const float *ls = hyp + 3;
  for (int k = t; k < d; k += 256) {
    zs[k] = cand_feature(sp, false, Xs[gr * d + k], k, x_mul, x_add, hyp);
    zs[d + k] = x_mul[k] * (1.0f / ls[k]);
  }
  const int De = EMB ? sp.De : 0;
  if (EMB) {
    for (int q = t; q < De; q += 256) zs[2 * d + q] = tab_s[emb_entry(sp, Xe_s, gr, q)];
  }
  float *v = V + r * np, *w = W + r * np;
  // |v|^2
  float p = 0.0f;
  for (int64_t i = t; i < n; i += 256) p = fmaf(v[i], v[i], p);
  p = warp_sum(p);
  if (lane == 0) red[warp] = p;
  __syncthreads();   // (also publishes zs)
  if (t == 0) {
    float q = 0.0f;
    for (int x = 0; x < 8; ++x) q += red[x];
    s_vsq = q;
  }
  const float s = hyp[2];
  // coefficients of the two gradient sums, in place
  for (int64_t i = t; i < np; i += 256) {
    float a = 0.0f, b = 0.0f;
    if (i < n) {
      float r2 = 0.0f;
      for (int k = 0; k < d; ++k) {
        const float df = zs[k] - Zt[(int64_t)k * np + i];
        r2 = fmaf(df, df, r2);
      }
      float kv, h;
      kern_eval_grad<KERN>(r2, kv, h);
      if (EMB) {
        float r2e = 0.0f;
        for (int q = 0; q < De; ++q) {
          const float df = zs[2 * d + q] - Zt[(int64_t)(d + q) * np + i];
          r2e = fmaf(df, df, r2e);
        }
        h *= kern_eval<HB_KERN_MATERN32>(r2e);
      }
      const float c = -s * h;
      a = alpha[i] * c;
      b = -2.0f * w[i] * c;
    }
    v[i] = a;
    w[i] = b;
  }
  __syncthreads();
  // value path, exactly as mace_kernel: the mean partials first, the constant last
  float mu_t = 0.0f;
  for (int g = 0; g < ncg; ++g) mu_t += mupart[(int64_t)g * mc_pad + r];
  mu_t += hyp[1];
  float raw_var = s - s_vsq;
  if (pred_likeli) raw_var += hyp[0];           // lik(pred) adds the noise before the variance floor (gp.py:158-161)
  const float var_t = fmaxf(raw_var, 1e-6f);
  const float ps2_raw = __fmul_rn(var_t, __fmul_rn(y_std, y_std));
  const float ps2 = fmaxf(ps2_raw, 1.1920929e-07f);
  const bool live = (raw_var > 1e-6f) && (ps2_raw > 1.1920929e-07f);   // clamp_min has zero gradient where it clamps
  if (t == 0) {
    mu_out[gr] = __fadd_rn(__fmul_rn(mu_t, y_std), y_mean);
    var_out[gr] = ps2;
  }
  // gradients: one warp per input dimension
  for (int k = warp; k < d; k += 8) {
    const float zk = zs[k];
    const float *zrow = Zt + (int64_t)k * np;
    float ga = 0.0f, gb = 0.0f;
    for (int64_t i = lane; i < n; i += 32) {
      const float df = zk - zrow[i];
      ga = fmaf(v[i], df, ga);
      gb = fmaf(w[i], df, gb);
    }
    ga = warp_sum(ga);
    gb = warp_sum(gb);
    if (lane == 0) {
      const float jac = zs[d + k];   // d z_k / d x_k
      dmu[gr * d + k] = ga * jac * y_std;
      dvar[gr * d + k] = live ? gb * jac * y_std * y_std : 0.0f;
    }
  }
}

int launch_posterior_grad(const Fitted &gp, const float *Xs, const int32_t *Xe_s, int64_t m, float *mu, float *var, float *dmu,
                          float *dvar, void *ws, int64_t ws_bytes, int64_t m_chunk, cudaStream_t st) {
  const ModelSpec &sp = gp.sp;
  const int64_t d = sp.d, np = gp.np;
  if (m <= 0 || m_chunk <= 0) return HB_ERR_INVALID;
  const PostWs w = carve_posterior_ws(ws, np, m_chunk);
  if (ws_bytes < 0 || (size_t)ws_bytes < w.bytes) return HB_ERR_INVALID;
  float *V = w.KS2[0], *W = w.KS;   // W overwrites K* once V is built
  const size_t dyn = (2 * (size_t)d + sp.De) * sizeof(float);
  for (int64_t c0 = 0; c0 < m; c0 += m_chunk) {
    const int64_t mc = min(m_chunk, m - c0);
    const int64_t mc_pad = round_up(mc, GT);
    int s = launch_kstar(gp, Xs + c0 * d, sp.e > 0 ? Xe_s + c0 * sp.e : nullptr, mc, w.KS, nullptr, w.mupart[0], w.mc_pad, nullptr,
                         nullptr, st);
    if (s != HB_OK) return s;
    const dim3 g((unsigned)(np / GT), (unsigned)(mc_pad / GT));
    rows_gemm_kernel<0><<<g, GTHREADS, 0, st>>>(w.KS, gp.Linv, np, V);
    rows_gemm_kernel<1><<<g, GTHREADS, 0, st>>>(V, gp.Linv, np, W);
    s = with_kernel(gp.kern, sp.e > 0, [&](auto kk, auto ee) {
      post_grad_kernel<decltype(kk)::value, decltype(ee)::value><<<(unsigned)mc, 256, dyn, st>>>(
          Xs, (int)d, gp.x_mul, gp.x_add, gp.Zt, gp.alpha, gp.hyp, gp.n, np, V, W, w.mupart[0], kstar_groups(np), w.mc_pad, c0,
          gp.y_mean, gp.y_std, gp.pred_likeli, mu, var, dmu, dvar, Xe_s, gp.tab_s, sp);
    });
    if (s != HB_OK) return s;
    count_launches(3);
  }
  HB_LAUNCH_CHECK("posterior_grad");
  return HB_OK;
}

}  // namespace hb

// =====================================================================================================================
// Joint posterior samples  (GP.sample_y, HEBO/hebo/models/gp/gp.py:166-177: pred = gp(Xc, Xe) [; pred = lik(pred)];
// pred.rsample(n_samples) -- gpytorch draws mu + R z with R a Cholesky root of the m x m predictive covariance).
//   Zs^T  : scaled (warped / embedded) candidate features, transposed            cand_features_kernel
//   K*    : kstar_kernel (plain fp32) + mean partials;  V = K* Linv^T             rows_gemm_kernel<0>
//   K**   : gram_kernel over the candidates' own features (lower tiles)
//   cov   : K** - V V^T (+ sigma_n^2 I with pred_likeli) + jitter I               cov_update_kernel
//   R     : our tile-DAG Cholesky (launch_cholesky), jitter ladder on failure
//   y     : (mu~ + R z) y_std + y_mean                                            sample_apply_kernel
namespace hb {

__global__ void cand_features_kernel(const float *__restrict__ Xs, const int32_t *__restrict__ Xe_s, int64_t m, int64_t mp,
                                     const float *__restrict__ x_mul, const float *__restrict__ x_add, const float *__restrict__ hyp,
                                     const float *__restrict__ tab_s, ModelSpec sp, float *__restrict__ ZsT) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (int64_t)sp.dtot() * mp) return;
  const int k = (int)(idx / mp);
  const int64_t i = idx - (int64_t)k * mp;
  float z = 0.0f;
  if (i < m) {
    if (k < sp.d) z = cand_feature(sp, sp.warp, Xs[i * sp.d + k], k, x_mul, x_add, hyp);
    else z = tab_s[emb_entry(sp, Xe_s, i, k - sp.d)];
  }
  ZsT[idx] = z;
}

// lower tiles of cov [mp, mp] (holding K** from gram_kernel):  cov -= V V^T, diagonal := base + jitter - |v_i|^2, pad := I
__global__ void __launch_bounds__(GTHREADS, 2) cov_update_kernel(float *__restrict__ cov, int64_t mp, int64_t m,
                                                                 const float *__restrict__ V, int64_t np, float diag_base) {
  __shared__ GemmSmem sm;
  int I, J;
  tri_decode((int)blockIdx.x, I, J);
  float acc[8][8];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[i][j] = 0.0f;
  gemm_mainloop<true, true>(V + (int64_t)I * GT * np, np, V + (int64_t)J * GT * np, np, 0, (int)np, acc, sm);
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int64_t gi = (int64_t)I * GT + gemm_row(i);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int64_t gj = (int64_t)J * GT + gemm_col(j);
      float *p = cov + gi * mp + gj;
      float v;
      if (gi >= m || gj >= m) v = (gi == gj) ? 1.0f : 0.0f;
      else if (gi == gj) v = diag_base - acc[i][j];
      else v = *p - acc[i][j];
      *p = v;
    }
  }
}

// out[s][i] = (c + sum_g mupart[g][i] + sum_{j <= i} R[i][j] z[s][j]) y_std + y_mean      (one warp per (s, i))
__global__ void __launch_bounds__(256) sample_apply_kernel(const float *__restrict__ R, int64_t mp, int64_t m, const float *__restrict__ z,
                                                           int n_samples, const float *__restrict__ mupart, int ncg, int64_t mc_pad,
                                                           const float *__restrict__ hyp, float y_mean, float y_std,
                                                           float *__restrict__ out) {
  const int64_t w = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (w >= (int64_t)n_samples * m) return;
  const int64_t s = w / m, i = w - s * m;
  float acc = 0.0f;
  for (int64_t j = lane; j <= i; j += 32) acc = fmaf(R[i * mp + j], z[s * m + j], acc);
  acc = warp_sum(acc);
  if (lane == 0) {
    float mu = hyp[1];
    for (int g = 0; g < ncg; ++g) mu += mupart[(int64_t)g * mc_pad + i];
    out[s * m + i] = __fadd_rn(__fmul_rn(mu + acc, y_std), y_mean);
  }
}

// The sampler workspace over mp padded candidate rows: K*, V [mp, np], the mean partials, cov [mp, mp], the transposed
// candidate features, and the scratch tile and status word of launch_cholesky.
struct SampleWs {
  float *KS, *Vb, *mupart, *cov, *ZsT, *cholws;
  int32_t *info;
  int64_t mp;
  size_t bytes;
};
static SampleWs carve_sample_ws(void *ws, int64_t np, int64_t dtot, int64_t mp) {
  SampleWs w;
  w.mp = mp;
  Carver c{reinterpret_cast<float *>(ws)};
  w.KS = c.take(mp * np);
  w.Vb = c.take(mp * np);
  w.mupart = c.take(kstar_groups(np) * mp);
  w.cov = c.take(mp * mp);
  w.ZsT = c.take(dtot * mp);
  w.cholws = c.take(GT * GT);
  w.info = reinterpret_cast<int32_t *>(c.take(0));   // one word of the 1024-byte tail
  w.bytes = (size_t)c.used * sizeof(float) + 1024;
  return w;
}

// both samplers share this size: launch_sample_y pads m to 2 GT, launch_sample_y_batch to GT
size_t sample_ws_bytes(int64_t np, int64_t dtot, int64_t m) { return carve_sample_ws(nullptr, np, dtot, round_up(m, 2 * GT)).bytes; }

// K* (+ mean partials), V = K* Linv^T and the candidates' own features of m rows padded to w.mp
static int enqueue_sample_panels(const Fitted &gp, const float *Xs, const int32_t *Xe_s, int64_t m, const SampleWs &w, cudaStream_t st) {
  const int64_t np = gp.np, mp = w.mp;
  HB_CUDA(cudaMemsetAsync(w.KS, 0, (size_t)mp * np * sizeof(float), st));     // rows m..mp of K* must be zero for the GEMMs
  const int s = launch_kstar(gp, Xs, Xe_s, m, w.KS, nullptr, w.mupart, mp, nullptr, nullptr, st);
  if (s != HB_OK) return s;
  rows_gemm_kernel<0><<<dim3((unsigned)(np / GT), (unsigned)(mp / GT)), GTHREADS, 0, st>>>(w.KS, gp.Linv, np, w.Vb);
  cand_features_kernel<<<(int)ceil_div((int64_t)gp.sp.dtot() * mp, 256), 256, 0, st>>>(Xs, Xe_s, m, mp, gp.x_mul, gp.x_add, gp.hyp,
                                                                                      gp.tab_s, gp.sp, w.ZsT);
  count_launches(2);
  return HB_OK;
}

// cov = K** - V V^T over the lower tiles, diagonal diag_base - |v_i|^2
static int enqueue_sample_cov(const Fitted &gp, int64_t m, const SampleWs &w, float diag_base, cudaStream_t st) {
  const int64_t mp = w.mp;
  ModelSpec sc = gp.sp;
  sc.warp = 1;                        // "prescaled features" switch of gram_kernel: ZsT is already warped and divided by l
  const int s = launch_gram(w.ZsT, w.ZsT + (int64_t)sc.d * mp, m, mp, sc, gp.hyp, gp.kern, nullptr, 0.0f, w.cov, st);
  if (s != HB_OK) return s;
  const int nt = (int)(mp / GT);
  cov_update_kernel<<<nt * (nt + 1) / 2, GTHREADS, 0, st>>>(w.cov, mp, m, w.Vb, gp.np, diag_base);
  count_launches(1);
  return HB_OK;
}

int launch_sample_y(const Fitted &gp, const float *Xs, const int32_t *Xe_s, int64_t m, const float *hyp_host, const float *z,
                    int n_samples, float *out, float *jitter_used, void *ws, int64_t ws_bytes, cudaStream_t st) {
  if (m <= 0 || m > 8192 || n_samples <= 0) return HB_ERR_INVALID;
  if (ws_bytes < 0 || (size_t)ws_bytes < sample_ws_bytes(gp.np, gp.sp.dtot(), m)) return HB_ERR_INVALID;
  const SampleWs w = carve_sample_ws(ws, gp.np, gp.sp.dtot(), round_up(m, 2 * GT));
  int s = enqueue_sample_panels(gp, Xs, Xe_s, m, w, st);
  if (s != HB_OK) return s;
  const float sn2 = hyp_host[0], sv = hyp_host[2];
  float jitter = 1e-6f;               // gpytorch psd_safe_cholesky: fp32 jitter 1e-6, x10 per retry
  for (;;) {
    s = enqueue_sample_cov(gp, m, w, sv + (gp.pred_likeli ? sn2 : 0.0f) + jitter, st);
    if (s != HB_OK) return s;
    HB_CUDA(cudaMemsetAsync(w.info, 0, sizeof(int32_t), st));
    s = launch_cholesky(w.cov, w.mp, w.cholws, w.info, st);
    if (s != HB_OK) return s;
    int32_t h = 0;
    HB_CUDA(cudaMemcpyAsync(&h, w.info, sizeof(int32_t), cudaMemcpyDeviceToHost, st));
    HB_CUDA(cudaStreamSynchronize(st));
    if (h == 0) break;
    jitter *= 10.0f;
    if (jitter > 10.0f) return HB_ERR_NOT_PD;
  }
  if (jitter_used) *jitter_used = jitter;
  sample_apply_kernel<<<(int)ceil_div((int64_t)n_samples * m * 32, 256), 256, 0, st>>>(w.cov, w.mp, m, z, n_samples, w.mupart,
                                                                                     kstar_groups(gp.np), w.mp, gp.hyp, gp.y_mean,
                                                                                     gp.y_std, out);
  count_launches(1);
  HB_LAUNCH_CHECK("sample_y");
  return HB_OK;
}

// ---- one joint draw over a GA batch, m <= SB_MAX rows, with no host round trip (hb_sample_y_batch; NoisyAcq.eval,
// acq.py:173-190, once per generation).  K*, V, K** and the rank-n update are the stages above; cov_update_kernel runs with
// diag_base = 0, so the diagonal holds -|v_i|^2 and the kernel below adds s (+ sigma_n^2) + jitter itself, the same fp32
// sum as launch_sample_y's diag_base - |v_i|^2.  Then one CTA:
//   1. row i is dropped when it duplicates an earlier row of the batch (same_row on the numeric columns, equal categories);
//   2. the distinct rows' lower triangle goes to packed shared memory (row a at a (a + 1) / 2) and is factored in place by
//      a right-looking fp32 Cholesky; a pivot that is not positive and finite reloads it with jitter x10, from 1e-6 until
//      the jitter exceeds 10 (launch_sample_y's ladder, same fp32 arithmetic);
//   3. f = (c + sum of the mean partials + R z) y_std + y_mean for the distinct rows, +inf for the dropped ones; on give-up
//      f = NaN everywhere and *status = HB_ERR_NOT_PD.
constexpr int SB_MAX = 256;
constexpr int SB_THREADS = 1024;
constexpr size_t SB_SMEM = ((size_t)SB_MAX * (SB_MAX + 1) / 2 + 2 * SB_MAX) * sizeof(float) + 2 * SB_MAX * sizeof(int);

__global__ void __launch_bounds__(SB_THREADS, 1) sample_batch_kernel(
    const float *__restrict__ Xs, const int32_t *__restrict__ Xe_s, int m, int d, int e, const float *__restrict__ cov, int64_t mp,
    const float *__restrict__ mupart, int ncg, const float *__restrict__ hyp, int pred_likeli, float y_mean, float y_std,
    const float *__restrict__ z, uint64_t seed, uint64_t counter, float *__restrict__ f, float *__restrict__ jitter_out,
    int32_t *__restrict__ status) {
  extern __shared__ float sb_smem[];
  float *A = sb_smem;                                   // packed lower triangle of the distinct rows
  float *col = A + SB_MAX * (SB_MAX + 1) / 2;           // column j of L below the pivot
  float *zv = col + SB_MAX;                             // z by batch row
  int *idx = reinterpret_cast<int *>(zv + SB_MAX);      // batch row of distinct row a
  int *dup = idx + SB_MAX;
  __shared__ int k_s;
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5, nw = SB_THREADS / 32;
  if (t < m) {
    bool dp = false;
    for (int j = 0; j < t && !dp; ++j) {
      dp = same_row(Xs + (int64_t)j * d, Xs + (int64_t)t * d, d);
      for (int c = 0; c < e && dp; ++c) dp = Xe_s[(int64_t)j * e + c] == Xe_s[(int64_t)t * e + c];
    }
    dup[t] = dp ? 1 : 0;
    if (z) zv[t] = z[t];
  }
  if (!z && 2 * t < m) {
    float z0, z1;
    philox_normal2(seed, (counter << 7) + (uint64_t)t, z0, z1);   // rows 2t, 2t + 1 of draw `counter`
    zv[2 * t] = z0;
    if (2 * t + 1 < m) zv[2 * t + 1] = z1;
  }
  __syncthreads();
  if (t < m && !dup[t]) {
    int a = 0;
    for (int j = 0; j < t; ++j) a += 1 - dup[j];
    idx[a] = t;
  }
  if (t == 0) {
    int k = 0;
    for (int j = 0; j < m; ++j) k += 1 - dup[j];
    k_s = k;
  }
  __syncthreads();
  const int k = k_s;
  const float sn2 = hyp[0], s = hyp[2];
  const float base = s + (pred_likeli ? sn2 : 0.0f);
  float jitter = 1e-6f;   // gpytorch psd_safe_cholesky: fp32 jitter 1e-6, x10 per retry (launch_sample_y's ladder)
  bool ok = false;
  for (;;) {
    const float diag = base + jitter;
    for (int a = warp; a < k; a += nw) {
      const float *src = cov + (int64_t)idx[a] * mp;
      float *row = A + a * (a + 1) / 2;
      for (int b = lane; b <= a; b += 32) row[b] = (b == a) ? diag + src[idx[b]] : src[idx[b]];
    }
    __syncthreads();
    bool fail = false;
    for (int j = 0; j < k; ++j) {
      const int jj = j * (j + 1) / 2 + j;
      const float pv = A[jj];                            // the same word in every thread: the branch is uniform
      if (!(pv > 0.0f) || !isfinite(pv)) {
        fail = true;
        break;
      }
      const float ljj = sqrtf(pv);
      for (int i = j + 1 + t; i < k; i += SB_THREADS) {
        const float c = A[i * (i + 1) / 2 + j] / ljj;
        A[i * (i + 1) / 2 + j] = c;
        col[i] = c;
      }
      __syncthreads();
      if (t == 0) A[jj] = ljj;
      for (int i = j + 1 + warp; i < k; i += nw) {
        const float ci = col[i];
        float *row = A + i * (i + 1) / 2;
        for (int l = j + 1 + lane; l <= i; l += 32) row[l] = fmaf(-ci, col[l], row[l]);
      }
      __syncthreads();
    }
    if (!fail) {
      ok = true;
      break;
    }
    __syncthreads();                                     // every thread has read the failed pivot before the reload
    const float next = jitter * 10.0f;
    if (next > 10.0f) break;                             // give up: `jitter` stays the last rung tried
    jitter = next;
  }
  if (t == 0) *jitter_out = jitter;
  if (!ok) {
    if (t == 0) *status = HB_ERR_NOT_PD;
    if (t < m) f[t] = NAN;
    return;
  }
  if (t < m && dup[t]) f[t] = INFINITY;
  for (int a = warp; a < k; a += nw) {
    const int r = idx[a];
    const float *row = A + a * (a + 1) / 2;
    float acc = 0.0f;
    for (int b = lane; b <= a; b += 32) acc = fmaf(row[b], zv[idx[b]], acc);
    acc = warp_sum(acc);
    if (lane == 0) {
      float mu = hyp[1];
      for (int g = 0; g < ncg; ++g) mu += mupart[(int64_t)g * mp + r];
      f[r] = __fadd_rn(__fmul_rn(mu + acc, y_std), y_mean);
    }
  }
}

int launch_sample_y_batch(const Fitted &gp, const float *Xs, const int32_t *Xe_s, int64_t m, const float *z, uint64_t seed,
                          uint64_t counter, float *f, float *jitter_out, int32_t *status, void *ws, int64_t ws_bytes,
                          cudaStream_t st) {
  if (m <= 0 || m > SB_MAX) return HB_ERR_INVALID;
  if (ws_bytes < 0 || (size_t)ws_bytes < sample_ws_bytes(gp.np, gp.sp.dtot(), m)) return HB_ERR_INVALID;
  static PerDevice once;   // the opt-in above 48 KB of dynamic shared memory is per device
  bool fresh = false;
  const int dev = once.slot(&fresh);
  if (dev < 0) return HB_ERR_CUDA;
  if (fresh) {
    HB_CUDA(cudaFuncSetAttribute(sample_batch_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SB_SMEM));
    once.done[dev] = true;
  }
  const SampleWs w = carve_sample_ws(ws, gp.np, gp.sp.dtot(), round_up(m, GT));   // the row tiles that hold the m rows
  int s = enqueue_sample_panels(gp, Xs, Xe_s, m, w, st);
  if (s != HB_OK) return s;
  s = enqueue_sample_cov(gp, m, w, 0.0f, st);
  if (s != HB_OK) return s;
  sample_batch_kernel<<<1, SB_THREADS, SB_SMEM, st>>>(Xs, Xe_s, (int)m, gp.sp.d, gp.sp.e, w.cov, w.mp, w.mupart, kstar_groups(gp.np),
                                                      gp.hyp, gp.pred_likeli, gp.y_mean, gp.y_std, z, seed, counter, f, jitter_out,
                                                      status);
  count_launches(1);
  HB_LAUNCH_CHECK("sample_y_batch");
  return HB_OK;
}

}  // namespace hb
