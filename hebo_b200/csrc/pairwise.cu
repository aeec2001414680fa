// Pairwise (n x n) kernels of the fit: Gram matrix build and the closed-form MLL gradient contraction,
// plus the tiny hyper-parameter transform / pSGLD update kernels.
//
// Both pairwise kernels walk the lower 128x128 tiles of the pair matrix with the same 8x8-per-thread
// mapping as the GEMM core.  Inputs are the TRANSPOSED scaled training matrix Xt [d, NP], so a tile's
// operand is d rows of 128 contiguous floats: coalesced float4 global loads straight into shared
// memory, no transpose, and conflict-free / broadcast LDS.128 in the inner loop.  Squared distances
// use the direct-difference form sum((zi - zj)^2) (no ||a||^2+||b||^2-2ab cancellation).
//
// Replaces GPyTorchModel.forward / default_kern (HEBO/hebo/models/gp/gp.py:203-207,
// HEBO/hebo/models/gp/gp_util.py:39-59) and autograd's backward through them (gp.py:115).
#include "kernels.h"

namespace hb {

constexpr int PT = 128;   // pair tile edge
constexpr int DC = 32;    // feature-dimension chunk staged in shared memory

struct PairSmem {
  __align__(16) float xi[DC][PT];
  __align__(16) float xj[DC][PT];
};

__device__ __forceinline__ int pr_row(int i) { return (i < 4 ? 0 : 60) + (threadIdx.x >> 4) * 4 + i; }
__device__ __forceinline__ int pr_col(int j) { return (j < 4 ? 0 : 60) + (threadIdx.x & 15) * 4 + j; }

// four consecutive feature values starting at column c, times inv; columns >= n are pad and staged as 0.  The pad columns
// of Xt are whatever the caller left there (include/hebo_b200.h): NaN, Inf or a huge value would turn the zero weight of a
// pad pair into NaN (0 * Inf) in the gradient contractions, so they must never reach the arithmetic.
__device__ __forceinline__ float4 stage4(float4 v, int64_t c, int64_t n, float inv) {
  return make_float4(c < n ? v.x * inv : 0.0f, c + 1 < n ? v.y * inv : 0.0f, c + 2 < n ? v.z * inv : 0.0f,
                     c + 3 < n ? v.w * inv : 0.0f);
}

// stage rows [k0, k0+kc) of Xt for the two tiles, scaled by 1/lengthscale (ls == nullptr: rows are already scaled --
// the embedding features Ets, gathered and divided by their lengthscale once per epoch)
__device__ __forceinline__ void stage_chunk(PairSmem &sm, const float *__restrict__ Xt, int64_t n, int64_t np, int I, int J,
                                            int k0, int kc, const float *__restrict__ ls) {
  for (int f = threadIdx.x; f < kc * (PT / 4); f += blockDim.x) {
    const int kk = f >> 5, c4 = f & 31;
    const float inv = ls ? 1.0f / ls[k0 + kk] : 1.0f;
    const int64_t ci = (int64_t)I * PT + c4 * 4, cj = (int64_t)J * PT + c4 * 4;
    const float4 a = __ldg(reinterpret_cast<const float4 *>(Xt + (int64_t)(k0 + kk) * np + ci));
    const float4 b = __ldg(reinterpret_cast<const float4 *>(Xt + (int64_t)(k0 + kk) * np + cj));
    *reinterpret_cast<float4 *>(&sm.xi[kk][c4 * 4]) = stage4(a, ci, n, inv);
    *reinterpret_cast<float4 *>(&sm.xj[kk][c4 * 4]) = stage4(b, cj, n, inv);
  }
}

__device__ __forceinline__ void accum_sqdist(const PairSmem &sm, int kc, float (&r2)[8][8]) {
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
#pragma unroll 4
  for (int kk = 0; kk < kc; ++kk) {
    const float4 a0 = *reinterpret_cast<const float4 *>(&sm.xi[kk][ty * 4]);
    const float4 a1 = *reinterpret_cast<const float4 *>(&sm.xi[kk][64 + ty * 4]);
    const float4 b0 = *reinterpret_cast<const float4 *>(&sm.xj[kk][tx * 4]);
    const float4 b1 = *reinterpret_cast<const float4 *>(&sm.xj[kk][64 + tx * 4]);
    const float a[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
    const float b[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float df = a[i] - b[j];
        r2[i][j] = fmaf(df, df, r2[i][j]);
      }
  }
}

// =============================================================================== Gram
// EMB: mixed model (gp_util.py:54-57): K = s * k_KERN(r over the numeric dims) * Matern32(r over the embedding dims, one
// lengthscale); Ets [De, NP] = embedding features of the training rows already divided by that lengthscale.
template <int KERN, bool EMB>
__global__ void __launch_bounds__(256, EMB ? 1 : 2) gram_kernel(const float *__restrict__ Xt, const float *__restrict__ Ets,
                                                                int64_t n, int64_t np, int d, int De,
                                                                const float *__restrict__ hyp,
                                                                const float *__restrict__ noise_diag, float jitter,
                                                                float *__restrict__ K, int prescaled, int64_t xs, int64_t wss) {
  __shared__ PairSmem sm;
  const int b = blockIdx.z;   // output (Batch): Xt is per output only when it is the warped Zt
  Xt = slice(Xt, xs, b);
  Ets = slice(Ets, wss, b);
  hyp = slice(hyp, wss, b);
  K = slice(K, wss, b);
  int I, J;
  tri_decode((int)blockIdx.x, I, J);
  float r2[8][8];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) r2[i][j] = 0.0f;
  const float *ls = prescaled ? nullptr : hyp + 3;   // prescaled: Xt already holds warp(x) / lengthscale (scale_zt_kernel)
  for (int k0 = 0; k0 < d; k0 += DC) {
    const int kc = min(DC, d - k0);
    __syncthreads();
    stage_chunk(sm, Xt, n, np, I, J, k0, kc, ls);
    __syncthreads();
    accum_sqdist(sm, kc, r2);
  }
  float r2e[8][8];   // (dead code unless EMB)
  if (EMB) {
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
      for (int j = 0; j < 8; ++j) r2e[i][j] = 0.0f;
    for (int k0 = 0; k0 < De; k0 += DC) {
      const int kc = min(DC, De - k0);
      __syncthreads();
      stage_chunk(sm, Ets, n, np, I, J, k0, kc, nullptr);
      __syncthreads();
      accum_sqdist(sm, kc, r2e);
    }
  }
  const float sn2 = hyp[0], s = hyp[2];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int64_t gi = (int64_t)I * PT + pr_row(i);
#pragma unroll
    for (int jh = 0; jh < 2; ++jh) {
      float o[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int64_t gj = (int64_t)J * PT + pr_col(jh * 4 + u);
        float v;
        if (gi >= n || gj >= n) {
          v = (gi == gj) ? 1.0f : 0.0f;
        } else {
          v = s * kern_eval<KERN>(r2[i][jh * 4 + u]);
          if (EMB) v *= kern_eval<HB_KERN_MATERN32>(r2e[i][jh * 4 + u]);
          if (gi == gj) v = s + sn2 + jitter + (noise_diag ? noise_diag[gi] : 0.0f);
        }
        o[u] = v;
      }
      *reinterpret_cast<float4 *>(K + gi * np + (int64_t)J * PT + pr_col(jh * 4)) = make_float4(o[0], o[1], o[2], o[3]);
    }
  }
}

int launch_gram(const float *Xt, const float *Ets, int64_t n, int64_t np, const ModelSpec &sp, const float *hyp, int kern,
                const float *noise_diag, float jitter, float *K, cudaStream_t st, const Batch &bt) {
  if (n <= 0 || sp.dtot() <= 0 || np % PT != 0 || n > np || (sp.e > 0 && !Ets)) return HB_ERR_INVALID;
  const int nt = (int)(np / PT);
  const dim3 grid((unsigned)(nt * (nt + 1) / 2), 1, (unsigned)bt.nout);
  const int pre = sp.warp ? 1 : 0;   // warped models: the caller passes Zt = warp(Xt) / lengthscale in place of Xt
  const int64_t xs = sp.warp ? bt.ws : 0;
  const int s = with_kernel(kern, sp.e > 0, [&](auto kk, auto ee) {
    gram_kernel<decltype(kk)::value, decltype(ee)::value><<<grid, 256, 0, st>>>(Xt, Ets, n, np, sp.d, sp.De, hyp, noise_diag,
                                                                                 jitter, K, pre, xs, bt.ws);
  });
  if (s != HB_OK) return s;
  count_launches(1);
  HB_LAUNCH_CHECK("gram");
  return HB_OK;
}

// =============================================================================== MLL gradient contraction
// Per lower tile:  G_ij = w * W_ij * s * h(r_ij)  with  W = alpha alpha^T - Khat^-1, then for every feature k
//   part[k]   = sum_ij G_ij * dz_ijk^2            (-> dK/dl_k contraction, divided by l_k in the finish kernel)
//   part[d]   = sum_ij w * W_ij * k(r_ij)         (-> d/d outputscale)
//   part[d+1] = sum_i  W_ii                       (-> d/d noise)
// w = 2 on strictly-lower tiles (symmetry), 1 on diagonal tiles (computed in full).  Per-block partials are
// written out and reduced in a fixed order in fp64 by mll_finish_kernel: deterministic, no float atomics.
// EMB (mixed model, k = phi1(r1) phi2(r2), oracle/emb_oracle.py): G1 = w W s phi2 h1 drives the numeric contraction,
//   part[d+2] = sum_ij w W s phi1 h2 r2_ij^2       (-> d/d embedding lengthscale, divided by it in the finish kernel)
template <int KERN, bool EMB>
__global__ void __launch_bounds__(256, EMB ? 1 : 2) mll_grad_kernel(const float *__restrict__ Xt, const float *__restrict__ Ets,
                                                                    int64_t n, int64_t np, int d, int De,
                                                                    const float *__restrict__ hyp,
                                                                    const float *__restrict__ Kinv,
                                                                    const float *__restrict__ alpha,
                                                                    float *__restrict__ part, const float *__restrict__ dZa,
                                                                    const float *__restrict__ dZb, int64_t xs, int64_t wss) {
  __shared__ PairSmem sm;
  // output (Batch): the per-output pointers are formed where they are used, so the parameters stay in the constant bank
#define OUT(p, st) slice(p, st, blockIdx.z)
  __shared__ float wpart[8][DC];   // per-warp partials of the current feature chunk, summed in warp order into `part`
  int I, J;
  tri_decode((int)blockIdx.x, I, J);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int stride = d + 2 + (EMB ? 1 : 0) + (dZa ? 2 * d : 0);   // dZa != nullptr: warped model, Xt = Zt is prescaled
  float *bpart = OUT(part, wss) + (int64_t)blockIdx.x * stride;
  // after a feature chunk: part slots [slot, slot + kc) of this block = sum over the warps, in warp order 0..7
  auto flush = [&](int slot, int kc) {
    __syncthreads();
    if ((int)threadIdx.x < kc) {
      float v = 0.0f;
#pragma unroll
      for (int wv = 0; wv < 8; ++wv) v += wpart[wv][threadIdx.x];
      bpart[slot + threadIdx.x] = v;
    }
  };

  float g[8][8];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) g[i][j] = 0.0f;
  const float *ls = dZa ? nullptr : OUT(hyp, wss) + 3;
  for (int k0 = 0; k0 < d; k0 += DC) {
    const int kc = min(DC, d - k0);
    __syncthreads();
    stage_chunk(sm, OUT(Xt, xs), n, np, I, J, k0, kc, ls);
    __syncthreads();
    accum_sqdist(sm, kc, g);
  }
  float r2e[8][8];   // (dead code unless EMB)
  if (EMB) {
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
      for (int j = 0; j < 8; ++j) r2e[i][j] = 0.0f;
    for (int k0 = 0; k0 < De; k0 += DC) {
      const int kc = min(DC, De - k0);
      __syncthreads();
      stage_chunk(sm, OUT(Ets, wss), n, np, I, J, k0, kc, nullptr);
      __syncthreads();
      accum_sqdist(sm, kc, r2e);
    }
  }
  // g currently holds r2; turn it into G and collect the scalar sums
  const float s = OUT(hyp, wss)[2];
  const float w = (I > J) ? 2.0f : 1.0f;
  float sum_wk = 0.0f, tr_w = 0.0f, sum_le = 0.0f;
  float ai[8], aj[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    ai[i] = OUT(alpha, wss)[(int64_t)I * PT + pr_row(i)];
    aj[i] = OUT(alpha, wss)[(int64_t)J * PT + pr_col(i)];
  }
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int64_t gi = (int64_t)I * PT + pr_row(i);
#pragma unroll
    for (int jh = 0; jh < 2; ++jh) {
      const float4 kv = __ldg(reinterpret_cast<const float4 *>(OUT(Kinv, wss) + gi * np + (int64_t)J * PT + pr_col(jh * 4)));
      const float kvv[4] = {kv.x, kv.y, kv.z, kv.w};
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int j = jh * 4 + u;
        const int64_t gj = (int64_t)J * PT + pr_col(j);
        float kk, hh;
        kern_eval_grad<KERN>(g[i][j], kk, hh);
        float W = fmaf(ai[i], aj[j], -kvv[u]);
        if (gi >= n || gj >= n) W = 0.0f;
        if (EMB) {
          float k2, h2;
          kern_eval_grad<HB_KERN_MATERN32>(r2e[i][j], k2, h2);
          sum_le = fmaf(w * W * s * kk * h2, r2e[i][j], sum_le);
          hh *= k2;
          kk *= k2;
        }
        sum_wk = fmaf(w * W, kk, sum_wk);
        if (gi == gj) tr_w += W;
        g[i][j] = w * W * s * hh;
      }
    }
  }
  // second pass over the features: per-dimension contraction
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  for (int k0 = 0; k0 < d; k0 += DC) {
    const int kc = min(DC, d - k0);
    __syncthreads();
    stage_chunk(sm, OUT(Xt, xs), n, np, I, J, k0, kc, ls);
    __syncthreads();
    for (int kk = 0; kk < kc; ++kk) {
      const float4 a0 = *reinterpret_cast<const float4 *>(&sm.xi[kk][ty * 4]);
      const float4 a1 = *reinterpret_cast<const float4 *>(&sm.xi[kk][64 + ty * 4]);
      const float4 b0 = *reinterpret_cast<const float4 *>(&sm.xj[kk][tx * 4]);
      const float4 b1 = *reinterpret_cast<const float4 *>(&sm.xj[kk][64 + tx * 4]);
      const float a[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
      const float b[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
      float p = 0.0f;
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const float df = a[i] - b[j];
          p = fmaf(g[i][j] * df, df, p);
        }
      p = warp_sum(p);
      if (lane == 0) wpart[warp][kk] = p;
    }
    flush(k0, kc);
  }
  // warped model: d K / d a_k = -s h dz_k dz'_k with z' = d z / d a_k (same for b): two more sweeps, 16 features at a time
  // (the z rows in the lower half of the staging buffers, the derivative rows in the upper half)
  if (dZa) {
    for (int which = 0; which < 2; ++which) {
      const float *dZ = which ? OUT(dZb, wss) : OUT(dZa, wss);
      const int slot0 = d + 2 + (EMB ? 1 : 0) + which * d;
      for (int k0 = 0; k0 < d; k0 += DC / 2) {
        const int kc = min(DC / 2, d - k0);
        __syncthreads();
        for (int f = threadIdx.x; f < 2 * kc * (PT / 4); f += blockDim.x) {
          const int kk = f >> 5, c4 = f & 31;
          const float *src = (kk < kc) ? OUT(Xt, xs) + (int64_t)(k0 + kk) * np : dZ + (int64_t)(k0 + kk - kc) * np;
          const int row = (kk < kc) ? kk : DC / 2 + (kk - kc);
          const int64_t ci = (int64_t)I * PT + c4 * 4, cj = (int64_t)J * PT + c4 * 4;
          *reinterpret_cast<float4 *>(&sm.xi[row][c4 * 4]) = stage4(__ldg(reinterpret_cast<const float4 *>(src + ci)), ci, n, 1.0f);
          *reinterpret_cast<float4 *>(&sm.xj[row][c4 * 4]) = stage4(__ldg(reinterpret_cast<const float4 *>(src + cj)), cj, n, 1.0f);
        }
        __syncthreads();
        for (int kk = 0; kk < kc; ++kk) {
          float a[8], b[8], da[8], db[8];
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const float4 av = *reinterpret_cast<const float4 *>(&sm.xi[kk][h * 64 + ty * 4]);
            const float4 bv = *reinterpret_cast<const float4 *>(&sm.xj[kk][h * 64 + tx * 4]);
            const float4 dav = *reinterpret_cast<const float4 *>(&sm.xi[DC / 2 + kk][h * 64 + ty * 4]);
            const float4 dbv = *reinterpret_cast<const float4 *>(&sm.xj[DC / 2 + kk][h * 64 + tx * 4]);
            a[h * 4 + 0] = av.x; a[h * 4 + 1] = av.y; a[h * 4 + 2] = av.z; a[h * 4 + 3] = av.w;
            b[h * 4 + 0] = bv.x; b[h * 4 + 1] = bv.y; b[h * 4 + 2] = bv.z; b[h * 4 + 3] = bv.w;
            da[h * 4 + 0] = dav.x; da[h * 4 + 1] = dav.y; da[h * 4 + 2] = dav.z; da[h * 4 + 3] = dav.w;
            db[h * 4 + 0] = dbv.x; db[h * 4 + 1] = dbv.y; db[h * 4 + 2] = dbv.z; db[h * 4 + 3] = dbv.w;
          }
          float p = 0.0f;
#pragma unroll
          for (int i = 0; i < 8; ++i)
#pragma unroll
            for (int j = 0; j < 8; ++j) p = fmaf(g[i][j] * (a[i] - b[j]), da[i] - db[j], p);
          p = warp_sum(p);
          if (lane == 0) wpart[warp][kk] = p;
        }
        flush(slot0 + k0, kc);
      }
    }
  }
  sum_wk = warp_sum(sum_wk);
  tr_w = warp_sum(tr_w);
  if (EMB) sum_le = warp_sum(sum_le);
  __syncthreads();   // the last chunk's partials have been read
  if (lane == 0) {
    wpart[warp][0] = sum_wk;
    wpart[warp][1] = tr_w;
    if (EMB) wpart[warp][2] = sum_le;
  }
  flush(d, EMB ? 3 : 2);
}
#undef OUT

// ---- gradient w.r.t. the embedding rows (mixed model):  d data / d e_i = -(1/le) sum_j G2_ij (E_i - E_j),
// G2 = W s phi1 h2 over the FULL pair matrix (both (i,j) and (j,i) contribute, which cancels the 1/2), E = e / le.
// Grid (J, I) over all tiles; tile (I, J) writes the partial row sums  gE[J][q][i in tile I] = sum_{j in tile J} G2_ij dE_ijq
// (fixed order: 8 columns in-thread, then a 16-lane butterfly) -> deterministic; emb_scatter_kernel adds them up per
// table entry.  Kinv holds lower tiles only: W_ij is read transposed for I < J.
template <int KERN>
__global__ void __launch_bounds__(256, 1) emb_rowgrad_kernel(const float *__restrict__ Xt, const float *__restrict__ Ets,
                                                             int64_t n, int64_t np, int d, int De,
                                                             const float *__restrict__ hyp, const float *__restrict__ Kinv,
                                                             const float *__restrict__ alpha, float *__restrict__ gE, int prescaled,
                                                             int64_t xs, int64_t wss) {
  __shared__ PairSmem sm;
  {
    const int b = blockIdx.z;   // output (Batch)
    Xt = slice(Xt, xs, b);
    Ets = slice(Ets, wss, b);
    hyp = slice(hyp, wss, b);
    Kinv = slice(Kinv, wss, b);
    alpha = slice(alpha, wss, b);
    gE = slice(gE, wss, b);
  }
  const int J = blockIdx.x, I = blockIdx.y;
  float g[8][8], r2e[8][8];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) g[i][j] = r2e[i][j] = 0.0f;
  const float *ls = prescaled ? nullptr : hyp + 3;
  for (int k0 = 0; k0 < d; k0 += DC) {
    const int kc = min(DC, d - k0);
    __syncthreads();
    stage_chunk(sm, Xt, n, np, I, J, k0, kc, ls);
    __syncthreads();
    accum_sqdist(sm, kc, g);
  }
  for (int k0 = 0; k0 < De; k0 += DC) {
    const int kc = min(DC, De - k0);
    __syncthreads();
    stage_chunk(sm, Ets, n, np, I, J, k0, kc, nullptr);
    __syncthreads();
    accum_sqdist(sm, kc, r2e);
  }
  const float s = hyp[2];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int64_t gi = (int64_t)I * PT + pr_row(i);
    const float ai = alpha[gi];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int64_t gj = (int64_t)J * PT + pr_col(j);
      const float kinv = (I >= J) ? Kinv[gi * np + gj] : Kinv[gj * np + gi];
      float W = fmaf(ai, alpha[gj], -kinv);
      if (gi >= n || gj >= n) W = 0.0f;
      float k2, h2;
      kern_eval_grad<HB_KERN_MATERN32>(r2e[i][j], k2, h2);
      g[i][j] = W * s * kern_eval<KERN>(g[i][j]) * h2;
    }
  }
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  for (int k0 = 0; k0 < De; k0 += DC) {
    const int kc = min(DC, De - k0);
    __syncthreads();
    stage_chunk(sm, Ets, n, np, I, J, k0, kc, nullptr);
    __syncthreads();
    for (int kk = 0; kk < kc; ++kk) {
      const float4 a0 = *reinterpret_cast<const float4 *>(&sm.xi[kk][ty * 4]);
      const float4 a1 = *reinterpret_cast<const float4 *>(&sm.xi[kk][64 + ty * 4]);
      const float4 b0 = *reinterpret_cast<const float4 *>(&sm.xj[kk][tx * 4]);
      const float4 b1 = *reinterpret_cast<const float4 *>(&sm.xj[kk][64 + tx * 4]);
      const float a[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
      const float b[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        float p = 0.0f;
#pragma unroll
        for (int j = 0; j < 8; ++j) p = fmaf(g[i][j], a[i] - b[j], p);
#pragma unroll
        for (int o = 8; o > 0; o >>= 1) p += __shfl_xor_sync(0xffffffffu, p, o);
        if (tx == 0) gE[((int64_t)J * De + k0 + kk) * np + (int64_t)I * PT + pr_row(i)] = p;
      }
    }
  }
}

// one block per table entry t = (column c, category u, coordinate q):  grad[1 + t] = (1 / (n le)) sum_{i: Xe[i,c] == u} sum_J gE[J][q][i]
__global__ void __launch_bounds__(256) emb_scatter_kernel(const float *__restrict__ gE, int nt, int64_t n, int64_t np, ModelSpec sp,
                                                          const float *__restrict__ hyp, float *__restrict__ grad, int64_t wss) {
  __shared__ double red[256];
  const int t = blockIdx.x;   // (output: blockIdx.z, Batch)
  const int c = sp.ent_col[t], u = sp.ent_u[t];
  int qg = sp.ent_q[t];   // global embedding coordinate = (#coordinates of earlier columns) + coordinate inside column c
  for (int cc = 0; cc < c; ++cc) qg += sp.emb_size[cc];
  double acc = 0.0;
  for (int64_t i = threadIdx.x; i < n; i += blockDim.x) {
    if (sp.Xe[i * sp.e + c] != u) continue;
    float a = 0.0f;
    for (int Jt = 0; Jt < nt; ++Jt) a += slice(gE, wss, blockIdx.z)[((int64_t)Jt * sp.De + qg) * np + i];
    acc += (double)a;
  }
  red[threadIdx.x] = acc;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if ((int)threadIdx.x < o) red[threadIdx.x] += red[threadIdx.x + o];
    __syncthreads();
  }
  if (threadIdx.x == 0)
    slice(grad, wss, blockIdx.z)[sp.i_tab() + t] = (float)(red[0] / ((double)n * (double)slice(hyp, wss, blockIdx.z)[3 + sp.d]));
}

// One block: reduce the per-tile partials in fp64, add the priors, chain through softplus, scale by -1/n.
// grad order = raw order (ModelSpec: raw_noise, [tables], mean, raw_outputscale, raw_lengthscale[n_ls], [raw emb lengthscale]).
__global__ void __launch_bounds__(256) mll_finish_kernel(const float *__restrict__ part, int nblocks, int64_t n, ModelSpec sp,
                                                         const float *__restrict__ raw, const float *__restrict__ hyp,
                                                         const float *__restrict__ alpha,
                                                         const double *__restrict__ scal, float noise_guess,
                                                         float *__restrict__ grad, float *__restrict__ loss, int64_t wss) {
  {
    const int b = blockIdx.z;   // output (Batch): raw rows are P apart
    part = slice(part, wss, b);
    raw += (int64_t)b * sp.P();
    hyp = slice(hyp, wss, b);
    alpha = slice(alpha, wss, b);
    scal = slice(scal, wss, b);
    grad = slice(grad, wss, b);
    loss = slice(loss, wss, b);
  }
  const int d = sp.d;
  const int stride = d + 2 + (sp.e > 0 ? 1 : 0) + sp.n_w();
  __shared__ double red[256];
  __shared__ double tot[4];  // sum_wk, tr_w, sum alpha, sum_le
  // per-dimension sums: thread k owns dimension k (strided), fixed summation order over blocks
  const double inv_n = -1.0 / (double)n;
  double shared_ls = 0.0;    // ard_kernel=False: one lengthscale, d l_k / d l = 1 for every k
  for (int k = threadIdx.x; k < d; k += blockDim.x) {
    double acc = 0.0;
    for (int b = 0; b < nblocks; ++b) acc += (double)part[(int64_t)b * stride + k];
    const double l = (double)hyp[3 + k];
    const double g_ls = 0.5 * acc / l;
    if (sp.ard) {
      const double sg = 1.0 / (1.0 + exp(-(double)raw[sp.i_ls() + k]));
      grad[sp.i_ls() + k] = (float)(g_ls * sg * inv_n);
    } else {
      shared_ls += g_ls;
    }
  }
  // Kumaraswamy exponents: g_a[k] = -1/2 sum G dz dz'_a, chained through a = lo + (hi - lo) sigmoid(raw) (layers.py:96-104);
  // a frozen warp (fixed exponents, sp.warp == 2) gets a zero gradient and is skipped by the optimiser step
  if (sp.warp) {
    const int slot0 = d + 2 + (sp.e > 0 ? 1 : 0);
    for (int k = threadIdx.x; k < 2 * d; k += blockDim.x) {
      double acc = 0.0;
      for (int b = 0; b < nblocks; ++b) acc += (double)part[(int64_t)b * stride + slot0 + k];
      const double sg = 1.0 / (1.0 + exp(-(double)raw[sp.i_wa() + k]));
      const double chain = (double)(WARP_HI - WARP_LO) * sg * (1.0 - sg);
      grad[sp.i_wa() + k] = sp.warp == 2 ? 0.0f : (float)(-0.5 * acc * chain * inv_n);
    }
  }
  for (int which = 0; which < 5; ++which) {
    double acc = 0.0;
    if (which < 2) {
      for (int b = threadIdx.x; b < nblocks; b += blockDim.x) acc += (double)part[(int64_t)b * stride + d + which];
    } else if (which == 2) {
      for (int64_t i = threadIdx.x; i < n; i += blockDim.x) acc += (double)alpha[i];
    } else if (which == 3) {
      if (sp.e > 0)
        for (int b = threadIdx.x; b < nblocks; b += blockDim.x) acc += (double)part[(int64_t)b * stride + d + 2];
    } else {
      acc = shared_ls;
    }
    red[threadIdx.x] = acc;
    __syncthreads();
    for (int o = 128; o > 0; o >>= 1) {
      if ((int)threadIdx.x < o) red[threadIdx.x] += red[threadIdx.x + o];
      __syncthreads();
    }
    if (threadIdx.x == 0) {
      if (which < 4) tot[which] = red[0];
      else if (!sp.ard && d > 0) grad[sp.i_ls()] = (float)(red[0] * (1.0 / (1.0 + exp(-(double)raw[sp.i_ls()]))) * inv_n);
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    const double s = (double)hyp[2], sn2 = (double)hyp[0];
    const double sig0 = 0.5, mu0 = log((double)noise_guess);
    double g_s = 0.5 * tot[0] + (-0.5 / s - 0.5);
    double g_n = 0.5 * tot[1] + (-1.0 / sn2 - (log(sn2) - mu0) / (sig0 * sig0 * sn2));
    double g_c = tot[2];
    const double sg_n = 1.0 / (1.0 + exp(-(double)raw[0]));
    const double sg_s = 1.0 / (1.0 + exp(-(double)raw[sp.i_os()]));
    grad[0] = (float)(g_n * sg_n * inv_n);
    grad[sp.i_mean()] = (float)(g_c * inv_n);
    grad[sp.i_os()] = (float)(g_s * sg_s * inv_n);
    if (sp.e > 0) {
      const double le = (double)hyp[3 + d];
      const double sg_e = 1.0 / (1.0 + exp(-(double)raw[sp.i_le()]));
      grad[sp.i_le()] = (float)(0.5 * tot[3] / le * sg_e * inv_n);
    }
    const double quad = scal[0], logdet = scal[1];
    const double data = -0.5 * (quad + logdet + (double)n * 1.8378770664093453);  // log(2 pi)
    const double lp_os = 0.5 * log(0.5) - 0.5723649429247001 - 0.5 * log(s) - 0.5 * s;  // lgamma(.5)=log(sqrt(pi))
    const double lp_n = -log(sn2 * sig0 * 2.5066282746310002) - (log(sn2) - mu0) * (log(sn2) - mu0) / (2 * sig0 * sig0);
    loss[0] = (float)(-(data + lp_os + lp_n) / (double)n);
  }
}

size_t grad_ws_bytes(int64_t np, const ModelSpec &sp) {
  const int64_t nt = np / PT;
  size_t b = (size_t)(nt * (nt + 1) / 2) * (size_t)(3 * sp.d + 3) * sizeof(float);
  b = (b + 255) / 256 * 256;
  if (sp.e > 0) b += (size_t)nt * sp.De * np * sizeof(float);   // gE partial row sums [nt][De][np]
  return b;
}

int launch_mll_grad(const float *Xt, const float *Ets, int64_t n, int64_t np, const ModelSpec &sp, const float *raw,
                    const float *hyp, int kern, const float *Kinv, const float *alpha, const double *scal, float noise_guess,
                    float *grad, float *loss, void *ws, cudaStream_t st, const float *dZa, const float *dZb, const Batch &bt) {
  if (sp.warp && (!dZa || !dZb)) return HB_ERR_INVALID;   // warped model: Xt must be Zt = warp(x) / l, with its derivative rows
  if (!sp.warp) dZa = dZb = nullptr;
  if (n <= 0 || sp.dtot() <= 0 || np % PT != 0 || n > np || (sp.e > 0 && !Ets)) return HB_ERR_INVALID;
  const int nt = (int)(np / PT);
  const int grid = nt * (nt + 1) / 2;
  const int d = sp.d;
  const unsigned nz = (unsigned)bt.nout;
  const int64_t xs = sp.warp ? bt.ws : 0;   // Xt is the per-output Zt of a warped model
  float *part = reinterpret_cast<float *>(ws);
  int s = with_kernel(kern, sp.e > 0, [&](auto kk, auto ee) {
    mll_grad_kernel<decltype(kk)::value, decltype(ee)::value><<<dim3((unsigned)grid, 1, nz), 256, 0, st>>>(
        Xt, Ets, n, np, d, sp.De, hyp, Kinv, alpha, part, dZa, dZb, xs, bt.ws);
  });
  if (s != HB_OK) return s;
  mll_finish_kernel<<<dim3(1, 1, nz), 256, 0, st>>>(part, grid, n, sp, raw, hyp, alpha, scal, noise_guess, grad, loss, bt.ws);
  count_launches(2);
  if (sp.e > 0) {
    size_t off = (size_t)grid * (size_t)(3 * d + 3) * sizeof(float);
    off = (off + 255) / 256 * 256;
    float *gE = reinterpret_cast<float *>(reinterpret_cast<unsigned char *>(ws) + off);
    const dim3 g2((unsigned)nt, (unsigned)nt, nz);
    s = with_kernel(kern, [&](auto kk) {
      emb_rowgrad_kernel<decltype(kk)::value><<<g2, 256, 0, st>>>(Xt, Ets, n, np, d, sp.De, hyp, Kinv, alpha, gE, sp.warp ? 1 : 0,
                                                                  xs, bt.ws);
    });
    if (s != HB_OK) return s;
    emb_scatter_kernel<<<dim3((unsigned)sp.T, 1, nz), 256, 0, st>>>(gE, nt, n, np, sp, hyp, grad, bt.ws);
    count_launches(2);
  }
  HB_LAUNCH_CHECK("mll_grad");
  return HB_OK;
}

// =============================================================================== small kernels
// gpytorch Positive() / GreaterThan() constraints (gp.py:86, gp_util.py:46,55,57): raw (ModelSpec layout) -> hyp
__global__ void transform_hypers_kernel(const float *__restrict__ raw, ModelSpec sp, float noise_lb, float *__restrict__ hyp,
                                        int64_t wss) {
  raw += (int64_t)blockIdx.z * sp.P();
  hyp = slice(hyp, wss, blockIdx.z);
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= sp.H()) return;
  float v;
  if (i == 0) v = softplus_f(raw[0]) + noise_lb;
  else if (i == 1) v = raw[sp.i_mean()];
  else if (i == 2) v = softplus_f(raw[sp.i_os()]);
  else if (i < 3 + sp.d) v = softplus_f(raw[sp.i_ls() + (sp.ard ? i - 3 : 0)]);
  else if (sp.e > 0 && i == 3 + sp.d) v = softplus_f(raw[sp.i_le()]);
  else v = WARP_LO + (WARP_HI - WARP_LO) * sigmoid_f(raw[sp.i_wa() + (i - sp.h_wa())]);   // a[d] then b[d]: layers.py:96-104
  hyp[i] = v;
}

int launch_transform_hypers(const float *raw, const ModelSpec &sp, float noise_lb, float *hyp, cudaStream_t st,
                            const Batch &bt) {
  if (sp.dtot() <= 0) return HB_ERR_INVALID;
  transform_hypers_kernel<<<dim3((unsigned)ceil_div(sp.H(), 128), 1, (unsigned)bt.nout), 128, 0, st>>>(raw, sp, noise_lb, hyp,
                                                                                                        bt.ws);
  count_launches(1);
  HB_LAUNCH_CHECK("transform_hypers");
  return HB_OK;
}

__global__ void psgld_kernel(float *__restrict__ raw, const float *__restrict__ grad, float *__restrict__ sq, int p,
                             float lr, float a, float eps, float factor, const float *__restrict__ xi) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= p) return;
  psgld_update(raw, grad, sq, i, lr, a, eps, factor, xi);
}

int launch_psgld(float *raw, const float *grad, float *sq, int64_t p, float lr, float a, float eps, float factor,
                 const float *xi, cudaStream_t st) {
  if (p <= 0) return HB_ERR_INVALID;
  psgld_kernel<<<(int)ceil_div(p, 128), 128, 0, st>>>(raw, grad, sq, (int)p, lr, a, eps, factor, xi);
  count_launches(1);
  HB_LAUNCH_CHECK("psgld");
  return HB_OK;
}

// Zt = f(Xt) / lengthscale with f = identity or the Kumaraswamy warp (exponents in hyp); with a warp also the derivative
// rows dZa = d z / d a_k, dZb = d z / d b_k the gradient contraction needs (O(n d): a prologue of the epoch, the n^2 kernels
// read Zt; the CANDIDATE side is warped inside the K* load stage, posterior.cu).
__global__ void scale_zt_kernel(const float *__restrict__ Xt, int64_t np, ModelSpec sp, const float *__restrict__ hyp,
                                float *__restrict__ Zt, float *__restrict__ dZa, float *__restrict__ dZb, int64_t wss) {
  hyp = slice(hyp, wss, blockIdx.z);   // (Xt is shared by the outputs of a batch)
  Zt = slice(Zt, wss, blockIdx.z);
  dZa = slice(dZa, wss, blockIdx.z);
  dZb = slice(dZb, wss, blockIdx.z);
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (int64_t)sp.d * np) return;
  const int k = (int)(idx / np);
  const float il = 1.0f / hyp[3 + k];
  if (!sp.warp) {
    Zt[idx] = Xt[idx] * il;
    return;
  }
  float da, db;
  const float w = kumar_warp(Xt[idx], hyp[sp.h_wa() + k], hyp[sp.h_wb() + k], &da, &db);
  Zt[idx] = w * il;
  if (dZa) dZa[idx] = da * il;
  if (dZb) dZb[idx] = db * il;
}

int launch_scale_zt(const float *Xt, int64_t np, const ModelSpec &sp, const float *hyp, float *Zt, float *dZa, float *dZb,
                    cudaStream_t st, const Batch &bt) {
  if (sp.d <= 0) return HB_OK;
  scale_zt_kernel<<<dim3((unsigned)ceil_div((int64_t)sp.d * np, 256), 1, (unsigned)bt.nout), 256, 0, st>>>(Xt, np, sp, hyp, Zt, dZa,
                                                                                                          dZb, bt.ws);
  count_launches(1);
  HB_LAUNCH_CHECK("scale_zt");
  return HB_OK;
}

// ---- embedding features (layers.py:33-34 EmbTransform.forward), already divided by the embedding lengthscale:
//   Ets [De, NP]: Ets[q][i] = table_{c(q)}[Xe[i, c(q)]][q_loc(q)] / le   (pad columns zero)
//   tab_s [T]   : tables / le   (the candidate side of the posterior gathers from it)
__global__ void emb_gather_kernel(const float *__restrict__ tables, ModelSpec sp, int64_t n, int64_t np,
                                  const float *__restrict__ hyp, float *__restrict__ Ets, float *__restrict__ tab_s, int64_t wss) {
  tables += (int64_t)blockIdx.z * sp.P();   // raw rows are P apart; the categories sp.Xe are shared
  hyp = slice(hyp, wss, blockIdx.z);
  Ets = slice(Ets, wss, blockIdx.z);
  tab_s = slice(tab_s, wss, blockIdx.z);
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const float inv = 1.0f / hyp[3 + sp.d];
  if (tab_s && idx < sp.T) tab_s[idx] = tables[idx] * inv;
  if (idx >= (int64_t)sp.De * np) return;
  const int q = (int)(idx / np);
  const int64_t i = idx - (int64_t)q * np;
  float v = 0.0f;
  if (i < n) v = tables[emb_entry(sp, sp.Xe, i, q)] * inv;
  Ets[idx] = v;
}

int launch_emb_gather(const float *tables, const ModelSpec &sp, int64_t n, int64_t np, const float *hyp, float *Ets, float *tab_s,
                      cudaStream_t st, const Batch &bt) {
  if (sp.e <= 0) return HB_OK;
  const int64_t work = sp.De * np > sp.T ? sp.De * np : sp.T;
  emb_gather_kernel<<<dim3((unsigned)ceil_div(work, 256), 1, (unsigned)bt.nout), 256, 0, st>>>(tables, sp, n, np, hyp, Ets, tab_s,
                                                                                             bt.ws);
  count_launches(1);
  HB_LAUNCH_CHECK("emb_gather");
  return HB_OK;
}

}  // namespace hb
