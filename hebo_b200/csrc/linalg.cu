// Dense linear algebra of the exact-GP fit on padded [NP, NP] fp32 matrices (NP multiple of 128), next to the
// Cholesky factorisation in cholesky.cu: triangular inverse by recursive doubling (all GEMM),
// K^-1 = Linv^T Linv, and alpha / quadratic form / log-det by fp64-accumulated GEMVs.
// These replace what gpytorch does inside ExactMarginalLogLikelihood + autograd for
// HEBO/hebo/models/gp/gp.py:112-115 (psd_safe_cholesky, cholesky_solve, logdet and their backward).
#include "gemm_core.cuh"
#include "kernels.h"

namespace hb {

// =============================================================================== triangular inverse
// Base case: each CTA inverts one 128x128 lower-triangular diagonal block; thread i produces row i of
// the inverse by back-substitution X L = I, running j = i .. 0 with its row kept in shared memory.
struct TriBaseSmem {
  float Ls[GT][GT + 1];
  float Xs[GT][GT + 1];
};

__global__ void __launch_bounds__(GT) triinv_base_kernel(const float *__restrict__ L, int64_t np,
                                                         float *__restrict__ Linv) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  TriBaseSmem &sm = *reinterpret_cast<TriBaseSmem *>(smem_raw);
  const int t = threadIdx.x;
  const int64_t o = (int64_t)blockIdx.x * GT;
  for (int f = t; f < GT * GT / 4; f += GT) {
    const int row = f >> 5, c4 = f & 31;
    const float4 v = *reinterpret_cast<const float4 *>(L + (o + row) * np + o + c4 * 4);
    sm.Ls[row][c4 * 4 + 0] = v.x;
    sm.Ls[row][c4 * 4 + 1] = v.y;
    sm.Ls[row][c4 * 4 + 2] = v.z;
    sm.Ls[row][c4 * 4 + 3] = v.w;
  }
  __syncthreads();
  const int i = t;
  for (int j = GT - 1; j > i; --j) sm.Xs[i][j] = 0.0f;
  // X[i][j] = (delta_ij - sum_{k=j+1..i} X[i][k] L[k][j]) / L[j][j]
  for (int j = i; j >= 0; --j) {
    float s0 = (j == i) ? 1.0f : 0.0f, s1 = 0.0f, s2 = 0.0f, s3 = 0.0f;
    int kk = j + 1;
    for (; kk + 3 <= i; kk += 4) {
      s0 = fmaf(-sm.Xs[i][kk + 0], sm.Ls[kk + 0][j], s0);
      s1 = fmaf(-sm.Xs[i][kk + 1], sm.Ls[kk + 1][j], s1);
      s2 = fmaf(-sm.Xs[i][kk + 2], sm.Ls[kk + 2][j], s2);
      s3 = fmaf(-sm.Xs[i][kk + 3], sm.Ls[kk + 3][j], s3);
    }
    for (; kk <= i; ++kk) s0 = fmaf(-sm.Xs[i][kk], sm.Ls[kk][j], s0);
    sm.Xs[i][j] = ((s0 + s1) + (s2 + s3)) / sm.Ls[j][j];
  }
  __syncthreads();
  for (int f = t; f < GT * GT / 4; f += GT) {
    const int row = f >> 5, c4 = f & 31;
    float4 v;
    v.x = sm.Xs[row][c4 * 4 + 0];
    v.y = sm.Xs[row][c4 * 4 + 1];
    v.z = sm.Xs[row][c4 * 4 + 2];
    v.w = sm.Xs[row][c4 * 4 + 3];
    *reinterpret_cast<float4 *>(Linv + (o + row) * np + o + c4 * 4) = v;
  }
}

// One doubling level: for every pair of adjacent b-blocks  [[A,0],[C,B]]^-1 = [[A^-1,0],[-B^-1 C A^-1, B^-1]].
//   PHASE 0:  T   = C * A^-1          (k >= column tile: A^-1 is lower triangular)
//   PHASE 1:  X21 = -B^-1 * T         (k <= row tile:    B^-1 is lower triangular)
template <int PHASE>
__global__ void __launch_bounds__(GTHREADS, 2) triinv_level_kernel(const float *__restrict__ L,
                                                                   float *__restrict__ Linv,
                                                                   float *__restrict__ T, int64_t np, int b) {
  __shared__ GemmSmem sm;
  const int64_t s = (int64_t)blockIdx.z * 2 * b;
  const int64_t s2 = min((int64_t)b, np - s - b);
  const int I = blockIdx.y, J = blockIdx.x;
  if (s2 <= 0 || (int64_t)I * GT >= s2) return;
  float acc[8][8];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[i][j] = 0.0f;
  const int64_t rbase = s + b + (int64_t)I * GT;   // global row of this tile
  const int64_t cbase = s + (int64_t)J * GT;       // global column of this tile
  if (PHASE == 0) {
    // A-op(r,k) = L[rbase+r][s+k];  B-op(c,k) = Linv[s+k][cbase+c]
    gemm_mainloop<true, false>(L + rbase * np + s, np, Linv + s * np + cbase, np, J * GT, b, acc, sm);
  } else {
    // A-op(r,k) = Linv[rbase+r][s+b+k];  B-op(c,k) = T[s+b+k][cbase+c]
    const int kend = (int)min((int64_t)(I + 1) * GT, s2);
    gemm_mainloop<true, false>(Linv + rbase * np + s + b, np, T + (s + b) * np + cbase, np, 0, kend, acc, sm);
  }
  float *out = (PHASE == 0) ? T : Linv;
  const float sgn = (PHASE == 0) ? 1.0f : -1.0f;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int64_t gi = rbase + gemm_row(i);
#pragma unroll
    for (int jh = 0; jh < 2; ++jh) {
      const int64_t gj = cbase + gemm_col(jh * 4);
      float4 v;
      v.x = sgn * acc[i][jh * 4 + 0];
      v.y = sgn * acc[i][jh * 4 + 1];
      v.z = sgn * acc[i][jh * 4 + 2];
      v.w = sgn * acc[i][jh * 4 + 3];
      *reinterpret_cast<float4 *>(out + gi * np + gj) = v;
    }
  }
}

int launch_tri_inverse(const float *L, int64_t np, float *Linv, float *tmp, cudaStream_t st) {
  if (np <= 0 || np % GT != 0) return HB_ERR_INVALID;
  static PerDevice once;
  bool fresh = false;
  const int dev = once.slot(&fresh);
  if (dev < 0) return HB_ERR_CUDA;
  if (fresh) {
    HB_CUDA(cudaFuncSetAttribute(triinv_base_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 (int)sizeof(TriBaseSmem)));
    once.done[dev] = true;
  }
  HB_CUDA(cudaMemsetAsync(Linv, 0, (size_t)np * np * sizeof(float), st));
  triinv_base_kernel<<<(int)(np / GT), GT, sizeof(TriBaseSmem), st>>>(L, np, Linv);
  count_launches(1);
  for (int64_t b = GT; b < np; b *= 2) {
    const int pairs = (int)ceil_div(np, 2 * b);
    dim3 grid((unsigned)(b / GT), (unsigned)(b / GT), (unsigned)pairs);
    triinv_level_kernel<0><<<grid, GTHREADS, 0, st>>>(L, Linv, tmp, np, (int)b);
    triinv_level_kernel<1><<<grid, GTHREADS, 0, st>>>(L, Linv, tmp, np, (int)b);
    count_launches(2);
  }
  HB_LAUNCH_CHECK("tri_inverse");
  return HB_OK;
}

// =============================================================================== refinement of L^-1 (prediction state)
// One Newton step  X <- X + X (I - L X)  on the explicit inverse X = L^-1 the posterior contracts with.  The residual
// R = I - L X is accumulated in fp64 (products of fp32 numbers are exact there), the correction X R in fp32 (R is
// ~1e-5 small, so its relative accuracy is ample).  After the step X differs from the exact inverse Lambda of the fp32
// factor L by at most u|X| + c u sqrt(NP) |X0||R| + |E0 L E0| (E0 = X0 - Lambda: exact Newton leaves -E0 L E0), with c
// below 1.2 measured: on well-conditioned factors every entry is within 0-2 ulp of the fp32 rounding of Lambda, against up
// to ~1e9 ulp (entries near zero) before the step; where cond_1(L) reaches 1e4 - 1e5 (d = 1, n = 4097, a factor after the
// jitter ladder) the quadratic term leaves tens to a thousand ulp on some entries (tests/test_gpu_fit_state.py).  The
// explicit inverse then carries about the error of the triangular solve of the reference (gp.py:148, gpytorch's cached
// prediction strategy), which matters exactly where sigma^2 = s - |L^-1 k*|^2 cancels (candidates on / next to training
// points).  Once per fit: ~n^3/3 DFMA + n^3/3 FFMA.
// the Cholesky works in place on the lower triangle: the strict upper part of the diagonal tiles still holds Khat
__global__ void __launch_bounds__(256) zero_upper_diag_kernel(float *__restrict__ L, int64_t np) {
  const int64_t o = (int64_t)blockIdx.x * GT;
  for (int f = threadIdx.x; f < GT * GT; f += blockDim.x) {
    const int r = f / GT, c = f - r * GT;
    if (c > r) L[(o + r) * np + o + c] = 0.0f;
  }
}

__global__ void __launch_bounds__(GTHREADS, 1) linv_resid_kernel(const float *__restrict__ L, const float *__restrict__ X,
                                                                 int64_t np, float *__restrict__ R) {
  __shared__ GemmSmem sm;
  int I, J;
  tri_decode((int)blockIdx.x, I, J);
  double acc[8][8];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[i][j] = 0.0;
  // (L X)[i][j] = sum_k L[i][k] X[k][j]:  L[i][k] = 0 for k > i,  X[k][j] = 0 for k < j
  gemm_mainloop<true, false, false, false, double>(L + (int64_t)I * GT * np, np, X + (int64_t)J * GT, np, J * GT, (I + 1) * GT,
                                                   acc, sm);
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int64_t gi = (int64_t)I * GT + gemm_row(i);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int64_t gj = (int64_t)J * GT + gemm_col(j);
      R[gi * np + gj] = (gi >= gj) ? (float)((gi == gj ? 1.0 : 0.0) - acc[i][j]) : 0.0f;
    }
  }
}

__global__ void __launch_bounds__(GTHREADS, 2) linv_corr_kernel(const float *__restrict__ X, const float *__restrict__ R,
                                                                int64_t np, float *__restrict__ out) {
  __shared__ GemmSmem sm;
  const int I = blockIdx.y, J = blockIdx.x;
  float acc[8][8];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[i][j] = 0.0f;
  if (I >= J) gemm_mainloop<true, false>(X + (int64_t)I * GT * np, np, R + (int64_t)J * GT, np, J * GT, (I + 1) * GT, acc, sm);
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int64_t gi = (int64_t)I * GT + gemm_row(i);
#pragma unroll
    for (int jh = 0; jh < 2; ++jh) {
      const int64_t gj = (int64_t)J * GT + gemm_col(jh * 4);
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (I >= J) {
        const float4 x = *reinterpret_cast<const float4 *>(X + gi * np + gj);
        v = make_float4(x.x + acc[i][jh * 4 + 0], x.y + acc[i][jh * 4 + 1], x.z + acc[i][jh * 4 + 2], x.w + acc[i][jh * 4 + 3]);
      }
      *reinterpret_cast<float4 *>(out + gi * np + gj) = v;
    }
  }
}

// Linv <- refined inverse; R and out: two [NP, NP] scratch matrices
int launch_linv_refine(float *L, float *Linv, int64_t np, float *R, float *out, cudaStream_t st) {
  if (np <= 0 || np % GT != 0) return HB_ERR_INVALID;
  const int nt = (int)(np / GT);
  zero_upper_diag_kernel<<<nt, 256, 0, st>>>(L, np);
  linv_resid_kernel<<<nt * (nt + 1) / 2, GTHREADS, 0, st>>>(L, Linv, np, R);
  linv_corr_kernel<<<dim3((unsigned)nt, (unsigned)nt), GTHREADS, 0, st>>>(Linv, R, np, out);
  HB_CUDA(cudaMemcpyAsync(Linv, out, (size_t)np * np * sizeof(float), cudaMemcpyDeviceToDevice, st));
  count_launches(3);
  HB_LAUNCH_CHECK("linv_refine");
  return HB_OK;
}

// =============================================================================== K^-1 = Linv^T Linv
__global__ void __launch_bounds__(GTHREADS, 2) kinv_kernel(const float *__restrict__ Linv, int64_t np,
                                                           float *__restrict__ Kinv) {
  __shared__ GemmSmem sm;
  int I, J;
  tri_decode((int)blockIdx.x, I, J);
  float acc[8][8];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[i][j] = 0.0f;
  // C[i][j] = sum_{k >= I*128} Linv[k][I*128+i] * Linv[k][J*128+j]
  gemm_mainloop<false, false>(Linv + (int64_t)I * GT, np, Linv + (int64_t)J * GT, np, I * GT, (int)np, acc, sm);
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int64_t gi = (int64_t)I * GT + gemm_row(i);
#pragma unroll
    for (int jh = 0; jh < 2; ++jh) {
      const int64_t gj = (int64_t)J * GT + gemm_col(jh * 4);
      float4 v;
      v.x = acc[i][jh * 4 + 0];
      v.y = acc[i][jh * 4 + 1];
      v.z = acc[i][jh * 4 + 2];
      v.w = acc[i][jh * 4 + 3];
      *reinterpret_cast<float4 *>(Kinv + gi * np + gj) = v;
    }
  }
}

int launch_kinv(const float *Linv, int64_t np, float *Kinv, cudaStream_t st) {
  if (np <= 0 || np % GT != 0) return HB_ERR_INVALID;
  const int nt = (int)(np / GT);
  kinv_kernel<<<nt * (nt + 1) / 2, GTHREADS, 0, st>>>(Linv, np, Kinv);
  count_launches(1);
  HB_LAUNCH_CHECK("kinv");
  return HB_OK;
}

// =============================================================================== alpha, quad, logdet
// v = Linv r  (warp per row, fp64 accumulate; r = y - c on the first n entries, 0 on the pad)
__global__ void __launch_bounds__(256) gemv_rows_kernel(const float *__restrict__ Linv, const float *__restrict__ y,
                                                        const float *__restrict__ hyp, int64_t n, int64_t np,
                                                        double *__restrict__ v, int64_t wss) {
  Linv = slice(Linv, wss, blockIdx.z);   // output (Batch): targets are n apart
  y += (int64_t)blockIdx.z * n;
  hyp = slice(hyp, wss, blockIdx.z);
  v = slice(v, wss, blockIdx.z);
  const int warp = (int)((blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5);
  const int lane = threadIdx.x & 31;
  if (warp >= np) return;
  const float c = hyp[1];
  const float *row = Linv + (int64_t)warp * np;
  double s = 0.0;
  const int kend = min((int64_t)warp + 1, n);
  for (int k4 = lane * 4; k4 < kend; k4 += 128) {
    const float4 l = *reinterpret_cast<const float4 *>(row + k4);
    const float lv[4] = {l.x, l.y, l.z, l.w};
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int k = k4 + u;
      if (k < kend) s += (double)lv[u] * (double)(y[k] - c);
    }
  }
  s = warp_sum_d(s);
  if (lane == 0) v[warp] = s;
}

// partial[rs][j] = sum_{i in row slab rs, i >= j} Linv[i][j] v[i]
constexpr int GEMVT_ROWS = 64;  // rows per slab
__global__ void __launch_bounds__(128) gemv_cols_kernel(const float *__restrict__ Linv, const double *__restrict__ v,
                                                        int64_t np, double *__restrict__ partial, int64_t wss) {
  Linv = slice(Linv, wss, blockIdx.z);
  v = slice(v, wss, blockIdx.z);
  partial = slice(partial, wss, blockIdx.z);
  const int j = blockIdx.x * 128 + threadIdx.x;
  const int64_t i0 = (int64_t)blockIdx.y * GEMVT_ROWS;
  double s = 0.0;
  if (i0 + GEMVT_ROWS > (int64_t)blockIdx.x * 128) {  // slab intersects rows >= first column of this block
    // entries above the diagonal (i < j) are exact zeros in Linv, so the whole slab can be summed without a branch;
    // 8 independent loads in flight per thread instead of one dependent load per row
    double acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
#pragma unroll 1
    for (int64_t i = i0; i < i0 + GEMVT_ROWS; i += 8) {
      float l[8];
#pragma unroll
      for (int u = 0; u < 8; ++u) l[u] = Linv[(i + u) * np + j];
#pragma unroll
      for (int u = 0; u < 8; ++u) acc[u] += (double)l[u] * v[i + u];
    }
    s = ((acc[0] + acc[1]) + (acc[2] + acc[3])) + ((acc[4] + acc[5]) + (acc[6] + acc[7]));
  }
  partial[(int64_t)blockIdx.y * np + j] = s;
}

__global__ void __launch_bounds__(256) solve_finish_kernel(const float *__restrict__ L, const double *__restrict__ v,
                                                           const double *__restrict__ partial, int64_t n,
                                                           int64_t np, int nslab, float *__restrict__ alpha,
                                                           double *__restrict__ scal, int64_t wss) {
  L = slice(L, wss, blockIdx.z);
  v = slice(v, wss, blockIdx.z);
  partial = slice(partial, wss, blockIdx.z);
  alpha = slice(alpha, wss, blockIdx.z);
  scal = slice(scal, wss, blockIdx.z);
  // alpha (every block handles a strip), block 0 additionally reduces quad and logdet
  const int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (j < np) {
    double s = 0.0;
    for (int r = 0; r < nslab; ++r) s += partial[(int64_t)r * np + j];
    alpha[j] = (j < n) ? (float)s : 0.0f;
  }
  if (blockIdx.x == 0) {
    __shared__ double sq[256], sl[256];
    double q = 0.0, ld = 0.0;
    for (int64_t i = threadIdx.x; i < n; i += blockDim.x) {
      q += v[i] * v[i];
      ld += log((double)L[i * np + i]);
    }
    sq[threadIdx.x] = q;
    sl[threadIdx.x] = ld;
    __syncthreads();
    for (int o = 128; o > 0; o >>= 1) {
      if ((int)threadIdx.x < o) {
        sq[threadIdx.x] += sq[threadIdx.x + o];
        sl[threadIdx.x] += sl[threadIdx.x + o];
      }
      __syncthreads();
    }
    if (threadIdx.x == 0) {
      scal[0] = sq[0];
      scal[1] = 2.0 * sl[0];
    }
  }
}

size_t solve_ws_bytes(int64_t np) { return (size_t)np * sizeof(double) * (1 + (size_t)(np / GEMVT_ROWS)); }

int launch_solve_logdet(const float *L, const float *Linv, const float *y, int64_t n, int64_t np, const float *hyp,
                        float *alpha, double *scal, void *ws, cudaStream_t st, const Batch &bt) {
  if (np <= 0 || np % GT != 0 || n <= 0 || n > np) return HB_ERR_INVALID;
  double *v = reinterpret_cast<double *>(ws);
  double *partial = v + np;
  const int nslab = (int)(np / GEMVT_ROWS);
  const unsigned nz = (unsigned)bt.nout;
  gemv_rows_kernel<<<dim3((unsigned)ceil_div(np * 32, 256), 1, nz), 256, 0, st>>>(Linv, y, hyp, n, np, v, bt.ws);
  gemv_cols_kernel<<<dim3((unsigned)(np / 128), (unsigned)nslab, nz), 128, 0, st>>>(Linv, v, np, partial, bt.ws);
  solve_finish_kernel<<<dim3((unsigned)ceil_div(np, 256), 1, nz), 256, 0, st>>>(L, v, partial, n, np, nslab, alpha, scal, bt.ws);
  count_launches(3);
  HB_LAUNCH_CHECK("solve_logdet");
  return HB_OK;
}

}  // namespace hb
