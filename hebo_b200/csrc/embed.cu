// Bound violation of a random linear embedding (HEBO_Embedding with clip = False, SURVEY §8 "HEBO_Embedding"): the fourth
// MACE_Embedding column of HEBO/hebo/optimizers/hebo_embedding.py:88-89,
//
//     G[i] = sum_j max(|sum_k Y[i,k] B[k,j]| - 1, 0),      Y [m, e] candidates in the embedding, B [e, D] projection,
//
// without forming the [m, D] projection.  The work is a GEMM followed by a row reduction, 2 m e D flop; with e <= a few
// dozen the operand tiles are re-read from L1/L2 and the kernel is bound by FP32 FMA issue on the SIMT pipe.
//
// embed_violation_kernel: CTA (bx, s) owns rows [128 bx, 128 bx + 128) and the column blocks s, s + S, s + 2S, ... of 128
// columns (S = min(#column blocks, 32) splits of D, so m = 10 000 still gives 79 S CTAs).  256 threads in a 16 x 16 grid
// each hold an 8 x 8 register tile of the projection (rows ty*4 + {0..3} and 64 + ty*4 + {0..3}, columns likewise with
// tx, so the float4 shared-memory reads are conflict-free).  e is streamed through shared memory 16 at a time (any
// 1 <= e <= HB_MAX_FEATURES; shared memory does not grow with e), double-buffered with cp.async so the next tile loads
// during the FMAs without passing through registers.  Each projected coordinate is one fp32 FMA chain over k ascending.
// When a column block is complete each thread sums its 8 clamped columns of a row in fp32, in column order, and adds that
// to an fp64 row sum; the 16 threads of a row then reduce in a fixed butterfly and the CTA writes one fp64 partial per
// (split, row).  A NaN coordinate propagates into G as it does through the reference's clamp (torch.clamp keeps NaN), so
// a candidate with NaN in its row of Y (or a NaN in B) is never feasible.
// embed_violation_sum_kernel adds the S partials of a row in split order in fp64 and rounds once to fp32.
// No float atomics, and the order of every sum is fixed by (m, e, D): G is bit-identical from run to run.
#include <algorithm>

#include "kernels.h"

namespace hb {

constexpr int EV_BM = 128, EV_BN = 128, EV_EK = 16, EV_THREADS = 256, EV_SPLIT = 32;

static int64_t ev_splits(int64_t D) { return std::min<int64_t>(ceil_div(D, EV_BN), EV_SPLIT); }

// 4-byte global -> shared copy that bypasses the register file; ok = false stores 0 (src-size 0 reads nothing)
__device__ __forceinline__ void cp_async4(float *dst, const float *src, bool ok) {
  const unsigned d = (unsigned)__cvta_generic_to_shared(dst);
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;\n" ::"r"(d), "l"(src), "r"(ok ? 4 : 0));
}

__global__ void __launch_bounds__(EV_THREADS, 2) embed_violation_kernel(const float *__restrict__ Y, int64_t m, int e,
                                                                        const float *__restrict__ B, int64_t D, int S,
                                                                        double *__restrict__ part) {
  __shared__ __align__(16) float Ys[2][EV_EK][EV_BM + 4];   // Y tile, transposed (k, row); the pad spreads the transposing stores
  __shared__ __align__(16) float Bs[2][EV_EK][EV_BN];
  const int tid = threadIdx.x, tx = tid % 16, ty = tid / 16;
  const int64_t row0 = (int64_t)blockIdx.x * EV_BM;
  const int split = blockIdx.y;
  const int64_t ncb = (ceil_div(D, EV_BN) - split + S - 1) / S;   // column blocks split, split + S, ...
  const int nk = (int)ceil_div(e, EV_EK);
  const int64_t nsteps = ncb * nk;
  // step = (column block, e chunk) -> shared buffer `buf`, asynchronously; zeros outside [0, m) x [0, e) x [0, D)
  // thread tid copies Y[row0 + tid/16 + 16 t, k0 + tid%16] (16 consecutive k of a row per 16 threads) and
  // B[k0 + tid/128 + 2 t, col0 + tid%128] (128 consecutive columns per 128 threads), t = 0..7
  const int yr = tid / EV_EK, yk = tid % EV_EK, bk = tid / EV_BN, bc = tid % EV_BN;
  auto issue = [&](int64_t step, int buf) {
    const int64_t col = (split + (step / nk) * S) * EV_BN + bc;
    const int k0 = (int)(step % nk) * EV_EK;
#pragma unroll 1
    for (int t = 0; t < 8; ++t) {
      const int64_t row = row0 + yr + 16 * t;
      const bool oky = row < m && k0 + yk < e;
      cp_async4(&Ys[buf][yk][yr + 16 * t], oky ? Y + row * e + k0 + yk : Y, oky);
      const int kb = k0 + bk + 2 * t;
      const bool okb = col < D && kb < e;
      cp_async4(&Bs[buf][bk + 2 * t][bc], okb ? B + (int64_t)kb * D + col : B, okb);
    }
    asm volatile("cp.async.commit_group;\n" ::);
  };
  float acc[8][8];
  double rsum[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    rsum[i] = 0.0;
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[i][j] = 0.0f;
  }
  issue(0, 0);
  for (int64_t step = 0; step < nsteps; ++step) {
    const int buf = (int)(step & 1);
    if (step + 1 < nsteps) {
      issue(step + 1, buf ^ 1);   // its buffer was last read in step - 1, before that step's closing barrier
      asm volatile("cp.async.wait_group 1;\n" ::);
    } else {
      asm volatile("cp.async.wait_group 0;\n" ::);
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < EV_EK; ++k) {
      const float4 a0 = *reinterpret_cast<const float4 *>(&Ys[buf][k][ty * 4]);
      const float4 a1 = *reinterpret_cast<const float4 *>(&Ys[buf][k][64 + ty * 4]);
      const float4 b0 = *reinterpret_cast<const float4 *>(&Bs[buf][k][tx * 4]);
      const float4 b1 = *reinterpret_cast<const float4 *>(&Bs[buf][k][64 + tx * 4]);
      const float a[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
      const float b[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    if ((step + 1) % nk == 0) {   // column block complete: padded rows / columns project to 0 and add nothing
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        float s = 0.0f;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const float over = fabsf(acc[i][j]) - 1.0f;
          s += (over > 0.0f || over != over) ? over : 0.0f;   // max(., 0) that keeps NaN
          acc[i][j] = 0.0f;
        }
        rsum[i] += (double)s;
      }
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    double v = rsum[i];
#pragma unroll
    for (int o = 8; o > 0; o >>= 1) v += __shfl_xor_sync(0xFFFFFFFFu, v, o);   // the 16 tx lanes of a row
    const int64_t row = row0 + (i < 4 ? ty * 4 + i : 64 + ty * 4 + i - 4);
    if (tx == 0 && row < m) part[(int64_t)split * m + row] = v;
  }
}

__global__ void embed_violation_sum_kernel(const double *__restrict__ part, int64_t m, int S, float *__restrict__ G) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= m) return;
  double s = 0.0;
  for (int p = 0; p < S; ++p) s += part[(int64_t)p * m + i];
  G[i] = (float)s;
}

int64_t embed_violation_ws_query(int64_t m, int64_t e, int64_t D) {
  if (m < 1 || e < 1 || e > HB_MAX_FEATURES || D < 1 || m > ((int64_t)1 << 40) || D > ((int64_t)1 << 40)) return -1;
  return round_up(ev_splits(D) * m * (int64_t)sizeof(double), 256);
}

int launch_embed_violation(const float *Y, int64_t m, int64_t e, const float *B, int64_t D, float *G, void *ws, int64_t ws_bytes,
                           cudaStream_t st) {
  const int64_t need = embed_violation_ws_query(m, e, D);
  if (need < 0 || ws_bytes < need) return HB_ERR_INVALID;
  const int S = (int)ev_splits(D);
  double *part = static_cast<double *>(ws);
  embed_violation_kernel<<<dim3((unsigned)ceil_div(m, EV_BM), (unsigned)S), EV_THREADS, 0, st>>>(Y, m, (int)e, B, D, S, part);
  embed_violation_sum_kernel<<<(unsigned)ceil_div(m, 256), 256, 0, st>>>(part, m, S, G);
  count_launches(2);
  HB_LAUNCH_CHECK("embed_violation");
  return HB_OK;
}

}  // namespace hb
