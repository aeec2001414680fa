// Blocked Cholesky factorisation of the padded [NP, NP] fp32 Gram matrix (lower, in place).
//
//   outer blocks of 512 columns.  ONE kernel per outer block factors the whole block column [cb, ce) x [cb, NP):
//     chol_block64_kernel : a left-looking TILE DAG over 64x64 tiles.  Task = "finish tile (i, j)":
//                             S = A(i,j) - sum_{k < j, k in this block} L(i,k) L(j,k)^T     (FP32 SIMT, 4x4 per thread)
//                             i == j : in-register Cholesky of the tile                    (sweep64)
//                             i >  j : X = S L(j,j)^-T by row substitution                 (trsm64)
//                           Tasks are numbered column-major and dealt round-robin to the CTAs of a co-resident
//                           (cooperative) grid, one CTA per SM; a finished tile publishes a release flag, consumers
//                           spin on an acquire load.  Every dependency of a task has a smaller number and every CTA
//                           works in increasing order, so the smallest unfinished task can always run: no deadlock.
//                           Accumulators live in registers across the k steps and every tile is written exactly once.
//                           The block costs its critical path -- per 64 columns: potrf -> trsm of the one tile below
//                           -> one K = 64 update of the next diagonal tile -- with the last two links fused into the
//                           diagonal task (the trsm result feeds the update straight from shared memory).
//   after the block     : A[r, c >= ce] -= P P^T  with K = 512 -- the one large dense contraction of the
//                         factorisation: wgmma 3xTF32 (fit_tc.cu) in the fit loop, FP32 SIMT core otherwise.
// This is what gpytorch's psd_safe_cholesky does through LAPACK potrf for HEBO/hebo/models/gp/gp.py:112-113,148.
// `info` follows LAPACK: j > 0 = leading minor j not positive definite (first failing pivot wins).
#include <limits.h>

#include "gemm_core.cuh"
#include "kernels.h"

namespace hb {

constexpr int OUTER = 512;             // outer block width
constexpr int TS = 64;                 // tile size of the block-column DAG
constexpr int MAXBC64 = OUTER / TS;    // tile columns per outer block
constexpr int SP64 = TS + 4;           // shared-tile pitch (16-byte aligned, staggers banks)

__device__ __forceinline__ int ld_acquire(const int *p) {
  int v;
  asm volatile("ld.acquire.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ float rsqrt_approx(float x) {   // MUFU.RSQ, 2 ulp
  float r;
  asm("rsqrt.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
  return r;
}
__device__ __forceinline__ void st_release(int *p, int v) {
  asm volatile("st.release.gpu.global.s32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
// block-wide wait for up to two tile flags
__device__ __forceinline__ void wait_tiles(const int *f0, const int *f1, int token) {
  if (threadIdx.x == 0) {
    while (ld_acquire(f0) != token) __nanosleep(32);
    if (f1 != f0)
      while (ld_acquire(f1) != token) __nanosleep(32);
  }
  __syncthreads();
}

// In-register Cholesky of a 64x64 tile distributed 4x4 per thread (ti = row block, tc = column block; the 16 threads
// of a column block are a half-warp), right-looking in steps of 4 columns.  Step jb: the warp owning column block jb
// fetches the 4x4 diagonal block by shuffles, every lane factors it redundantly (no divergence), the half-warp turns
// its 4 columns into L (rows above the diagonal block := 0) and publishes them in shared memory -- ONE barrier per
// 4 pivots -- and the column blocks to the right apply the rank-4 update.  On return S holds L (upper part zero).
// `deferred` (may be null): a tile flag whose global stores were issued before the call; the last warp releases it after
// the first barrier, hiding the fence behind the first panel chains (which run in warp 0).
__device__ __forceinline__ void sweep64(float (&S)[4][4], float *Lp, int *fail, int fail_base, int warp, int lane, int ti,
                                        int tc, int *deferred, int token) {
#pragma unroll 1
  for (int jb = 0; jb < 16; ++jb) {
    // published panel, column-major: P[k * TS + row], k = 0..3 (a thread's 4 rows are one conflict-free LDS.128)
    float *P = Lp + (jb & 1) * 4 * TS;
    if (warp == (jb >> 1)) {
      const int src = ((jb & 1) << 4) | jb;   // lane of (ti = jb, tc = jb)
      const unsigned FULL = 0xffffffffu;
      const float d00 = __shfl_sync(FULL, S[0][0], src);
      const float d10 = __shfl_sync(FULL, S[1][0], src), d11 = __shfl_sync(FULL, S[1][1], src);
      const float d20 = __shfl_sync(FULL, S[2][0], src), d21 = __shfl_sync(FULL, S[2][1], src);
      const float d22 = __shfl_sync(FULL, S[2][2], src);
      const float d30 = __shfl_sync(FULL, S[3][0], src), d31 = __shfl_sync(FULL, S[3][1], src);
      const float d32 = __shfl_sync(FULL, S[3][2], src), d33 = __shfl_sync(FULL, S[3][3], src);
      const float r0 = rsqrt_approx(d00);
      const float l00 = d00 * r0, l10 = d10 * r0, l20 = d20 * r0, l30 = d30 * r0;
      const float p1 = fmaf(-l10, l10, d11);
      const float r1 = rsqrt_approx(p1);
      const float l11 = p1 * r1;
      const float l21 = fmaf(-l20, l10, d21) * r1, l31 = fmaf(-l30, l10, d31) * r1;
      const float p2 = fmaf(-l21, l21, fmaf(-l20, l20, d22));
      const float r2 = rsqrt_approx(p2);
      const float l22 = p2 * r2;
      const float l32 = fmaf(-l31, l21, fmaf(-l30, l20, d32)) * r2;
      const float p3 = fmaf(-l32, l32, fmaf(-l31, l31, fmaf(-l30, l30, d33)));
      const float r3 = rsqrt_approx(p3);
      const float l33 = p3 * r3;
      if (lane == src) {
        int f = -1;
        if (!(d00 > 0.0f)) f = 0;
        else if (!(p1 > 0.0f)) f = 1;
        else if (!(p2 > 0.0f)) f = 2;
        else if (!(p3 > 0.0f)) f = 3;
        if (f >= 0) atomicMin(fail, fail_base + 4 * jb + f);
      }
      if (tc == jb) {
        const float Ld[4][4] = {{l00, 0.f, 0.f, 0.f}, {l10, l11, 0.f, 0.f}, {l20, l21, l22, 0.f}, {l30, l31, l32, l33}};
#pragma unroll
        for (int a = 0; a < 4; ++a) {
          float x0 = S[a][0] * r0;
          float x1 = fmaf(-x0, l10, S[a][1]) * r1;
          float x2 = fmaf(-x1, l21, fmaf(-x0, l20, S[a][2])) * r2;
          float x3 = fmaf(-x2, l32, fmaf(-x1, l31, fmaf(-x0, l30, S[a][3]))) * r3;
          if (ti == jb) {
            x0 = Ld[a][0]; x1 = Ld[a][1]; x2 = Ld[a][2]; x3 = Ld[a][3];
          } else if (ti < jb) {
            x0 = x1 = x2 = x3 = 0.0f;
          }
          S[a][0] = x0; S[a][1] = x1; S[a][2] = x2; S[a][3] = x3;
        }
#pragma unroll
        for (int k = 0; k < 4; ++k)
          *reinterpret_cast<float4 *>(P + k * TS + 4 * ti) = make_float4(S[0][k], S[1][k], S[2][k], S[3][k]);
      }
    }
    __syncthreads();
    if (jb == 0 && deferred && threadIdx.x == GTHREADS - 32) {
      __threadfence();
      st_release(deferred, token);
    }
    if (tc > jb) {   // the panel's own columns and the finished column blocks are final
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const float4 v = *reinterpret_cast<const float4 *>(P + k * TS + 4 * ti);
        const float4 w = *reinterpret_cast<const float4 *>(P + k * TS + 4 * tc);
        const float lr[4] = {v.x, v.y, v.z, v.w};
        const float lc[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
        for (int a = 0; a < 4; ++a)
#pragma unroll
          for (int b = 0; b < 4; ++b) S[a][b] = fmaf(-lr[a], lc[b], S[a][b]);
      }
    }
  }
}

struct Block64Smem {
  __align__(16) float T[TS][SP64];    // the tile being finished (row-major)
  __align__(16) float Lt[TS][SP64];   // trsm: Lt[p][c] = L(j,j)[c][p];  potrf: the published 4-column panels (2 KiB)
  __align__(16) float At[TS][SP64];   // update operands, transposed: At[p][r] = L(i,k)[r][p], Bt[p][c] = L(j,k)[c][p]
  __align__(16) float Bt[TS][SP64];
  float rinv[TS];
  int fail;
};
constexpr int BLOCK64_SMEM = 120 * 1024;   // > half an SM: one CTA per SM, the critical tasks never share an FMA pipe

// stage a 64x64 global tile transposed into shared memory (lane <-> row => conflict-free stores)
__device__ __forceinline__ void stage_transposed(const float *__restrict__ G, int64_t ld, float (&S)[TS][SP64]) {
  const int t = threadIdx.x;
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const int f = t + q * GTHREADS;
    const int row = f & (TS - 1), c4 = f >> 6;
    const float4 v = __ldcg(reinterpret_cast<const float4 *>(G + (int64_t)row * ld + c4 * 4));
    S[c4 * 4 + 0][row] = v.x;
    S[c4 * 4 + 1][row] = v.y;
    S[c4 * 4 + 2][row] = v.z;
    S[c4 * 4 + 3][row] = v.w;
  }
}

// Forward substitution a <- a L^-T of one 64-wide row shared by a lane PAIR (lanes 2r, 2r+1): half h owns the float4
// column groups g with (g & 1) == h, stored locally as a[4 * (g >> 1) + q].  The owner of pivot column p forms
// x_p and hands it to its partner with one shuffle; each half then updates only its own columns, so the FMA work per
// thread halves and a 64-row tile keeps four warps busy.  Ltp[p * PITCH + c] = L[c][p].
template <int PITCH>
__device__ __forceinline__ void sub64_pair(float (&a)[32], int h, int lane, const float *__restrict__ Ltp,
                                           const float *__restrict__ rinv) {
#pragma unroll
  for (int p = 0; p < 64; ++p) {
    const int gp = p >> 2, own = gp & 1, lgp = gp >> 1, q0 = p & 3;
    const float xc = a[4 * lgp + q0] * rinv[p];
    const float x = __shfl_sync(0xffffffffu, xc, (lane & ~1) | own);
    if (h == own) a[4 * lgp + q0] = x;
    {   // the local group that holds (or neighbours) the pivot column
      const float4 l = *reinterpret_cast<const float4 *>(Ltp + p * PITCH + 4 * (2 * lgp + h));
      const bool full = h > own, mine = h == own;
      if (full || (mine && 0 > q0)) a[4 * lgp + 0] = fmaf(-x, l.x, a[4 * lgp + 0]);
      if (full || (mine && 1 > q0)) a[4 * lgp + 1] = fmaf(-x, l.y, a[4 * lgp + 1]);
      if (full || (mine && 2 > q0)) a[4 * lgp + 2] = fmaf(-x, l.z, a[4 * lgp + 2]);
      if (full || (mine && 3 > q0)) a[4 * lgp + 3] = fmaf(-x, l.w, a[4 * lgp + 3]);
    }
#pragma unroll
    for (int lg = lgp + 1; lg < 8; ++lg) {
      const float4 l = *reinterpret_cast<const float4 *>(Ltp + p * PITCH + 4 * (2 * lg + h));
      a[4 * lg + 0] = fmaf(-x, l.x, a[4 * lg + 0]);
      a[4 * lg + 1] = fmaf(-x, l.y, a[4 * lg + 1]);
      a[4 * lg + 2] = fmaf(-x, l.z, a[4 * lg + 2]);
      a[4 * lg + 3] = fmaf(-x, l.w, a[4 * lg + 3]);
    }
  }
}

// X = T L^-T for the 64 rows in sm.T (factor in sm.Lt / sm.rinv), in place; threads < 128 (two per row).
// TO_AT: also leave X transposed in sm.At (the operand layout of the update loop).
template <bool TO_AT>
__device__ __forceinline__ void trsm64(Block64Smem &sm) {
  const int t = threadIdx.x;
  if (t >= 2 * TS) return;
  const int r = t >> 1, h = t & 1, lane = t & 31;
  float a[32];
#pragma unroll
  for (int lg = 0; lg < 8; ++lg) {
    const float4 v = *reinterpret_cast<const float4 *>(&sm.T[r][4 * (2 * lg + h)]);
    a[4 * lg + 0] = v.x; a[4 * lg + 1] = v.y; a[4 * lg + 2] = v.z; a[4 * lg + 3] = v.w;
  }
  sub64_pair<SP64>(a, h, lane, &sm.Lt[0][0], sm.rinv);
#pragma unroll
  for (int lg = 0; lg < 8; ++lg) {
    *reinterpret_cast<float4 *>(&sm.T[r][4 * (2 * lg + h)]) = make_float4(a[4 * lg + 0], a[4 * lg + 1], a[4 * lg + 2], a[4 * lg + 3]);
    if (TO_AT) {
#pragma unroll
      for (int q = 0; q < 4; ++q) sm.At[4 * (2 * lg + h) + q][r] = a[4 * lg + q];
    }
  }
}

// S -= A B^T for one staged operand pair: S[a][b] -= sum_p At[p][4 ti + a] Bt[p][4 tc + b]
__device__ __forceinline__ void update64(float (&S)[4][4], const float (&At)[TS][SP64], const float (&Bt)[TS][SP64], int ti, int tc) {
#pragma unroll 8
  for (int p = 0; p < TS; ++p) {
    const float4 av = *reinterpret_cast<const float4 *>(&At[p][4 * ti]);
    const float4 bv = *reinterpret_cast<const float4 *>(&Bt[p][4 * tc]);
    const float a4[4] = {av.x, av.y, av.z, av.w};
    const float b4[4] = {bv.x, bv.y, bv.z, bv.w};
#pragma unroll
    for (int a = 0; a < 4; ++a)
#pragma unroll
      for (int b = 0; b < 4; ++b) S[a][b] = fmaf(-a4[a], b4[b], S[a][b]);
  }
}

__device__ __forceinline__ void load_tile4x4(float (&S)[4][4], const float *__restrict__ G, int64_t ld, int ti, int tc) {
#pragma unroll
  for (int a = 0; a < 4; ++a) {
    const float4 c = __ldcg(reinterpret_cast<const float4 *>(G + (int64_t)(4 * ti + a) * ld + 4 * tc));
    S[a][0] = c.x; S[a][1] = c.y; S[a][2] = c.z; S[a][3] = c.w;
  }
}
__device__ __forceinline__ void tile4x4_to_smem(const float (&S)[4][4], float (&T)[TS][SP64], int ti, int tc) {
#pragma unroll
  for (int a = 0; a < 4; ++a)
    *reinterpret_cast<float4 *>(&T[4 * ti + a][4 * tc]) = make_float4(S[a][0], S[a][1], S[a][2], S[a][3]);
}
// coalesced store of sm.T to a global tile
__device__ __forceinline__ void store_tile(Block64Smem &sm, float *__restrict__ G, int64_t ld) {
  const int t = threadIdx.x;
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const int f = t + q * GTHREADS;
    const int row = f >> 4, c4 = f & 15;
    *reinterpret_cast<float4 *>(G + (int64_t)row * ld + c4 * 4) = *reinterpret_cast<const float4 *>(&sm.T[row][c4 * 4]);
  }
}
// ... then publish its flag (all threads must call)
__device__ __forceinline__ void publish_tile(Block64Smem &sm, float *__restrict__ G, int64_t ld, int *flag, int token) {
  const int t = threadIdx.x;
  store_tile(sm, G, ld);
  __syncthreads();   // all stores issued (and sm.T free again)
  if (t == 0) {
    __threadfence();
    st_release(flag, token);
  }
}
// wait for the diagonal factor L(j,j), stage it transposed with its reciprocal diagonal
__device__ __forceinline__ void stage_factor(Block64Smem &sm, const float *__restrict__ A, int64_t np, int j, const int *flag,
                                             int token) {
  wait_tiles(flag, flag, token);   // (its barrier also orders earlier sm.T / sm.Lt traffic)
  stage_transposed(A + (int64_t)j * TS * np + (int64_t)j * TS, np, sm.Lt);
  __syncthreads();
  if (threadIdx.x < TS) sm.rinv[threadIdx.x] = 1.0f / sm.Lt[threadIdx.x][threadIdx.x];
  __syncthreads();
}

// Task numbering inside a block column (column-major, jl = 0 .. nbc-1, j = jb0 + jl):
//   D(j)            : composite = sub-diagonal tile (j, j-1) [jl >= 1] followed by the diagonal tile (j, j), both
//                     finished by ONE CTA so that the trsm result feeds the diagonal update straight from shared memory
//   R(i, j), i >= j+2 (i >= j+1 in the last column of the block): the other tiles of column j
//   Batch: the tasks of the `nout` outputs are interleaved, global task = task * nout + output, so the pivot chains of all
//   outputs advance together.  A task only depends on smaller tasks of its own output, which have smaller global numbers:
//   the argument above still holds.  A, the flags and info of output b live in its workspace slice (wss bytes apart).
__global__ void __launch_bounds__(GTHREADS, 1) chol_block64_kernel(float *__restrict__ A0, int64_t np, int jb0, int nbc,
                                                                   int ntasks, int *__restrict__ flags0, int token,
                                                                   int32_t *info0, int nout, int64_t wss) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  Block64Smem &sm = *reinterpret_cast<Block64Smem *>(smem_raw);
  const int t = threadIdx.x;
  const int warp = t >> 5, lane = t & 31;
  const int tc = 2 * warp + (lane >> 4), ti = lane & 15;   // 4x4 micro-tile: rows 4 ti.., cols 4 tc..
  const int nt = (int)(np / TS);
  for (int gtask = blockIdx.x; gtask < ntasks * nout; gtask += gridDim.x) {
    const int task = gtask / nout, ob = gtask - task * nout;
    float *__restrict__ A = slice(A0, wss, ob);
    int *__restrict__ flags = slice(flags0, wss, ob);
    int32_t *info = slice(info0, wss, ob);
    int jl = 0, tt = task;
    for (;;) {
      const int j_ = jb0 + jl;
      const int cnt = 1 + (nt - (j_ + (jl == nbc - 1 ? 1 : 2)) > 0 ? nt - (j_ + (jl == nbc - 1 ? 1 : 2)) : 0);
      if (tt < cnt) break;
      tt -= cnt;
      ++jl;
    }
    const int j = jb0 + jl;
    const int64_t col = (int64_t)j * TS;
    if (t == 0) sm.fail = INT_MAX;
    if (tt == 0) {
      // ------------------------------------------------------------------ D(j)
      float S[4][4], S2[4][4];
      float *Cd = A + (int64_t)j * TS * np + col;
      load_tile4x4(S, Cd, np, ti, tc);
      if (jl >= 1) {
        float *Cs = Cd - TS;   // tile (j, j-1)
        load_tile4x4(S2, Cs, np, ti, tc);
        for (int kl = 0; kl + 1 < jl; ++kl) {
          wait_tiles(flags + j * MAXBC64 + kl, flags + (j - 1) * MAXBC64 + kl, token);
          stage_transposed(A + (int64_t)j * TS * np + (int64_t)(jb0 + kl) * TS, np, sm.At);
          stage_transposed(A + (int64_t)(j - 1) * TS * np + (int64_t)(jb0 + kl) * TS, np, sm.Bt);
          __syncthreads();
          update64(S2, sm.At, sm.Bt, ti, tc);
          update64(S, sm.At, sm.At, ti, tc);
        }
        tile4x4_to_smem(S2, sm.T, ti, tc);
        stage_factor(sm, A, np, j - 1, flags + (j - 1) * MAXBC64 + (jl - 1), token);
        trsm64<true>(sm);
        __syncthreads();
        store_tile(sm, Cs, np);                       // L(j, j-1): its flag is released inside the sweep
        update64(S, sm.At, sm.At, ti, tc);            // the one update on the critical path, straight from smem
      }
      sweep64(S, &sm.Lt[0][0], &sm.fail, j * TS, warp, lane, ti, tc, jl >= 1 ? flags + j * MAXBC64 + (jl - 1) : nullptr, token);
      tile4x4_to_smem(S, sm.T, ti, tc);
      __syncthreads();
      if (t == 0 && sm.fail != INT_MAX) atomicCAS(info, 0, sm.fail + 1);
      publish_tile(sm, Cd, np, flags + j * MAXBC64 + jl, token);
    } else {
      // ------------------------------------------------------------------ R(i, j)
      const int i = j + (jl == nbc - 1 ? 1 : 2) + (tt - 1);
      float *Cg = A + (int64_t)i * TS * np + col;
      float S[4][4];
      load_tile4x4(S, Cg, np, ti, tc);
      for (int kl = 0; kl < jl; ++kl) {
        wait_tiles(flags + i * MAXBC64 + kl, flags + j * MAXBC64 + kl, token);   // (its barrier also frees At/Bt)
        stage_transposed(A + (int64_t)i * TS * np + (int64_t)(jb0 + kl) * TS, np, sm.At);
        stage_transposed(A + (int64_t)j * TS * np + (int64_t)(jb0 + kl) * TS, np, sm.Bt);
        __syncthreads();
        update64(S, sm.At, sm.Bt, ti, tc);
      }
      tile4x4_to_smem(S, sm.T, ti, tc);
      stage_factor(sm, A, np, j, flags + j * MAXBC64 + jl, token);
      trsm64<false>(sm);
      __syncthreads();
      publish_tile(sm, Cg, np, flags + i * MAXBC64 + jl, token);
    }
  }
}

// ------------------------------------------------------------------------------------------------------------------
// Base case of the tensor-core triangular inverse (fit_tc.cu): one CTA inverts one 128x128 diagonal block of L,
//   L = [A 0; B C]  ->  L^-1 = [A^-1 0; -C^-1 B A^-1  C^-1],
// the two 64x64 inverses by the lane-pair substitution above applied to the identity (both at once, 128 threads each),
// the coupling block by two 64^3 register-tiled products -- ~15 kcycles instead of the ~165 kcycles of a
// thread-per-row back substitution -- and writes Linv (fp32 + 3xTF32 hi/lo) and U = Linv^T (hi/lo).
struct TriBase2Smem {
  __align__(16) float Lt[2][TS][SP64];   // A^T, C^T: operands of the substitution
  __align__(16) float X[2][TS][SP64];    // X0 = A^-T, X1 = C^-T   (row-major)  = U11, U22
  __align__(16) float Xt[2][TS][SP64];   // A^-1, C^-1              (row-major)  = Linv11, Linv22
  __align__(16) float Bt[TS][SP64];      // B^T
  __align__(16) float S[TS][SP64];       // B A^-1
  __align__(16) float R[TS][SP64];       // Linv21 = -C^-1 B A^-1
  __align__(16) float Rt[TS][SP64];      // its transpose = U12
  float rinv[2][TS];
};

__device__ __forceinline__ void split_store4(float *__restrict__ f32, float *__restrict__ hi, float *__restrict__ lo,
                                             int64_t off, float4 v) {
  float h[4], l[4];
  const float x[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    uint32_t hb;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(hb) : "f"(x[i]));
    h[i] = __uint_as_float(hb);
    l[i] = x[i] - h[i];
  }
  if (f32) *reinterpret_cast<float4 *>(f32 + off) = v;
  *reinterpret_cast<float4 *>(hi + off) = make_float4(h[0], h[1], h[2], h[3]);
  *reinterpret_cast<float4 *>(lo + off) = make_float4(l[0], l[1], l[2], l[3]);
}

__global__ void __launch_bounds__(GTHREADS, 1) triinv_base2_kernel(const float *__restrict__ L, int64_t np,
                                                                   float *__restrict__ Linv, float *__restrict__ Linv_hi,
                                                                   float *__restrict__ Linv_lo, float *__restrict__ U_hi,
                                                                   float *__restrict__ U_lo, int64_t wss) {
  L = slice(L, wss, blockIdx.z);   // output (Batch)
  Linv = slice(Linv, wss, blockIdx.z);
  Linv_hi = slice(Linv_hi, wss, blockIdx.z);
  Linv_lo = slice(Linv_lo, wss, blockIdx.z);
  U_hi = slice(U_hi, wss, blockIdx.z);
  U_lo = slice(U_lo, wss, blockIdx.z);
  extern __shared__ __align__(16) unsigned char smem_raw[];
  TriBase2Smem &sm = *reinterpret_cast<TriBase2Smem *>(smem_raw);
  const int t = threadIdx.x;
  const int warp = t >> 5, lane = t & 31;
  const int tc = 2 * warp + (lane >> 4), ti = lane & 15;
  const int64_t o = (int64_t)blockIdx.x * GT;
  const float *Lb = L + o * np + o;
  stage_transposed(Lb, np, sm.Lt[0]);                          // A^T
  stage_transposed(Lb + (int64_t)TS * np + TS, np, sm.Lt[1]);  // C^T
  stage_transposed(Lb + (int64_t)TS * np, np, sm.Bt);          // B^T
  __syncthreads();
  if (t < 2 * TS) sm.rinv[t >> 6][t & 63] = 1.0f / sm.Lt[t >> 6][t & 63][t & 63];
  __syncthreads();
  {   // X_g = I L_g^-T : two threads per row, group g = t >> 7
    const int g = t >> 7, r = (t & 127) >> 1, h = t & 1;
    float a[32];
#pragma unroll
    for (int lg = 0; lg < 8; ++lg)
#pragma unroll
      for (int q = 0; q < 4; ++q) a[4 * lg + q] = (4 * (2 * lg + h) + q == r) ? 1.0f : 0.0f;
    sub64_pair<SP64>(a, h, lane, &sm.Lt[g][0][0], sm.rinv[g]);
#pragma unroll
    for (int lg = 0; lg < 8; ++lg) {
      *reinterpret_cast<float4 *>(&sm.X[g][r][4 * (2 * lg + h)]) = make_float4(a[4 * lg + 0], a[4 * lg + 1], a[4 * lg + 2], a[4 * lg + 3]);
#pragma unroll
      for (int q = 0; q < 4; ++q) sm.Xt[g][4 * (2 * lg + h) + q][r] = a[4 * lg + q];
    }
  }
  __syncthreads();
  float S[4][4];
#pragma unroll
  for (int a = 0; a < 4; ++a)
#pragma unroll
    for (int b = 0; b < 4; ++b) S[a][b] = 0.0f;
  update64(S, sm.Bt, sm.Xt[0], ti, tc);   // S = -sum_p B[i][p] A^-1[p][j]
#pragma unroll
  for (int a = 0; a < 4; ++a)
#pragma unroll
    for (int b = 0; b < 4; ++b) S[a][b] = -S[a][b];
  tile4x4_to_smem(S, sm.S, ti, tc);
  __syncthreads();
#pragma unroll
  for (int a = 0; a < 4; ++a)
#pragma unroll
    for (int b = 0; b < 4; ++b) S[a][b] = 0.0f;
  update64(S, sm.X[1], sm.S, ti, tc);     // R = -sum_p C^-1[i][p] (B A^-1)[p][j]   (X1[p][i] = C^-1[i][p])
  tile4x4_to_smem(S, sm.R, ti, tc);
#pragma unroll
  for (int a = 0; a < 4; ++a)
#pragma unroll
    for (int b = 0; b < 4; ++b) sm.Rt[4 * tc + b][4 * ti + a] = S[a][b];
  __syncthreads();
  // coalesced output: 128 rows x 32 float4 of Linv and of U
#pragma unroll
  for (int q = 0; q < 16; ++q) {
    const int f = t + q * GTHREADS;
    const int row = f >> 5, c4 = f & 31;
    const int rh = row >> 6, rr = row & 63, ch = c4 >> 4, cc = (c4 & 15) * 4;
    float4 lv, uv;
    if (rh == ch) {
      lv = *reinterpret_cast<const float4 *>(&sm.Xt[rh][rr][cc]);
      uv = *reinterpret_cast<const float4 *>(&sm.X[rh][rr][cc]);
    } else if (rh == 1) {   // lower-left of Linv, zero in U
      lv = *reinterpret_cast<const float4 *>(&sm.R[rr][cc]);
      uv = make_float4(0.f, 0.f, 0.f, 0.f);
    } else {                // upper-right: zero in Linv, R^T in U
      lv = make_float4(0.f, 0.f, 0.f, 0.f);
      uv = *reinterpret_cast<const float4 *>(&sm.Rt[rr][cc]);
    }
    const int64_t off = (o + row) * np + o + c4 * 4;
    split_store4(Linv, Linv_hi, Linv_lo, off, lv);
    split_store4(nullptr, U_hi, U_lo, off, uv);
  }
}

int launch_triinv_base2(const float *L, int64_t np, float *Linv, float *Linv_hi, float *Linv_lo, float *U_hi, float *U_lo,
                        cudaStream_t st, const Batch &bt) {
  static PerDevice once;
  bool fresh = false;
  const int dev = once.slot(&fresh);
  if (dev < 0) return HB_ERR_CUDA;
  if (fresh) {
    HB_CUDA(cudaFuncSetAttribute(triinv_base2_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(TriBase2Smem)));
    once.done[dev] = true;
  }
  triinv_base2_kernel<<<dim3((unsigned)(np / GT), 1, (unsigned)bt.nout), GTHREADS, sizeof(TriBase2Smem), st>>>(
      L, np, Linv, Linv_hi, Linv_lo, U_hi, U_lo, bt.ws);
  count_launches(1);
  HB_LAUNCH_CHECK("triinv_base2");
  return HB_OK;
}

// C[I,J] -= P_I P_J^T for the lower tiles with J >= J_begin, P = A[:, kcol0 : kcol0+K); entries with a row or
// column index < r0 are left untouched.  (FP32 SIMT form of the outer update.)
__global__ void __launch_bounds__(GTHREADS, 2) chol_update_kernel(float *__restrict__ A, int64_t np, int kcol0, int K,
                                                                  int r0, int J_begin) {
  __shared__ GemmSmem sm;
  const int nt = (int)(np / GT);
  int tt = blockIdx.x, J = J_begin;
  while (tt >= nt - J) {
    tt -= nt - J;
    ++J;
  }
  const int I = J + tt;
  float acc[8][8];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[i][j] = 0.0f;
  gemm_mainloop<true, true>(A + (int64_t)I * GT * np + kcol0, np, A + (int64_t)J * GT * np + kcol0, np, 0, K, acc, sm);
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int64_t gi = (int64_t)I * GT + gemm_row(i);
    if (gi < r0) continue;
#pragma unroll
    for (int jh = 0; jh < 2; ++jh) {
      const int64_t gj = (int64_t)J * GT + gemm_col(jh * 4);
      if (gj < r0) continue;
      float4 *p = reinterpret_cast<float4 *>(A + gi * np + gj);
      float4 c = *p;
      c.x -= acc[i][jh * 4 + 0];
      c.y -= acc[i][jh * 4 + 1];
      c.z -= acc[i][jh * 4 + 2];
      c.w -= acc[i][jh * 4 + 3];
      *p = c;
    }
  }
}

int launch_cholesky(float *A, int64_t np, float *ws, int32_t *info, cudaStream_t st, const TcBuffers *tc, const Batch &bt) {
  if (np <= 0 || np % GT != 0) return HB_ERR_INVALID;
  if (!tc && bt.nout != 1) return HB_ERR_INVALID;   // the FP32 SIMT outer update serves single factorisations only
  static PerDevice once;   // aux[dev] = co-resident CTAs of the cooperative block kernel on that device
  bool fresh = false;
  const int dev = once.slot(&fresh);
  if (dev < 0) return HB_ERR_CUDA;
  if (fresh) {
    static_assert(sizeof(Block64Smem) <= BLOCK64_SMEM, "Block64Smem");
    HB_CUDA(cudaFuncSetAttribute(chol_block64_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, BLOCK64_SMEM));
    int sms = 0, per_sm = 0, coop = 0;
    HB_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    HB_CUDA(cudaDeviceGetAttribute(&coop, cudaDevAttrCooperativeLaunch, dev));
    HB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, chol_block64_kernel, GTHREADS, BLOCK64_SMEM));
    if (!coop || per_sm < 1) {
      set_error(cudaErrorNotSupported, "cholesky: cooperative launch unavailable");
      return HB_ERR_CUDA;
    }
    once.aux[dev] = sms * per_sm;
    once.done[dev] = true;
  }
  const int max_ctas = once.aux[dev];
  const int nt = (int)(np / GT), nt64 = (int)(np / TS);
  int *flags = reinterpret_cast<int *>(ws);   // [nt64][MAXBC64] tile flags (ws holds >= 64 KiB)
  if ((size_t)nt64 * MAXBC64 * sizeof(int) > (size_t)GT * GT * sizeof(float)) return HB_ERR_INVALID;
  HB_CUDA(memset_slices(flags, 0, (size_t)nt64 * MAXBC64 * sizeof(int), bt, st));
  int token = 0;
  for (int64_t cb = 0; cb < np; cb += OUTER) {
    const int64_t ce = cb + OUTER < np ? cb + OUTER : np;
    int jb0 = (int)(cb / TS), nbc = (int)((ce - cb) / TS);
    int ntasks = 0;   // per column: the diagonal composite + the tiles below it (see the kernel's task numbering)
    for (int jl = 0; jl < nbc; ++jl) {
      const int rest = nt64 - (jb0 + jl + (jl == nbc - 1 ? 1 : 2));
      ntasks += 1 + (rest > 0 ? rest : 0);
    }
    ++token;
    {
      int nout = bt.nout;
      int64_t wss = bt.ws;
      const int grid = ntasks * nout < max_ctas ? ntasks * nout : max_ctas;
      void *args[] = {&A, &np, &jb0, &nbc, &ntasks, &flags, &token, &info, &nout, &wss};
      HB_CUDA(cudaLaunchCooperativeKernel((const void *)chol_block64_kernel, dim3(grid), dim3(GTHREADS), args, BLOCK64_SMEM, st));
      count_launches(1);
    }
    if (ce == np) break;
    if (tc) {   // outer update on the tensor cores (wgmma 3xTF32, fit_tc.cu)
      const int s = launch_chol_outer_update_tc(A, np, cb, ce, *tc, st, bt);
      if (s != HB_OK) return s;
    } else {    // everything right of the block, K = block width
      const int J0 = (int)(ce / GT);
      int ntiles = 0;
      for (int J = J0; J < nt; ++J) ntiles += nt - J;
      chol_update_kernel<<<ntiles, GTHREADS, 0, st>>>(A, np, (int)cb, (int)(ce - cb), (int)ce, J0);
      count_launches(1);
    }
  }
  HB_LAUNCH_CHECK("cholesky");
  return HB_OK;
}

}  // namespace hb
