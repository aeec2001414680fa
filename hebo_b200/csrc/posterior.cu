// Posterior predict + MACE acquisition over candidate batches.
//   GP.predict   HEBO/hebo/models/gp/gp.py:137-164   mu = c + K* alpha ; var = s - ||Linv k*||^2 (floors, un-scaling)
//   MACE.eval    HEBO/hebo/acquisitions/acq.py:146-171  (LCB, -log EI, -log PI) with the log-approximation branch
//
// Three kernels per candidate chunk (chunked so the K* panel stays a bounded, L2-sized workspace):
//   kstar_kernel : raw candidates -> MinMax scale -> 1/lengthscale -> K* rows (and the K* alpha partial sums)
//   vnorm_kernel : V = K* Linv^T on the shared 128x128 SIMT GEMM core, triangular k-range, epilogue reduces
//                  ||v||^2 per row (V itself is never stored)
//   mace_kernel  : variance floors, un-scaling, MACE arithmetic (fp32, same operation order as the reference)
// All partial sums go to workspace slots and are combined in a fixed order: results are deterministic.
#include "gemm_core.cuh"
#include "h16.cuh"
#include "kernels.h"
#include "vnorm_sched.h"

namespace hb {

constexpr int KS_ROWS = 128;    // candidates per kstar_kernel tile
constexpr int KS_COLS = 128;    // training points per sub-tile
constexpr int KS_GROUP = 512;   // training points per tile (4 sub-tiles; one mean partial per candidate and group)
constexpr int KS_KC = 16;       // features per pipeline stage
constexpr int KS_FSLOTS = 2;    // feature stages in shared memory; a tile with at most this many keeps them all
// chunk rows of the workspace are rounded to whole clusters of 128-row bands: the tensor contraction pads the band count
// of a chunk to a multiple of the cluster size
constexpr int64_t CHUNK_ROWS = h16::CLUSTER * h16::BM;
static_assert(CHUNK_ROWS % (2 * GT) == 0, "chunk rows: a multiple of 2 GT");

// 16-byte global -> shared copy that bypasses the register file (L2 only)
__device__ __forceinline__ void cp_async16(void *dst, const void *src) {
  const unsigned ds = (unsigned)__cvta_generic_to_shared(dst);
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(ds), "l"(src) : "memory");
}

// acc[i][j] += (a_i - b_j)^2 over the kc features of one stage: a_i the feature of tile row (i < 4 ? 0 : 60) + ty*4 + i,
// b_j the Zt entry of sub-tile column (j < 4 ? 0 : 60) + tx*4 + j.  Per k: two broadcast and two conflict-free LDS.128
// against 64 FADD + 64 FFMA.
__device__ __forceinline__ void ks_contract(const float (&zs)[KS_KC][KS_ROWS], const float (&zt)[KS_KC][KS_COLS], int kc,
                                            float (&acc)[8][8]) {
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
#pragma unroll 4
  for (int kk = 0; kk < kc; ++kk) {
    const float4 a0 = *reinterpret_cast<const float4 *>(&zs[kk][ty * 4]);
    const float4 a1 = *reinterpret_cast<const float4 *>(&zs[kk][64 + ty * 4]);
    const float4 b0 = *reinterpret_cast<const float4 *>(&zt[kk][tx * 4]);
    const float4 b1 = *reinterpret_cast<const float4 *>(&zt[kk][64 + tx * 4]);
    const float a[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
    const float b[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float df = a[i] - b[j];
        acc[i][j] = fmaf(df, df, acc[i][j]);
      }
  }
}

// SPLIT: 0 = plain fp32 K* in KS (SIMT contraction / guard pass); 2 = the two-level fp16 split in the KS_lo buffer
// (h0 [mc_pad, np] halfs, then h1) and nothing else.
// fixlist != nullptr (SPLIT 0 only): the guard's second pass -- output row `slot` is the exact fp32 K* row of candidate
// fixlist[slot], for slot < *fixcount; no mean partials.  Its grid is at most one resident wave, whose CTAs walk the
// tiles of the first *fixcount slots.
// EMB: mixed model (gp_util.py:54-57): Zt holds d numeric rows followed by De embedding rows (both already divided by
// their lengthscales); the candidate's embedding features are gathered from tab_s (tables / le) by its categories
// Xe_s [m, e]; k* = s k_KERN(r over the numeric rows) Matern32(r over the embedding rows).
//
// A tile is KS_ROWS candidates x one KS_GROUP column group, walked as four 128 x 128 sub-tiles, 8 x 8 pairs per thread
// (two CTAs per SM for the tensor path's split rows; one, with room for r2e, for fp32 rows and the mixed model).
// Features move in stages of KS_KC: while one stage is contracted, the next stage's Zt slab is in flight (cp.async) and
// the next stage's candidate features are computed into the other slot, one barrier per stage.  A tile of at most
// KS_FSLOTS stages (d + De <= 32) computes its candidates' features once for all four sub-tiles; a deeper one recomputes
// them per sub-tile, so shared memory is 48 KB whatever d + De is.  Rows of the last tile past the candidate count get
// the K* row of an all-zero feature vector.
// Per pair the arithmetic is the Gram kernel's: fmaf(a - b, a - b, r2) in ascending k (numeric rows, then embedding rows),
// then s k_KERN(r2) [* Matern32(r2e)], pad columns (index >= n) zeroed.  The K* alpha mean partial of a row is summed in
// fmaf per 4-column lane of a sub-tile (a thread holds two lanes: columns tx*4.. and 64+tx*4..), sub-tiles then columns
// ascending, and the 32 lanes of a group are added in the xor 16, 8, 4, 2, 1 butterfly order.
template <int KERN, int SPLIT, bool EMB>
__global__ void __launch_bounds__(256, (EMB || SPLIT == 0) ? 1 : 2) kstar_kernel(const float *__restrict__ Xs, int64_t mc, int d,
                                                                 const float *__restrict__ x_mul, const float *__restrict__ x_add,
                                                                 const float *__restrict__ Zt, const float *__restrict__ alpha,
                                                                 const float *__restrict__ hyp, int64_t n, int64_t np,
                                                                 float *__restrict__ KS, float *__restrict__ KS_lo,
                                                                 float *__restrict__ mupart, int64_t mc_pad,
                                                                 const int32_t *__restrict__ fixlist,
                                                                 const int32_t *__restrict__ fixcount,
                                                                 const int32_t *__restrict__ Xe_s, const float *__restrict__ tab_s,
                                                                 ModelSpec sp) {
  __shared__ __align__(16) float zs[KS_FSLOTS][KS_KC][KS_ROWS];   // candidate features of a stage, transposed
  __shared__ __align__(16) float zt[2][KS_KC][KS_COLS];           // Zt slab of a stage, double-buffered
  __shared__ float mu_acc[8][2][256];   // per thread and row: its lanes tx and tx + 16 of the 32 four-column lanes
  const int t = threadIdx.x;
  const int tx = t & 15, ty = t >> 4;
  if (SPLIT != 0) fixlist = nullptr;   // (the guard pass writes fp32 rows)
  const int64_t nrows = fixlist ? (int64_t)*fixcount : mc;
  const int nrt = (int)ceil_div(nrows, KS_ROWS);
  const int ntiles = nrt * (int)ceil_div(np, KS_GROUP);
  const int De = EMB ? sp.De : 0;
  const int nnum = (int)ceil_div(d, KS_KC);                  // stages of the numeric rows, then of the embedding rows
  const int nst = nnum + (int)ceil_div(De, KS_KC);
  const bool keep = nst <= KS_FSLOTS;                        // features staged once per tile
  const float s = hyp[2];
  const float sa = pow2_scale(s, 1);   // fp16 operand scale: K* <= s lands in [0, 2)
  // feature rows [k0, k0 + kc) of stage c, and whether they are embedding rows
  auto stage_rows = [&](int c, int &k0, int &kc) {
    const bool emb = EMB && c >= nnum;
    k0 = emb ? d + (c - nnum) * KS_KC : c * KS_KC;
    kc = min(KS_KC, (emb ? d + De : d) - k0);
    return emb;
  };
  for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const int64_t r0 = (int64_t)(tile % nrt) * KS_ROWS;
    const int grp = tile / nrt;
    const int cg0 = grp * KS_GROUP;
    const int nstage = min(KS_GROUP / KS_COLS, (int)(np - cg0) / KS_COLS) * nst;
    // features: thread t computes those of tile row t % KS_ROWS
    const int64_t frow = r0 + (t & (KS_ROWS - 1));
    const bool flive = frow < nrows;
    const int src = flive ? (fixlist ? fixlist[frow] : (int)frow) : 0;
    // stage g of the tile is stage c of sub-tile sub (g = sub * nst + c)
    auto load_zt = [&](int g, int sub, int c) {   // into buffer g & 1
      int k0, kc;
      stage_rows(c, k0, kc);
      const float *base = Zt + cg0 + sub * KS_COLS;
#pragma unroll
      for (int q = 0; q < 2; ++q) {
        const int f = t + q * 256, kk = f >> 5, c4 = f & 31;
        if (kk < kc) cp_async16(&zt[g & 1][kk][c4 * 4], base + (int64_t)(k0 + kk) * np + c4 * 4);
      }
      asm volatile("cp.async.commit_group;\n" ::: "memory");
    };
    auto zslot = [&](int g, int c) { return keep ? c : g & 1; };
    auto load_zs = [&](int g, int c) {
      int k0, kc;
      const bool emb = stage_rows(c, k0, kc);
      float(&z)[KS_KC][KS_ROWS] = zs[zslot(g, c)];
#pragma unroll 1
      for (int q = 0; q < KS_KC / 2; ++q) {
        const int kk = (t >> 7) + 2 * q;
        if (kk < kc) {
          float v = 0.0f;
          if (flive)
            v = emb ? tab_s[emb_entry(sp, Xe_s, src, k0 + kk - d)]
                    : cand_feature(sp, sp.warp, Xs[(int64_t)src * d + k0 + kk], k0 + kk, x_mul, x_add, hyp);   // input warp fused here
          z[kk][t & (KS_ROWS - 1)] = v;
        }
      }
    };
    float r2[8][8], r2e[8][8];   // (r2e dead unless EMB)
#pragma unroll
    for (int i = 0; i < 8; ++i) mu_acc[i][0][t] = mu_acc[i][1][t] = 0.0f;
    load_zt(0, 0, 0);
    load_zs(0, 0);
    asm volatile("cp.async.wait_all;\n" ::: "memory");
    __syncthreads();
    for (int g = 0, sub = 0, c = 0; g < nstage; ++g) {
      const int c1 = c + 1 == nst ? 0 : c + 1, sub1 = c1 ? sub : sub + 1;   // the next stage
      if (c == 0) {
#pragma unroll
        for (int i = 0; i < 8; ++i)
#pragma unroll
          for (int j = 0; j < 8; ++j) r2[i][j] = r2e[i][j] = 0.0f;
      }
      if (g + 1 < nstage) load_zt(g + 1, sub1, c1);
      {
        int k0, kc;
        const bool emb = stage_rows(c, k0, kc);
        if (emb) ks_contract(zs[zslot(g, c)], zt[g & 1], kc, r2e);
        else ks_contract(zs[zslot(g, c)], zt[g & 1], kc, r2);
      }
      if (g + 1 < nstage && (!keep || sub1 == 0)) load_zs(g + 1, c1);
      if (c == nst - 1) {   // sub-tile done: K* rows, mean partials
        const int c0 = cg0 + sub * KS_COLS;
        float al[2][4];
        int ncol[2];   // valid columns among each 4-column half (pad columns, training index >= n, must come out as exact
                       // zeros: the pad block of Linv is the identity)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int cc = c0 + h * 64 + tx * 4;
          const float4 a4 = __ldg(reinterpret_cast<const float4 *>(alpha + cc));
          al[h][0] = a4.x; al[h][1] = a4.y; al[h][2] = a4.z; al[h][3] = a4.w;
          ncol[h] = (int)min((int64_t)4, max((int64_t)0, n - cc));
        }
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const int64_t rowoff = (r0 + (i < 4 ? 0 : 60) + ty * 4 + i) * np + c0 + tx * 4;
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            float o[4], mu = mu_acc[i][h][t];
#pragma unroll
            for (int j = 0; j < 4; ++j) {
              float kv = s * kern_eval<KERN>(r2[i][h * 4 + j]);
              if (EMB) kv *= kern_eval<HB_KERN_MATERN32>(r2e[i][h * 4 + j]);
              if (j >= ncol[h]) kv = 0.0f;
              o[j] = kv;
              mu = fmaf(kv, al[h][j], mu);
            }
            mu_acc[i][h][t] = mu;
            const int64_t off = rowoff + h * 64;
            if (SPLIT == 2) {
              unsigned int a01, a23, b01, b23;
              split_h16x2(o[0] * sa, o[1] * sa, a01, b01);
              split_h16x2(o[2] * sa, o[3] * sa, a23, b23);
              __half *h0 = reinterpret_cast<__half *>(KS_lo) + off;   // h0 [mc_pad, np], then h1
              *reinterpret_cast<uint2 *>(h0) = make_uint2(a01, a23);
              *reinterpret_cast<uint2 *>(h0 + mc_pad * np) = make_uint2(b01, b23);
            } else {
              *reinterpret_cast<float4 *>(KS + off) = make_float4(o[0], o[1], o[2], o[3]);
            }
          }
        }
      }
      asm volatile("cp.async.wait_all;\n" ::: "memory");
      __syncthreads();
      c = c1;
      sub = sub1;
    }
    // lanes tx and tx + 16 first (the xor-16 step), then xor 8..1 across the 16 threads of this row group
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      float v = mu_acc[i][0][t] + mu_acc[i][1][t];
#pragma unroll
      for (int o = 8; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
      if (tx == 0 && mupart) mupart[(int64_t)grp * mc_pad + r0 + (i < 4 ? 0 : 60) + ty * 4 + i] = v;
    }
  }
}

// ||Linv k*||^2 per candidate and column tile J:  vpart[J][row] = sum_{c in tile J} (sum_{k <= c} KS[row][k] Linv[c][k])^2
__global__ void __launch_bounds__(GTHREADS, 2) vnorm_kernel(const float *__restrict__ KS, const float *__restrict__ Linv,
                                                            int64_t np, int64_t mc_pad, float *__restrict__ vpart) {
  __shared__ GemmSmem sm;
  const int nt = (int)(np / GT);
  const int J = nt - 1 - (int)blockIdx.x;   // heaviest (longest k range) tiles first
  const int64_t rt = blockIdx.y;
  float acc[8][8];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[i][j] = 0.0f;
  gemm_mainloop<true, true>(KS + rt * GT * np, np, Linv + (int64_t)J * GT * np, np, 0, (J + 1) * GT, acc, sm);
  const int tx = threadIdx.x & 15;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    float s = 0.0f;
#pragma unroll
    for (int j = 0; j < 8; ++j) s = fmaf(acc[i][j], acc[i][j], s);
#pragma unroll
    for (int o = 8; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (tx == 0) vpart[(int64_t)J * mc_pad + rt * GT + gemm_row(i)] = s;
  }
}

// ---- precision guard of the tensor path ------------------------------------------------------------------
// sigma^2 = s - ||v||^2 cancels when a candidate sits on the data; the tensor cores' fp32 accumulation is
// not round-to-nearest, which would exceed the 1e-4 sigma criterion once
// sigma^2 < ~s/40.  Rows whose variance falls below GUARD_THETA * s are therefore flagged and their ||v||^2 is
// recomputed on the FP32 SIMT pipe from the same operands (K* = hi + lo); typical BO batches flag few rows, a
// batch that sits entirely on the data degrades gracefully to the SIMT contraction.
constexpr float GUARD_THETA = 0.12f;

// measurement hook (bench.py "guard_flagged_frac"): rows seen / rows flagged by the guard since the last reset
__device__ unsigned long long g_guard_stats[2];

__global__ void __launch_bounds__(256) guard_kernel(const float *__restrict__ vpart, int nslots, int64_t mc,
                                                    int64_t mc_pad, const float *__restrict__ hyp,
                                                    float theta, int32_t *__restrict__ fixmap,
                                                    int32_t *__restrict__ fixlist, int32_t *__restrict__ count) {
  const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= mc) return;
  const float s = hyp[2];
  float vsq = 0.0f;
  for (int j = 0; j < nslots; ++j) vsq += vpart[(int64_t)j * mc_pad + r];
  int32_t slot = -1;
  if ((s - vsq) < theta * s) {
    slot = atomicAdd(count, 1);
    fixlist[slot] = (int32_t)r;
    atomicAdd(&g_guard_stats[1], 1ull);
  }
  fixmap[r] = slot;
  if (threadIdx.x == 0) atomicAdd(&g_guard_stats[0], (unsigned long long)min((int64_t)blockDim.x, mc - (int64_t)blockIdx.x * blockDim.x));
}

int guard_stats(unsigned long long *out, int reset) {
  HB_CUDA(cudaMemcpyFromSymbol(out, g_guard_stats, 2 * sizeof(unsigned long long)));
  if (reset) {
    const unsigned long long z[2] = {0ull, 0ull};
    HB_CUDA(cudaMemcpyToSymbol(g_guard_stats, z, sizeof(z)));
  }
  return HB_OK;
}

__global__ void __launch_bounds__(GTHREADS, 1) vnorm_fix_kernel(const float *__restrict__ KS_hi,
                                                                const float *__restrict__ KS_lo,
                                                                const float *__restrict__ Linv, int64_t np,
                                                                int64_t mc_pad, const int32_t *__restrict__ fixlist,
                                                                const int32_t *__restrict__ count,
                                                                float *__restrict__ vfix, int compact) {
  __shared__ GemmSmem sm;
  const int cnt = *count;
  const int nt = (int)(np / GT);
  const int64_t ngr = ceil_div(cnt, GT);   // row groups of the flagged slots
  const int tx = threadIdx.x & 15;
  // units (J, g) ordered by decreasing k range (J = nt - 1 first), dealt out in rounds of gridDim.x, every other round in
  // reverse CTA order, so that every CTA gets about the same number of k-tiles
  for (int64_t round = 0;; ++round) {
    const int64_t u = round * gridDim.x + ((round & 1) ? gridDim.x - 1 - blockIdx.x : blockIdx.x);
    if (u >= ngr * nt) break;
    const int J = nt - 1 - (int)(u / ngr);
    const int64_t g = u % ngr;
    int64_t rows[2];
#pragma unroll
    for (int q = 0; q < 2; ++q) {
      const int64_t slot = g * GT + ((threadIdx.x + q * GTHREADS) >> 2);
      rows[q] = compact ? (slot < cnt ? slot : 0) : fixlist[slot < cnt ? slot : 0];   // compact: KS_hi row = slot
    }
    double acc[8][8];
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[i][j] = 0.0;
    gemm_mainloop_gatherA(KS_hi, KS_lo, np, rows, Linv + (int64_t)J * GT * np, np, 0, (J + 1) * GT, acc, sm);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      double s = 0.0;
#pragma unroll
      for (int j = 0; j < 8; ++j) s = fma(acc[i][j], acc[i][j], s);
#pragma unroll
      for (int o = 8; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
      if (tx == 0) vfix[(int64_t)J * mc_pad + g * GT + gemm_row(i)] = (float)s;
    }
  }
}

// (philox_normal2, common.cuh: Philox4x32-10 + Box-Muller for the production (non-parity) noise path)

// MACE.eval arithmetic for one row (acq.py:151-171), fp32, same operation order as the reference
__device__ __forceinline__ void mace_row(float py, float ps2, float noise_var, float tau, float kappa, float eps,
                                         float z1, float z2, float &lcb, float &o1, float &o2) {
  const float noise = __fmul_rn(1.4142135623730951f, sqrtf(noise_var));      // acq.py:152
  const float ps = fmaxf(sqrtf(ps2), 1.1920929e-07f);                        // acq.py:153
  lcb = __fsub_rn(__fadd_rn(py, __fmul_rn(noise, z1)), __fmul_rn(kappa, ps));   // acq.py:154
  const float num = __fsub_rn(__fsub_rn(__fsub_rn(tau, eps), py), __fmul_rn(noise, z2));
  const float zz = __fdiv_rn(num, ps);                                       // acq.py:155
  const float zsq = __fmul_rn(zz, zz);
  const float log_phi = __fsub_rn(__fdiv_rn(-zsq, 2.0f), 0.9189385332046727f);   // Normal.log_prob
  const float Phi = __fmul_rn(0.5f, __fadd_rn(1.0f, erff(__fdiv_rn(zz, 1.4142135623730951f))));   // Normal.cdf
  const float EI = __fmul_rn(ps, __fadd_rn(__fmul_rn(Phi, zz), expf(log_phi)));   // acq.py:160
  const float logEI = logf(EI), logPI = logf(Phi);
  const bool ok = (zz > -6.0f) && isfinite(logEI) && isfinite(logPI);        // acq.py:164
  if (ok) {
    o1 = -logEI;
    o2 = -logPI;
  } else {
    const float half_z2 = __fmul_rn(0.5f, zsq);
    const float logEIapp = __fsub_rn(__fsub_rn(logf(ps), half_z2), logf(__fsub_rn(zsq, 1.0f)));     // acq.py:161
    const float logPIapp = __fsub_rn(__fsub_rn(-half_z2, logf(-zz)), 0.9189385332046727f);          // acq.py:162
    o1 = -logEIapp;
    o2 = -logPIapp;
  }
}

// standalone epilogue: MACE over any model's (mu, var) already on the device
__global__ void __launch_bounds__(256) mace_only_kernel(const float *__restrict__ mu, const float *__restrict__ var,
                                                        int64_t m, float noise_var, float tau, float kappa, float eps,
                                                        const float *__restrict__ xi1, const float *__restrict__ xi2,
                                                        uint64_t seed, float *__restrict__ F) {
  const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= m) return;
  float z1, z2;
  if (xi1 && xi2) {
    z1 = xi1[r];
    z2 = xi2[r];
  } else {
    philox_normal2(seed, (uint64_t)r, z1, z2);
  }
  float lcb, o1, o2;
  mace_row(mu[r], var[r], noise_var, tau, kappa, eps, z1, z2, lcb, o1, o2);
  F[r * 3 + 0] = lcb;
  F[r * 3 + 1] = o1;
  F[r * 3 + 2] = o2;
}

int launch_mace_only(const float *mu, const float *var, int64_t m, float noise_var, float tau, float kappa, float eps,
                     const float *xi1, const float *xi2, uint64_t seed, float *F, cudaStream_t st) {
  if (m <= 0) return HB_ERR_INVALID;
  mace_only_kernel<<<(int)ceil_div(m, 256), 256, 0, st>>>(mu, var, m, noise_var, tau, kappa, eps, xi1, xi2, seed, F);
  count_launches(1);
  HB_LAUNCH_CHECK("mace_only");
  return HB_OK;
}

// single-objective acquisitions over (mu, var) (acq.py:55-82, nomr.py:32-34), each the reference's torch expression in
// IEEE fp32 with every rounding explicit, so that no FMA contraction changes a bit
__global__ void __launch_bounds__(256) acq1_kernel(const float *__restrict__ mu, const float *__restrict__ var, int64_t m,
                                                   int mode, float kappa, float eta, float *__restrict__ f) {
  const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= m) return;
  const float py = mu[r], ps = __fsqrt_rn(var[r]);
  float v;
  switch (mode) {
    case HB_ACQ1_LCB: v = __fsub_rn(py, __fmul_rn(kappa, ps)); break;                       // py - kappa * ps2.sqrt()
    case HB_ACQ1_MEAN: v = py; break;                                                      // py
    case HB_ACQ1_SIGMA: v = __fmul_rn(-1.0f, ps); break;                                   // -1 * ps2.sqrt()
    default: v = __fsub_rn(fabsf(__fsub_rn(py, eta)), __fmul_rn(kappa, ps)); break;       // |py - eta| - kappa * ps2.sqrt()
  }
  f[r] = v;
}

int launch_acq1(const float *mu, const float *var, int64_t m, int mode, float kappa, float eta, float *f, cudaStream_t st) {
  if (m <= 0 || mode < HB_ACQ1_LCB || mode > HB_ACQ1_ABS_ETA) return HB_ERR_INVALID;
  acq1_kernel<<<(int)ceil_div(m, 256), 256, 0, st>>>(mu, var, m, mode, kappa, eta, f);
  count_launches(1);
  HB_LAUNCH_CHECK("acq1");
  return HB_OK;
}


// GeneralAcq.eval (acq.py:211-242) over K = num_obj + num_constr outputs: mu / var [K, m] output-major (row b of output b,
// as K single-output posterior calls write them).  Every operation is correctly rounded and nothing is contracted into an
// FMA, so each column is bit-identical to the IEEE fp32 evaluation of the reference's torch expression:
//   ps = sqrt(ps2).clamp(min = FLT_EPSILON)  (a NaN stays NaN, as torch.clamp keeps it)
//   py = py + noise_sd * xi                  (when noise_sd != NULL, i.e. use_noise)
//   Fo = py - kappa * ps (objectives),  Fc = py - c_kappa * ps (constraints)
// cv = sum_j max(0, Fc[:, j]) in fp32, columns ascending (NaN propagates, so a NaN constraint is never feasible).
// xi [m, K] (the reference's torch.randn(py.shape)) or NULL: Philox draws keyed by (seed, counter), element q = r K + b
// takes half q % 2 of the pair q / 2.
__global__ void __launch_bounds__(256) general_acq_kernel(const float *__restrict__ mu, const float *__restrict__ var, int64_t m,
                                                          int num_obj, int num_constr, float kappa, float c_kappa,
                                                          const float *__restrict__ noise_sd, const float *__restrict__ xi,
                                                          uint64_t seed, uint64_t counter, float *__restrict__ Fo,
                                                          float *__restrict__ Fc, float *__restrict__ cv) {
  const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= m) return;
  const int K = num_obj + num_constr;
  float viol = 0.0f;
  for (int b = 0; b < K; ++b) {
    float py = mu[(int64_t)b * m + r];
    const float s = __fsqrt_rn(var[(int64_t)b * m + r]);
    const float ps = s < 1.1920929e-07f ? 1.1920929e-07f : s;
    if (noise_sd) {
      const int64_t q = r * K + b;
      float z;
      if (xi) {
        z = xi[q];
      } else {
        float z0, z1;
        philox_normal2(seed, (uint64_t)(q >> 1), counter, z0, z1);
        z = (q & 1) ? z1 : z0;
      }
      py = __fadd_rn(py, __fmul_rn(noise_sd[b], z));
    }
    if (b < num_obj) {
      Fo[r * num_obj + b] = __fsub_rn(py, __fmul_rn(kappa, ps));
    } else {
      const float c = __fsub_rn(py, __fmul_rn(c_kappa, ps));
      if (Fc) Fc[r * num_constr + (b - num_obj)] = c;
      viol = __fadd_rn(viol, isnan(c) ? c : fmaxf(c, 0.0f));
    }
  }
  if (cv) cv[r] = viol;
}

int launch_general_acq(const float *mu, const float *var, int64_t m, int64_t num_obj, int64_t num_constr, float kappa,
                       float c_kappa, const float *noise_sd, const float *xi, uint64_t seed, uint64_t counter, float *Fo,
                       float *Fc, float *cv, cudaStream_t st) {
  if (m <= 0 || num_obj < 1 || num_constr < 0 || num_obj + num_constr > HB_MAX_OUTPUTS) return HB_ERR_INVALID;
  general_acq_kernel<<<(int)ceil_div(m, 256), 256, 0, st>>>(mu, var, m, (int)num_obj, (int)num_constr, kappa, c_kappa, noise_sd,
                                                            xi, seed, counter, Fo, Fc, cv);
  count_launches(1);
  HB_LAUNCH_CHECK("general_acq");
  return HB_OK;
}

// MOMeanSigmaLCB.eval (acq.py:99-129) over one output's mu / var [m].  Correctly rounded operations, no FMA contraction, so
// each column is bit-identical to the IEEE fp32 evaluation of the reference's torch expression:
//   py = py + noise_sd * xi,  ps = sqrt(ps2)  (no clamp: a NaN or negative ps2 gives NaN)
//   F [m, 2] = (py, -1 * ps),  G [m] = (py - kappa * ps) - best_y
// xi [m] (the reference's torch.randn(py.shape)) or NULL: Philox draws keyed by (seed, counter), row r takes half r % 2 of
// the pair r / 2 -- general_acq_kernel's layout with K = 1.
__global__ void __launch_bounds__(256) mo_lcb_kernel(const float *__restrict__ mu, const float *__restrict__ var, int64_t m,
                                                     float noise_sd, float best_y, float kappa, const float *__restrict__ xi,
                                                     uint64_t seed, uint64_t counter, float *__restrict__ F,
                                                     float *__restrict__ G) {
  const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= m) return;
  float z;
  if (xi) {
    z = xi[r];
  } else {
    float z0, z1;
    philox_normal2(seed, (uint64_t)(r >> 1), counter, z0, z1);
    z = (r & 1) ? z1 : z0;
  }
  const float py = __fadd_rn(mu[r], __fmul_rn(noise_sd, z));
  const float ps = __fsqrt_rn(var[r]);
  F[r * 2 + 0] = py;
  F[r * 2 + 1] = __fmul_rn(-1.0f, ps);                                                     // exact: ps = 0 gives -0
  G[r] = __fsub_rn(__fsub_rn(py, __fmul_rn(kappa, ps)), best_y);
}

int launch_mo_lcb(const float *mu, const float *var, int64_t m, float noise_sd, float best_y, float kappa, const float *xi,
                  uint64_t seed, uint64_t counter, float *F, float *G, cudaStream_t st) {
  if (m <= 0) return HB_ERR_INVALID;
  mo_lcb_kernel<<<(int)ceil_div(m, 256), 256, 0, st>>>(mu, var, m, noise_sd, best_y, kappa, xi, seed, counter, F, G);
  count_launches(1);
  HB_LAUNCH_CHECK("mo_lcb");
  return HB_OK;
}


__global__ void __launch_bounds__(256) mace_kernel(const float *__restrict__ mupart, int ncg,
                                                   const float *__restrict__ vpart, int nt,
                                                   const int32_t *__restrict__ fixmap,
                                                   const float *__restrict__ vfix, int nt_fix, int64_t mc,
                                                   int64_t mc_pad, int64_t row_offset, int64_t rng_offset,
                                                   const float *__restrict__ hyp, float y_mean, float y_std,
                                                   int pred_likeli, float tau, float kappa, float eps,
                                                   const float *__restrict__ xi1, const float *__restrict__ xi2,
                                                   uint64_t seed, float *__restrict__ F, float *__restrict__ mu_out,
                                                   float *__restrict__ var_out) {
  const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= mc) return;
  const float sn2 = hyp[0], c = hyp[1], s = hyp[2];
  float mu_t = 0.0f;
  for (int g = 0; g < ncg; ++g) mu_t += mupart[(int64_t)g * mc_pad + r];
  mu_t += c;
  float vsq = 0.0f;
  const int fm = fixmap ? fixmap[r] : -1;
  if (fm >= 0) {
    for (int j = 0; j < nt_fix; ++j) vsq += vfix[(int64_t)j * mc_pad + fm];     // guarded row: FP32 SIMT recomputation
  } else {
    for (int j = 0; j < nt; ++j) vsq += vpart[(int64_t)j * mc_pad + r];
  }
  float var_t = s - vsq;
  if (pred_likeli) var_t += sn2;                            // gp.py:158-159: pred = lik(pred) adds the noise FIRST,
  var_t = fmaxf(var_t, 1e-6f);                              // then .variance applies gpytorch's min_variance floor (fp32)
  const float py = __fadd_rn(__fmul_rn(mu_t, y_std), y_mean);                 // gp.py:162
  const float ps2 = fmaxf(__fmul_rn(var_t, __fmul_rn(y_std, y_std)), 1.1920929e-07f);   // gp.py:163-164
  const int64_t gr = row_offset + r;
  if (mu_out) mu_out[gr] = py;
  if (var_out) var_out[gr] = ps2;
  if (!F) return;
  // ---- MACE, acq.py:151-171
  float z1, z2;
  if (xi1 && xi2) {
    z1 = xi1[gr];
    z2 = xi2[gr];
  } else {
    philox_normal2(seed, (uint64_t)(rng_offset + gr), z1, z2);
  }
  const float noise_var = __fmul_rn(sn2, __fmul_rn(y_std, y_std));           // gp.py:184
  float lcb, o1, o2;
  mace_row(py, ps2, noise_var, tau, kappa, eps, z1, z2, lcb, o1, o2);
  F[gr * 3 + 0] = lcb;
  F[gr * 3 + 1] = o1;
  F[gr * 3 + 2] = o2;
}

int kstar_groups(int64_t np) { return (int)ceil_div(np, KS_GROUP); }

// K* rows of the mc candidates xs [mc, d] (categories xe [mc, e]), in one of three output forms:
//   KS_h16 != nullptr:  the two-level fp16 split into KS_h16 (tensor path), mean partials into mupart;
//   fixlist != nullptr: the guard pass: KS row `slot` is the exact fp32 row of candidate fixlist[slot], slot < *fixcount
//                       (mupart nullptr);
//   otherwise:          fp32 rows into KS, mean partials into mupart.
// CTAs of `kernel` (256 threads) that are resident on the current device at once, looked up once per device
template <class Kernel>
static int resident_wave(Kernel kernel, PerDevice &once, int64_t *ctas) {
  bool fresh = false;
  const int dev = once.slot(&fresh);
  if (dev < 0) return HB_ERR_CUDA;
  if (fresh) {
    int sms = 0, per_sm = 0;
    HB_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    HB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, 256, 0));
    once.aux[dev] = sms * max(per_sm, 1);
    once.done[dev] = true;
  }
  *ctas = once.aux[dev];
  return HB_OK;
}
template <int KERN, bool EMB>
static int kstar_guard_wave(int64_t *ctas) {
  static PerDevice once;
  return resident_wave(kstar_kernel<KERN, 0, EMB>, once, ctas);
}

int launch_kstar(const Fitted &gp, const float *xs, const int32_t *xe, int64_t mc, float *KS, float *KS_h16, float *mupart,
                 int64_t mc_pad, const int32_t *fixlist, const int32_t *fixcount, cudaStream_t st) {
  const ModelSpec &sp = gp.sp;
  const int64_t tiles = ceil_div(mc, KS_ROWS) * kstar_groups(gp.np);   // (the guard pass: the most its count can need)
  int r = HB_OK;
  const int s = with_kernel(gp.kern, sp.e > 0, [&](auto kk, auto ee) {
    constexpr int KERN = decltype(kk)::value;
    constexpr bool EMB = decltype(ee)::value;
    if (KS_h16) {
      kstar_kernel<KERN, 2, EMB><<<(unsigned)tiles, 256, 0, st>>>(xs, mc, sp.d, gp.x_mul, gp.x_add, gp.Zt, gp.alpha, gp.hyp, gp.n,
                                                                  gp.np, KS, KS_h16, mupart, mc_pad, fixlist, fixcount, xe,
                                                                  gp.tab_s, sp);
    } else {
      int64_t grid = tiles;
      if (fixlist) {   // the flagged count is only known on the device: one resident wave walks its tiles
        int64_t wave = 0;
        r = kstar_guard_wave<KERN, EMB>(&wave);
        if (r != HB_OK) return;
        grid = min(grid, wave);
      }
      kstar_kernel<KERN, 0, EMB><<<(unsigned)grid, 256, 0, st>>>(xs, mc, sp.d, gp.x_mul, gp.x_add, gp.Zt, gp.alpha, gp.hyp, gp.n,
                                                                 gp.np, KS, KS_h16, mupart, mc_pad, fixlist, fixcount, xe,
                                                                 gp.tab_s, sp);
    }
  });
  if (s != HB_OK) return s;
  if (r != HB_OK) return r;
  count_launches(1);
  return HB_OK;
}

// The library's stream of the current device for the contraction stages of a pipelined posterior call, created once at
// the highest priority, and the events that order it against the caller's stream.  Every call records the events
// again; a wait orders against the record that precedes it.
struct Pipeline {
  cudaStream_t hi;
  cudaEvent_t entry, kstar, started;
};
static int pipeline(Pipeline **out) {
  static PerDevice once;
  static Pipeline p[MAX_DEVICES];
  bool fresh = false;
  const int dev = once.slot(&fresh);
  if (dev < 0) return HB_ERR_CUDA;
  if (fresh) {
    int least = 0, greatest = 0;
    HB_CUDA(cudaDeviceGetStreamPriorityRange(&least, &greatest));
    HB_CUDA(cudaStreamCreateWithPriority(&p[dev].hi, cudaStreamNonBlocking, greatest));
    for (cudaEvent_t *e : {&p[dev].entry, &p[dev].kstar, &p[dev].started})
      HB_CUDA(cudaEventCreateWithFlags(e, cudaEventDisableTiming));
    once.done[dev] = true;
  }
  *out = &p[dev];
  return HB_OK;
}

PostWs carve_posterior_ws(void *ws, int64_t np, int64_t m_chunk) {
  PostWs w;
  w.mc_pad = round_up(m_chunk, CHUNK_ROWS);
  const int64_t nt = np / GT;
  Carver c{reinterpret_cast<float *>(ws)};
  w.KS = c.take(w.mc_pad * np);
  for (int b = 0; b < 2; ++b) w.KS2[b] = c.take(w.mc_pad * np);
  for (int b = 0; b < 2; ++b) w.mupart[b] = c.take(kstar_groups(np) * w.mc_pad);
  w.vpart = c.take(nt * w.mc_pad);
  w.vfix = c.take(nt * w.mc_pad);
  w.fixmap = reinterpret_cast<int32_t *>(c.take(w.mc_pad));
  w.fixlist = reinterpret_cast<int32_t *>(c.take(w.mc_pad));
  w.fixcount = reinterpret_cast<int32_t *>(c.take(0));   // one word of the 512-byte tail
  w.bytes = (size_t)c.used * sizeof(float) + 512;
  return w;
}

int launch_posterior_mace(const Fitted &gp, const float *Xs, const int32_t *Xe_s, int64_t m, int64_t rng_offset,
                          const float *Linv_hi, const float *Linv_lo, float tau, float kappa, float eps, const float *xi1,
                          const float *xi2, uint64_t seed, float *F, float *mu, float *var, void *ws, int64_t ws_bytes,
                          int64_t m_chunk, cudaStream_t st) {
  const ModelSpec &sp = gp.sp;
  const int64_t np = gp.np;
  if (m <= 0 || m_chunk <= 0) return HB_ERR_INVALID;
  const PostWs w = carve_posterior_ws(ws, np, m_chunk);
  if (ws_bytes < 0 || (size_t)ws_bytes < w.bytes) return HB_ERR_INVALID;
  const int nt = (int)(np / GT);
  const bool tensor = Linv_hi != nullptr && Linv_lo != nullptr;   // wgmma path (two-level fp16 split), else FP32 SIMT
  // A tensor-path call of two or more chunks is pipelined: K* of every chunk runs on the caller's stream `st`, the
  // contraction, guard and MACE stages on the library's highest-priority stream `cs`, so that the K* of chunk i + 1 runs on
  // the SMs the contraction of chunk i leaves free (it fills at most 30 clusters of 4 CTAs, 120 of an H100's 132 SMs, and
  // its 193 KiB CTAs leave no room for a K* CTA beside them).  K* of chunk i + 1 waits until `cs` has reached the
  // contraction of chunk i (event `started`), so that the contraction's clusters are dispatched before the K* CTAs can
  // fill the SMs -- its schedule is static, one late cluster delays the whole launch -- and the stream's priority gives
  // the guard and MACE stages the SMs as K* CTAs retire.  `started` also follows MACE of chunk i - 1, the last reader of
  // the KS2 / mupart buffer that K* of chunk i + 1 writes (the other buffer holds chunk i).  The rest of the workspace is
  // only touched on `cs`.  One-chunk calls and the SIMT path run everything on `st`.
  const bool pipelined = tensor && m > m_chunk;
  Pipeline *pl = nullptr;
  cudaStream_t cs = st;
  if (pipelined) {
    const int s = pipeline(&pl);
    if (s != HB_OK) return s;
    cs = pl->hi;
    HB_CUDA(cudaEventRecord(pl->entry, st));
    HB_CUDA(cudaStreamWaitEvent(cs, pl->entry, 0));
  }
  auto chunk = [&](int64_t c0, int b) -> int {
    const int64_t mc = min(m_chunk, m - c0);
    const int64_t mc_pad = round_up(mc, GT);
    const float *xs = Xs + c0 * sp.d;
    const int32_t *xe = sp.e > 0 ? Xe_s + c0 * sp.e : nullptr;
    if (pipelined && c0 > 0) HB_CUDA(cudaStreamWaitEvent(st, pl->started, 0));
    int s = launch_kstar(gp, xs, xe, mc, w.KS, tensor ? w.KS2[b] : nullptr, w.mupart[b], w.mc_pad, nullptr, nullptr, st);
    if (s != HB_OK) return s;
    if (pipelined) {
      HB_CUDA(cudaEventRecord(pl->kstar, st));
      HB_CUDA(cudaStreamWaitEvent(cs, pl->kstar, 0));
      HB_CUDA(cudaEventRecord(pl->started, cs));
    }
    int nslots = nt;
    if (tensor) {
      const __half *kh0 = reinterpret_cast<const __half *>(w.KS2[b]), *kh1 = kh0 + w.mc_pad * np;
      s = launch_vnorm_h16(kh0, kh1, w.mc_pad, reinterpret_cast<const __half *>(Linv_hi),
                           reinterpret_cast<const __half *>(Linv_lo), Linv_lo + np * np / 2, gp.hyp, np, mc_pad, w.mc_pad, w.vpart, cs);
      if (s != HB_OK) return s;
      nslots = (int)ceil_div(np, 128);
      HB_CUDA(cudaMemsetAsync(w.fixcount, 0, sizeof(int32_t), cs));
      guard_kernel<<<(int)ceil_div(mc, 256), 256, 0, cs>>>(w.vpart, nslots, mc, w.mc_pad, gp.hyp, GUARD_THETA, w.fixmap, w.fixlist,
                                                           w.fixcount);
      // exact fp32 K* rows of the flagged candidates only (compact, row = slot), then their FP32 contraction
      s = launch_kstar(gp, xs, xe, mc, w.KS, nullptr, nullptr, w.mc_pad, w.fixlist, w.fixcount, cs);
      if (s != HB_OK) return s;
      static PerDevice fix_once;
      int64_t wave = 0;
      s = resident_wave(vnorm_fix_kernel, fix_once, &wave);
      if (s != HB_OK) return s;
      const unsigned gf = (unsigned)min((int64_t)nt * (mc_pad / GT), wave);   // one resident wave walks the flagged rows
      vnorm_fix_kernel<<<gf, GTHREADS, 0, cs>>>(w.KS, nullptr, gp.Linv, np, w.mc_pad, w.fixlist, w.fixcount, w.vfix, 1);
      count_launches(3);
    } else {
      const dim3 g2((unsigned)nt, (unsigned)(mc_pad / GT));
      prof_begin(cs);
      vnorm_kernel<<<g2, GTHREADS, 0, cs>>>(w.KS, gp.Linv, np, w.mc_pad, w.vpart);
      prof_end(cs);
      count_launches(2);
    }
    mace_kernel<<<(int)ceil_div(mc, 256), 256, 0, cs>>>(w.mupart[b], kstar_groups(np), w.vpart, nslots, tensor ? w.fixmap : nullptr,
                                                        w.vfix, nt, mc, w.mc_pad, c0, rng_offset, gp.hyp, gp.y_mean, gp.y_std,
                                                        gp.pred_likeli, tau, kappa, eps, xi1, xi2, seed, F, mu, var);
    return HB_OK;
  };
  int s = HB_OK;
  for (int64_t c0 = 0, i = 0; c0 < m && s == HB_OK; c0 += m_chunk, ++i) s = chunk(c0, pipelined ? (int)(i & 1) : 0);
  if (pipelined) {   // the caller's stream waits for the last stage (after an error too, so that nothing outlives the call)
    HB_CUDA(cudaEventRecord(pl->entry, cs));
    HB_CUDA(cudaStreamWaitEvent(st, pl->entry, 0));
  }
  if (s != HB_OK) return s;
  HB_LAUNCH_CHECK("posterior_mace");
  return HB_OK;
}

}  // namespace hb
