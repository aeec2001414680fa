// Posterior variance contraction V = K* Linv^T, row sums of squares, on the Hopper tensor cores (wgmma).  The operands are
// two-level fp16 splits (instead of the 3xTF32 hi/lo pairs of the fit GEMMs, tcgemm.cu),
//     x * scale = h0 + h1 / 2048,   h0 = rn_fp16(x * scale),  h1 = rn_fp16((x * scale - h0) * 2048)
// (11 + 11 significant bits, the same 2^-22 as tf32 hi/lo; `scale` a power of two per matrix so that the largest entry
// sits well inside the fp16 range, and the 2048-fold residual keeps small entries out of the subnormals).  f16 MMAs
// run at TWICE the tf32 rate and an fp16 k-block of 64 elements occupies the same 128-byte swizzle row as 32 tf32
// elements, so the contraction costs half the tensor time and half the L2 / shared-memory bytes per MAC:
//     main  = sum h0a h0b            (accumulator 0)
//     cross = sum h0a h1b + h1a h0b  (accumulator 1)         v = (main + cross / 2048) / (scale_a scale_b)
// The dropped h1a h1b term is 2^-22 relative, as the lo*lo term of 3xTF32.  fp32 accumulation in registers (half as
// many accumulate steps per dot product).  A 128 x 128 tile keeps both accumulators of a consumer thread in 128
// registers.  Pipeline protocol: tc_common.cuh.
#include <cuda.h>

#include <cuda_fp16.h>

#include <algorithm>
#include <map>
#include <vector>

#include "h16.cuh"
#include "kernels.h"
#include "tc_common.cuh"
#include "vnorm_sched.h"

namespace hb {
namespace h16 {
using namespace hb::tc;

constexpr int UK = 16;             // wgmma K for f16
constexpr int STAGES = 3;
constexpr uint32_t A_BYTES = BM * BK * 2;                  // 16 KiB
constexpr uint32_t B_BYTES = BN * BK * 2;                  // 16 KiB
constexpr uint32_t B_SLICE = B_BYTES / CLUSTER;            // the Linv rows of a box that one CTA loads for the cluster
constexpr uint32_t STAGE_BYTES = 2 * A_BYTES + 2 * B_BYTES;  // 64 KiB
constexpr uint32_t SMEM_BYTES = STAGES * STAGE_BYTES + 1024 /*align*/ + 256 /*barriers*/;
static_assert(B_SLICE % 1024 == 0, "a multicast Linv slice must start on a SWIZZLE_128B atom (8 rows x 128 B)");

__device__ __forceinline__ bool next_tile(const int32_t *__restrict__ list, int it, int &p, int &J) {
  const int code = __ldg(list + it);
  p = code >> 16;
  J = code & 0xffff;
  return code >= 0;
}

// Clusters of CLUSTER CTAs (schedule: vnorm_sched.h).  The CTAs of a cluster run the same column tile J on neighbouring
// bands, so they need the same Linv boxes: each producer loads 1 / CLUSTER of the rows of every Linv box and multicasts it
// to the same stage offset in every CTA of the cluster, signalling each CTA's own full[stage].  The K* boxes stay per CTA.
// Because a producer writes into its peers' stages, a stage is free only when the consumers of ALL CTAs of the cluster
// have released it: one lane per consumer warp arrives on empty[stage] of every CTA.
__global__ void __launch_bounds__(384, 1)
vnorm_h16_kernel(const __grid_constant__ CUtensorMap map_a_hi, const __grid_constant__ CUtensorMap map_a_lo,
                 const __grid_constant__ CUtensorMap map_b_hi, const __grid_constant__ CUtensorMap map_b_lo, int np,
                 const int32_t *__restrict__ sched, int sched_len, int64_t mc_pad, float *__restrict__ vpart,
                 const float *__restrict__ hyp, const float *__restrict__ scale_b) {
  extern __shared__ unsigned char smem_raw[];
  const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;   // SWIZZLE_128B tiles need 1024-byte alignment
  const uint32_t full_bar = base + STAGES * STAGE_BYTES;          // [STAGES] 8-byte mbarriers after the tiles
  const uint32_t empty_bar = full_bar + 8 * STAGES;               // [STAGES]
  const int wg = threadIdx.x >> 7;
  const int rank = (int)cluster_ctarank();
  const int32_t *my_tiles = sched + (int64_t)cluster_id_x() * sched_len;

  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(full_bar + 8 * s, 1);                             // the local producer's arrive + all bytes
      mbar_init(empty_bar + 8 * s, CLUSTER * CONSUMER_THREADS / 32);   // one lane per consumer warp of the cluster
    }
    mbar_init_fence();
  }
  cluster_sync();   // the peers' barriers are initialised before any multicast or remote arrive reaches them

  if (threadIdx.x == 0) {
    // ------------------------------------------------------------------ TMA producer
    int stage = 0;
    uint32_t phase = 0;
    for (int it = 0;; ++it) {
      int p, J;
      if (!next_tile(my_tiles, it, p, J)) break;
      const int rt = p * CLUSTER + rank;
      const int kend = min((J + 1) * BN, np);
      for (int k0 = 0; k0 < kend; k0 += BK) {
        mbar_wait(empty_bar + 8 * stage, phase ^ 1u);
        const uint32_t sb = base + stage * STAGE_BYTES;
        const uint32_t fb = full_bar + 8 * stage;
        // the whole stage, the peers' multicast slices included (their complete_tx may land before this expect_tx; the
        // phase cannot complete before this arrive)
        mbar_expect_tx(fb, STAGE_BYTES);
        tma_load_2d(sb, &map_a_hi, fb, k0, rt * BM);
        tma_load_2d(sb + A_BYTES, &map_a_lo, fb, k0, rt * BM);
        const uint32_t slice = rank * B_SLICE;
        const int brow = J * BN + rank * (BN / CLUSTER);
        tma_load_2d_multicast(sb + 2 * A_BYTES + slice, &map_b_hi, fb, k0, brow, (1u << CLUSTER) - 1);
        tma_load_2d_multicast(sb + 2 * A_BYTES + B_BYTES + slice, &map_b_lo, fb, k0, brow, (1u << CLUSTER) - 1);
        if (++stage == STAGES) {
          stage = 0;
          phase ^= 1u;
        }
      }
    }
  } else if (wg > 0) {
    // ------------------------------------------------------------------ consumers: 64 candidate rows each
    const int half = wg - 1;
    const int w = (threadIdx.x >> 5) & 3, lane = threadIdx.x & 31;
    const uint32_t a_off = (uint32_t)half * 64 * BK * 2;
    const float inv = 1.0f / (pow2_scale(hyp[2], 1) * scale_b[0]);   // undo the operand scales (exact: powers of two)
    const float lo_w = inv * (1.0f / 2048.0f);
    // after the warp's wgmma.wait_group: the MMAs that read the stage have retired for the whole warp
    auto release = [&](int s) {
      if (lane == 0)
        for (int c = 0; c < CLUSTER; ++c) mbar_arrive_cluster(empty_bar + 8 * s, (uint32_t)c);
    };
    int stage = 0;
    uint32_t phase = 0;
    // two accumulators per tile: MAIN takes hi*hi only, CROSS the two small hi*lo terms.  The tensor core's fp32
    // accumulation truncates; keeping the 2^-11-sized cross terms out of the main sum cuts the truncations on it by 3x.
    float acc_main[BN / 2], acc_cross[BN / 2];
    for (int it = 0;; ++it) {
      int p, J;
      if (!next_tile(my_tiles, it, p, J)) break;
      const int rt = p * CLUSTER + rank;
      const int kend = min((J + 1) * BN, np);
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) {
        acc_main[i] = 0.0f;
        acc_cross[i] = 0.0f;
      }
      int prev = -1;
      for (int k0 = 0; k0 < kend; k0 += BK) {
        mbar_wait(full_bar + 8 * stage, phase);              // TMA bytes have landed
        const uint32_t sb = base + stage * STAGE_BYTES;
        const uint64_t da_hi = make_sw128_desc(sb + a_off);
        const uint64_t da_lo = make_sw128_desc(sb + A_BYTES + a_off);
        const uint64_t db_hi = make_sw128_desc(sb + 2 * A_BYTES);
        const uint64_t db_lo = make_sw128_desc(sb + 2 * A_BYTES + B_BYTES);
        fence_regs(acc_main);
        fence_regs(acc_cross);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < BK / UK; ++k) {
          const uint64_t adv = (uint64_t)((k * UK * 2) >> 4);   // 32 bytes per k-step inside the 128-byte swizzle row
          wgmma_f16_n128(acc_main, da_hi + adv, db_hi + adv);
          wgmma_f16_n128(acc_cross, da_hi + adv, db_lo + adv);
          wgmma_f16_n128(acc_cross, da_lo + adv, db_hi + adv);
        }
        wgmma_commit();
        wgmma_wait<1>();                                     // the previous k-block's MMAs have retired
        fence_regs(acc_main);
        fence_regs(acc_cross);
        if (prev >= 0) release(prev);
        prev = stage;
        if (++stage == STAGES) {
          stage = 0;
          phase ^= 1u;
        }
      }
      wgmma_wait<0>();
      fence_regs(acc_main);
      fence_regs(acc_cross);
      release(prev);

      // epilogue: thread holds rows r and r + 8 of its warpgroup's 64, two columns of every 8; the 4 lanes of a quad share
      // the rows
      float s0 = 0.f, s1 = 0.f, t0 = 0.f, t1 = 0.f;
#pragma unroll
      for (int j = 0; j < BN / 8; ++j) {
        const float x0 = fmaf(acc_cross[4 * j + 0], lo_w, acc_main[4 * j + 0] * inv);
        const float x1 = fmaf(acc_cross[4 * j + 1], lo_w, acc_main[4 * j + 1] * inv);
        const float x2 = fmaf(acc_cross[4 * j + 2], lo_w, acc_main[4 * j + 2] * inv);
        const float x3 = fmaf(acc_cross[4 * j + 3], lo_w, acc_main[4 * j + 3] * inv);
        s0 = fmaf(x0, x0, s0);
        s1 = fmaf(x1, x1, s1);
        t0 = fmaf(x2, x2, t0);
        t1 = fmaf(x3, x3, t1);
      }
      float s = s0 + s1, t = t0 + t1;
      s += __shfl_xor_sync(0xffffffffu, s, 1);
      t += __shfl_xor_sync(0xffffffffu, t, 1);
      s += __shfl_xor_sync(0xffffffffu, s, 2);
      t += __shfl_xor_sync(0xffffffffu, t, 2);
      if ((lane & 3) == 0) {
        float *out = vpart + (int64_t)J * mc_pad + (int64_t)rt * BM + half * 64 + w * 16 + (lane >> 2);
        out[0] = s;
        out[8] = t;
      }
    }
  }
  // no CTA leaves while a peer may still multicast into its shared memory or arrive on its barriers
  cluster_sync();
}


// fp16 matrix [rows, cols] row-major -> 2-D tiled map with boxes [box_rows x 64 halfs], 128-byte swizzle
static bool make_map(CUtensorMap *m, const __half *ptr, uint64_t rows, uint64_t cols, uint32_t box_rows) {
  EncodeTiledFn enc = encode_fn();
  if (!enc) return false;
  cuuint64_t gdim[2] = {cols, rows};
  cuuint64_t gstride[1] = {cols * sizeof(__half)};
  cuuint32_t box[2] = {(cuuint32_t)BK, box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<__half *>(ptr), gdim, gstride, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS;
}

}  // namespace h16

// ---- host side: schedule tables (device-resident, built once per shape and device) and the launcher
namespace h16 {

// The most clusters a contraction launch takes; the SMs it leaves free run the next chunk's K* (posterior.cu).  30 is
// all that fit on a 132-SM H100 SXM.  Capping at 28 or 26 to give K* more SMs measured slower: scoring step 12.03 / 11.94
// ms at 30, 12.41 / 12.37 at 28, 12.44 / 12.55 at 26 (bench.py, two runs each; H100 80GB HBM3, 700 W power limit, power-
// capped at ~1.55-1.6 GHz): the contraction lost time in proportion to its SMs (2.60, 2.80, 2.93 ms per launch) while
// the K* it let run alongside gained less.
constexpr int MAX_CLUSTERS = 30;

struct SchedEntry {
  int32_t *dev = nullptr;
  int len = 0;
};
struct SchedKey {
  int dev, np, n_rt, clusters, cluster;
  bool operator<(const SchedKey &o) const {
    if (dev != o.dev) return dev < o.dev;
    if (np != o.np) return np < o.np;
    if (n_rt != o.n_rt) return n_rt < o.n_rt;
    if (clusters != o.clusters) return clusters < o.clusters;
    return cluster < o.cluster;
  }
};

static const SchedEntry *get_schedule(int dev, int np, int n_rt, int clusters, cudaStream_t st) {
  static std::map<SchedKey, SchedEntry> cache;
  const SchedKey key{dev, np, n_rt, clusters, CLUSTER};
  auto it = cache.find(key);
  if (it != cache.end()) return &it->second;
  SchedEntry e;
  const std::vector<int32_t> flat = build_schedule(np, n_rt, clusters, &e.len);
  if (cudaMalloc(&e.dev, flat.size() * sizeof(int32_t)) != cudaSuccess) return nullptr;
  if (cudaMemcpyAsync(e.dev, flat.data(), flat.size() * sizeof(int32_t), cudaMemcpyHostToDevice, st) != cudaSuccess ||
      cudaStreamSynchronize(st) != cudaSuccess)   // `flat` is pageable and dies with this frame
    return nullptr;
  return &(cache[key] = e);
}

}  // namespace h16

// ks_h0 / ks_h1 [ks_rows, np] fp16 split of K* (scale 2^k from the outputscale hyp[2]); linv_h0 / linv_h1 [np, np] fp16 split
// of Linv with the device scalar scale_b; ks_rows and mc_pad multiples of 128.  The rows of K* and vpart up to
// round_up(mc_pad, CLUSTER * BM) must exist: the last cluster runs padding bands there when the band count is not a
// multiple of CLUSTER.
int launch_vnorm_h16(const __half *ks_h0, const __half *ks_h1, int64_t ks_rows, const __half *linv_h0, const __half *linv_h1,
                     const float *scale_b, const float *hyp, int64_t np, int64_t mc_pad, int64_t vpart_stride, float *vpart,
                     cudaStream_t st) {
  using namespace h16;
  const int64_t rows = round_up(mc_pad, (int64_t)CLUSTER * BM);   // bands rounded up to whole clusters
  if (np % TILE != 0 || mc_pad % BM != 0 || rows > ks_rows || rows > vpart_stride || np > 65535 * BN || mc_pad / BM > 32767)
    return HB_ERR_INVALID;
  static PerDevice once;   // aux: the most clusters of this kernel that fit on the device at once
  bool fresh = false;
  const int dev = once.slot(&fresh);
  if (dev < 0) return HB_ERR_CUDA;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = CLUSTER;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(CLUSTER);
  cfg.blockDim = dim3(384);
  cfg.dynamicSmemBytes = SMEM_BYTES;
  cfg.stream = st;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  if (fresh) {   // per DEVICE: cudaFuncSetAttribute applies to the current device only
    HB_CUDA(cudaFuncSetAttribute(vnorm_h16_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM_BYTES));
    HB_CUDA(cudaOccupancyMaxActiveClusters(&once.aux[dev], vnorm_h16_kernel, &cfg));
    if (once.aux[dev] < 1) {
      set_error(cudaErrorInvalidConfiguration, "vnorm_h16: no cluster fits on the device");
      return HB_ERR_CUDA;
    }
    once.done[dev] = true;
  }
  CUtensorMap ma_hi, ma_lo, mb_hi, mb_lo;
  if (!make_map(&ma_hi, ks_h0, (uint64_t)ks_rows, (uint64_t)np, BM) ||
      !make_map(&ma_lo, ks_h1, (uint64_t)ks_rows, (uint64_t)np, BM) ||
      !make_map(&mb_hi, linv_h0, (uint64_t)np, (uint64_t)np, BN / CLUSTER) ||
      !make_map(&mb_lo, linv_h1, (uint64_t)np, (uint64_t)np, BN / CLUSTER)) {
    set_error(cudaErrorUnknown, "cuTensorMapEncodeTiled");
    return HB_ERR_CUDA;
  }
  const int n_rt = (int)(mc_pad / BM);
  const int n_j = (int)ceil_div(np, BN);
  const int units = (int)(rows / BM / CLUSTER) * n_j;
  const int clusters = std::min({once.aux[dev], units, MAX_CLUSTERS});
  const SchedEntry *sc = get_schedule(dev, (int)np, n_rt, clusters, st);
  if (!sc) {
    set_error(cudaErrorMemoryAllocation, "vnorm_h16 schedule table");
    return HB_ERR_CUDA;
  }
  cfg.gridDim = dim3((unsigned)(clusters * CLUSTER));
  prof_begin(st);
  const cudaError_t e = cudaLaunchKernelEx(&cfg, vnorm_h16_kernel, ma_hi, ma_lo, mb_hi, mb_lo, (int)np, (const int32_t *)sc->dev,
                                           sc->len, vpart_stride, vpart, hyp, scale_b);
  prof_end(st);
  if (e != cudaSuccess) {
    set_error(e, "vnorm_h16 cluster launch");
    return HB_ERR_CUDA;
  }
  count_launches(1);
  HB_LAUNCH_CHECK("vnorm_h16");
  return HB_OK;
}

// ---- operand preparation for the prediction state: |Linv| maximum -> power-of-two scale -> two-level fp16 split
__global__ void absmax_kernel(const float *__restrict__ x, int64_t n4, unsigned int *__restrict__ out) {
  float m = 0.0f;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (int64_t)gridDim.x * blockDim.x) {
    const float4 v = reinterpret_cast<const float4 *>(x)[i];
    m = fmaxf(m, fmaxf(fmaxf(fabsf(v.x), fabsf(v.y)), fmaxf(fabsf(v.z), fabsf(v.w))));
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0 && m > 0.0f) atomicMax(out, __float_as_uint(m));   // non-negative floats order as integers
}
__global__ void split_h16_kernel(const float *__restrict__ x, int64_t n4, __half *__restrict__ h0, __half *__restrict__ h1,
                                 float *__restrict__ scale_slot) {
  // scale_slot[1] = max |x| (written by absmax_kernel); every thread derives the same power-of-two scale from it and
  // one thread publishes it in scale_slot[0] for the contraction's epilogue
  const float sc = pow2_scale(fmaxf(scale_slot[1], 1e-30f), 10);
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (int64_t)gridDim.x * blockDim.x) {
    const float4 v = reinterpret_cast<const float4 *>(x)[i];
    const float xv[4] = {v.x * sc, v.y * sc, v.z * sc, v.w * sc};
    __half a[4], b[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) split_h16(xv[j], a[j], b[j]);
    reinterpret_cast<uint2 *>(h0)[i] = make_uint2(pack_half2(a[0], a[1]), pack_half2(a[2], a[3]));
    reinterpret_cast<uint2 *>(h1)[i] = make_uint2(pack_half2(b[0], b[1]), pack_half2(b[2], b[3]));
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) scale_slot[0] = sc;
}

// Linv [np, np] fp32 -> h0 / h1 fp16 [np, np]; scale_slot: 2 floats of device scratch, [0] = scale on return
int launch_split_h16(const float *x, int64_t count, __half *h0, __half *h1, float *scale_slot, cudaStream_t st) {
  if (count % 4 != 0) return HB_ERR_INVALID;
  HB_CUDA(cudaMemsetAsync(scale_slot, 0, 2 * sizeof(float), st));
  const int blocks = (int)std::min<int64_t>(ceil_div(count / 4, 256), 1024);
  absmax_kernel<<<blocks, 256, 0, st>>>(x, count / 4, reinterpret_cast<unsigned int *>(scale_slot + 1));
  split_h16_kernel<<<blocks, 256, 0, st>>>(x, count / 4, h0, h1, scale_slot);
  count_launches(2);
  HB_LAUNCH_CHECK("split_h16");
  return HB_OK;
}

}  // namespace hb
