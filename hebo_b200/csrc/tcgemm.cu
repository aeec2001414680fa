// Generic error-compensated (3xTF32) tensor-core GEMM for the n^3-class pieces of the GP fit:
//
//     C[tile] (op)= sum_{k in [kbeg, kend)} A[a_row + r][a_k0 + k] * B[b_row + c][b_k0 + k]
//
// Both operands K-major fp32, given as hi/lo split pairs (hi = rn_tf32(x), lo = x - hi).  Same machinery as
// vnorm_h16.cu (protocol: tc_common.cuh) -- TMA SWIZZLE_128B boxes, mbarrier full/empty ring, wgmma.mma_async kind tf32
// with fp32 accumulators in registers, warp-specialised persistent CTAs -- but driven by a TILE TABLE (built once per
// problem size on the host, cached on the device) so triangular k-ranges, batched sub-problems and odd shapes need no
// device-side index arithmetic, and with a store epilogue that can emit, from the accumulator registers:
//     fp32 C, the hi/lo split of C, and the hi/lo split of C^T -- or subtract the product from C in place (Cholesky
//     trailing update).
// Users: Cholesky outer trailing update (cholesky.cu), triangular inverse levels and K^-1 = U U^T (linalg.cu).
#include <cuda.h>

#include <map>
#include <vector>

#include "kernels.h"
#include "tc_common.cuh"
#include "tcgemm.h"

namespace hb {
namespace tcg {
using namespace hb::tc;

constexpr int BM = 128;            // rows per tile: two consumer warpgroups of 64
constexpr int BK = 32;             // fp32 elements per k-block = one 128-byte swizzle row
constexpr int UK = 8;              // wgmma K for tf32

template <int BN>
struct Cfg {
  static constexpr int STAGES = (BN == 256) ? 2 : 3;
  static constexpr uint32_t A_BYTES = BM * BK * 4;
  static constexpr uint32_t B_BYTES = BN * BK * 4;
  static constexpr uint32_t STAGE_BYTES = 2 * A_BYTES + 2 * B_BYTES;
  static constexpr uint32_t SMEM_BYTES = STAGES * STAGE_BYTES + 1024 + 256;
  static constexpr int ACC = BN / 2;                       // accumulator registers per consumer thread
};

template <int BN>
__device__ __forceinline__ void mma3(float (&acc)[BN / 2], uint64_t da_hi, uint64_t da_lo, uint64_t db_hi, uint64_t db_lo) {
  if constexpr (BN == 256) {
    wgmma_tf32_n256(acc, da_hi, db_hi);
    wgmma_tf32_n256(acc, da_hi, db_lo);
    wgmma_tf32_n256(acc, da_lo, db_hi);
  } else {
    wgmma_tf32_n128(acc, da_hi, db_hi);
    wgmma_tf32_n128(acc, da_hi, db_lo);
    wgmma_tf32_n128(acc, da_lo, db_hi);
  }
}

template <int BN>
__global__ void __launch_bounds__(384, 1)
tcgemm_kernel(const __grid_constant__ CUtensorMap map_a_hi, const __grid_constant__ CUtensorMap map_a_lo,
              const __grid_constant__ CUtensorMap map_b_hi, const __grid_constant__ CUtensorMap map_b_lo,
              const TcTile *__restrict__ tiles, int ntiles, TcEpilogue epi, int64_t wss) {
  using C = Cfg<BN>;
  extern __shared__ unsigned char smem_raw[];
  const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;   // SWIZZLE_128B tiles need 1024-byte alignment
  const uint32_t full_bar = base + C::STAGES * C::STAGE_BYTES;
  const uint32_t empty_bar = full_bar + 8 * C::STAGES;
  const int wg = threadIdx.x >> 7;

  if (threadIdx.x == 0) {
    for (int s = 0; s < C::STAGES; ++s) {
      mbar_init(full_bar + 8 * s, 1);
      mbar_init(empty_bar + 8 * s, CONSUMER_THREADS);
    }
    mbar_init_fence();
  }
  __syncthreads();

  if (wg == 0) {
    // ------------------------------------------------------------------ TMA producer
    if (threadIdx.x != 0) return;
    int stage = 0;
    uint32_t phase = 0;
    for (int t = blockIdx.x; t < ntiles; t += gridDim.x) {
      const TcTile tl = tiles[t];
      for (int k0 = tl.kbeg; k0 < tl.kend; k0 += BK) {
        mbar_wait(empty_bar + 8 * stage, phase ^ 1u);
        const uint32_t sb = base + stage * C::STAGE_BYTES;
        const uint32_t fb = full_bar + 8 * stage;
        mbar_expect_tx(fb, C::STAGE_BYTES);
        tma_load_3d(sb, &map_a_hi, fb, tl.a_k0 + k0, tl.a_row, tl.out);
        tma_load_3d(sb + C::A_BYTES, &map_a_lo, fb, tl.a_k0 + k0, tl.a_row, tl.out);
        tma_load_3d(sb + 2 * C::A_BYTES, &map_b_hi, fb, tl.b_k0 + k0, tl.b_row, tl.out);
        tma_load_3d(sb + 2 * C::A_BYTES + C::B_BYTES, &map_b_lo, fb, tl.b_k0 + k0, tl.b_row, tl.out);
        if (++stage == C::STAGES) {
          stage = 0;
          phase ^= 1u;
        }
      }
    }
    return;
  }

  // -------------------------------------------------------------------- consumers: 64 rows each
  const int half = wg - 1;
  const int w = (threadIdx.x >> 5) & 3, lane = threadIdx.x & 31;
  const uint32_t a_off = (uint32_t)half * 64 * BK * 4;    // this warpgroup's rows inside the A box
  int stage = 0;
  uint32_t phase = 0;
  float acc[C::ACC];
  for (int t = blockIdx.x; t < ntiles; t += gridDim.x) {
    const TcTile tl = tiles[t];
#pragma unroll
    for (int i = 0; i < C::ACC; ++i) acc[i] = 0.0f;
    int prev = -1;
    for (int k0 = tl.kbeg; k0 < tl.kend; k0 += BK) {
      mbar_wait(full_bar + 8 * stage, phase);
      const uint32_t sb = base + stage * C::STAGE_BYTES;
      const uint64_t da_hi = make_sw128_desc(sb + a_off);
      const uint64_t da_lo = make_sw128_desc(sb + C::A_BYTES + a_off);
      const uint64_t db_hi = make_sw128_desc(sb + 2 * C::A_BYTES);
      const uint64_t db_lo = make_sw128_desc(sb + 2 * C::A_BYTES + C::B_BYTES);
      fence_regs(acc);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < BK / UK; ++k) {
        const uint64_t adv = (uint64_t)((k * UK * 4) >> 4);   // 32 bytes per k-step inside the 128-byte swizzle row
        mma3<BN>(acc, da_hi + adv, da_lo + adv, db_hi + adv, db_lo + adv);
      }
      wgmma_commit();
      wgmma_wait<1>();                                         // the previous k-block's MMAs have retired
      fence_regs(acc);
      if (prev >= 0) mbar_arrive(empty_bar + 8 * prev);
      prev = stage;
      if (++stage == C::STAGES) {
        stage = 0;
        phase ^= 1u;
      }
    }
    wgmma_wait<0>();
    fence_regs(acc);
    mbar_arrive(empty_bar + 8 * prev);                         // tables never contain empty k ranges

    // epilogue from registers: thread holds rows rr and rr + 8, columns 8 j + cq, 8 j + cq + 1
    float *const Cb = slice(epi.C, wss, tl.out);
    float *const Cb_hi = slice(epi.C_hi, wss, tl.out), *const Cb_lo = slice(epi.C_lo, wss, tl.out);
    float *const Ctb_hi = slice(epi.Ct_hi, wss, tl.out), *const Ctb_lo = slice(epi.Ct_lo, wss, tl.out);
    const int64_t rr = (int64_t)tl.c_row + half * 64 + w * 16 + (lane >> 2);
    const int cq = 2 * (lane & 3);
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) {
      const int64_t col = (int64_t)tl.c_col + 8 * j + cq;
      if (col >= epi.ncols) continue;                          // tile overhangs the matrix edge
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int64_t row = rr + 8 * h;
        float v0 = acc[4 * j + 2 * h], v1 = acc[4 * j + 2 * h + 1];
        if (epi.mode == TC_EPI_RMW_SUB) {
          if (row >= epi.r0 && col >= epi.r0) {
            float2 *p = reinterpret_cast<float2 *>(Cb + row * epi.ldc + col);
            float2 cv = *p;
            cv.x -= v0;
            cv.y -= v1;
            *p = cv;
          }
          continue;
        }
        v0 *= epi.sign;
        v1 *= epi.sign;
        if (Cb) *reinterpret_cast<float2 *>(Cb + row * epi.ldc + col) = make_float2(v0, v1);
        if (Cb_hi || Ctb_hi) {
          float h0, l0, h1, l1;
          split1(v0, h0, l0);
          split1(v1, h1, l1);
          if (Cb_hi) {
            *reinterpret_cast<float2 *>(Cb_hi + row * epi.ldc + col) = make_float2(h0, h1);
            *reinterpret_cast<float2 *>(Cb_lo + row * epi.ldc + col) = make_float2(l0, l1);
          }
          if (Ctb_hi) {
            Ctb_hi[col * epi.ldct + row] = h0;
            Ctb_lo[col * epi.ldct + row] = l0;
            Ctb_hi[(col + 1) * epi.ldct + row] = h1;
            Ctb_lo[(col + 1) * epi.ldct + row] = l1;
          }
        }
      }
    }
  }
}

// [nout][rows][cols] with the outputs `slice` bytes apart; the box covers one output
static bool make_map(CUtensorMap *m, const float *ptr, uint64_t rows, uint64_t cols, uint64_t ld, uint32_t box_rows, int nout,
                     uint64_t slice) {
  EncodeTiledFn enc = encode_fn();
  if (!enc) return false;
  cuuint64_t gdim[3] = {cols, rows, (cuuint64_t)nout};
  cuuint64_t gstride[2] = {ld * sizeof(float), slice};
  cuuint32_t box[3] = {(cuuint32_t)BK, box_rows, 1};
  cuuint32_t estr[3] = {1, 1, 1};
  return enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, const_cast<float *>(ptr), gdim, gstride, box, estr,
             CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
             CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

// device-resident tile tables, cached by key (tables depend only on the padded size and the operation)
struct TableEntry {
  TcTile *dev = nullptr;
  int n = 0;
};
static std::map<TcTableKey, TableEntry> g_tables;

}  // namespace tcg

const TcTile *tc_table_lookup(const TcTableKey &key, int *count) {
  auto it = tcg::g_tables.find(key);
  if (it == tcg::g_tables.end()) return nullptr;
  *count = it->second.n;
  return it->second.dev;
}

const TcTile *tc_table_store(const TcTableKey &key, const std::vector<TcTile> &host, int *count) {
  std::vector<TcTile> all;
  all.reserve(host.size() * key.nout);
  for (const TcTile &t : host)
    for (int b = 0; b < key.nout; ++b) {
      all.push_back(t);
      all.back().out = b;
    }
  tcg::TableEntry e;
  e.n = (int)all.size();
  if (e.n == 0) return nullptr;
  if (cudaMalloc(&e.dev, sizeof(TcTile) * all.size()) != cudaSuccess) return nullptr;
  if (cudaMemcpy(e.dev, all.data(), sizeof(TcTile) * all.size(), cudaMemcpyHostToDevice) != cudaSuccess) return nullptr;
  tcg::g_tables[key] = e;
  *count = e.n;
  return e.dev;
}

int launch_tcgemm(const TcOperand &A, const TcOperand &B, int bn, const TcTile *tiles, int ntiles, const TcEpilogue &epi,
                  cudaStream_t st, const Batch &bt) {
  using namespace tcg;
  if (ntiles <= 0) return HB_OK;
  if (bn != 128 && bn != 256) return HB_ERR_INVALID;
  static PerDevice once;
  bool fresh = false;
  const int dev = once.slot(&fresh);
  if (dev < 0) return HB_ERR_CUDA;
  if (fresh) {
    HB_CUDA(cudaDeviceGetAttribute(&once.sms[dev], cudaDevAttrMultiProcessorCount, dev));
    HB_CUDA(cudaFuncSetAttribute(tcgemm_kernel<128>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)Cfg<128>::SMEM_BYTES));
    HB_CUDA(cudaFuncSetAttribute(tcgemm_kernel<256>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)Cfg<256>::SMEM_BYTES));
    once.done[dev] = true;
  }
  const int num_sms = once.sms[dev];
  if (bt.nout > 1 && (bt.ws <= 0 || bt.ws % 16 != 0)) return HB_ERR_INVALID;
  // (one output: the outermost dimension has extent 1 and its stride is never applied; any legal value will do)
  const uint64_t sl = bt.nout > 1 ? (uint64_t)bt.ws : (A.rows > B.rows ? A.rows : B.rows) * (A.ld > B.ld ? A.ld : B.ld) * 4;
  const int no = bt.nout;
  CUtensorMap ma_hi, ma_lo, mb_hi, mb_lo;
  if (!make_map(&ma_hi, A.hi, A.rows, A.cols, A.ld, BM, no, sl) || !make_map(&ma_lo, A.lo, A.rows, A.cols, A.ld, BM, no, sl) ||
      !make_map(&mb_hi, B.hi, B.rows, B.cols, B.ld, (uint32_t)bn, no, sl) ||
      !make_map(&mb_lo, B.lo, B.rows, B.cols, B.ld, (uint32_t)bn, no, sl)) {
    set_error(cudaErrorUnknown, "cuTensorMapEncodeTiled");
    return HB_ERR_CUDA;
  }
  const int grid = ntiles < num_sms ? ntiles : num_sms;
  if (bn == 256)
    tcgemm_kernel<256><<<grid, 384, Cfg<256>::SMEM_BYTES, st>>>(ma_hi, ma_lo, mb_hi, mb_lo, tiles, ntiles, epi, bt.ws);
  else
    tcgemm_kernel<128><<<grid, 384, Cfg<128>::SMEM_BYTES, st>>>(ma_hi, ma_lo, mb_hi, mb_lo, tiles, ntiles, epi, bt.ws);
  count_launches(1);
  HB_LAUNCH_CHECK("tcgemm");
  return HB_OK;
}

// element-wise split of a sub-matrix: src/hi/lo may have different leading dimensions
__global__ void split_region_kernel(const float *__restrict__ x, int64_t ldx, float *__restrict__ hi, float *__restrict__ lo,
                                    int64_t ldo, int64_t rows, int64_t cols4, int64_t wss) {
  x = slice(x, wss, blockIdx.z);   // output (Batch)
  hi = slice(hi, wss, blockIdx.z);
  lo = slice(lo, wss, blockIdx.z);
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= rows * cols4) return;
  const int64_t r = i / cols4, c4 = i - r * cols4;
  const float4 v = *reinterpret_cast<const float4 *>(x + r * ldx + c4 * 4);
  float4 h, l;
  tcg::split1(v.x, h.x, l.x);
  tcg::split1(v.y, h.y, l.y);
  tcg::split1(v.z, h.z, l.z);
  tcg::split1(v.w, h.w, l.w);
  *reinterpret_cast<float4 *>(hi + r * ldo + c4 * 4) = h;
  *reinterpret_cast<float4 *>(lo + r * ldo + c4 * 4) = l;
}

int launch_split_region(const float *x, int64_t ldx, float *hi, float *lo, int64_t ldo, int64_t rows, int64_t cols,
                        cudaStream_t st, const Batch &bt) {
  if (rows <= 0 || cols <= 0) return HB_OK;
  if (cols % 4 != 0) return HB_ERR_INVALID;
  const int64_t tot = rows * (cols / 4);
  split_region_kernel<<<dim3((unsigned)ceil_div(tot, 256), 1, (unsigned)bt.nout), 256, 0, st>>>(x, ldx, hi, lo, ldo, rows,
                                                                                                cols / 4, bt.ws);
  count_launches(1);
  HB_LAUNCH_CHECK("split_region");
  return HB_OK;
}

}  // namespace hb
