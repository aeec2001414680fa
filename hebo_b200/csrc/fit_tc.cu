// Tensor-core (wgmma, 3xTF32) versions of the n^3-class stages of one MLL epoch, expressed as tile tables for
// the generic kernel in tcgemm.cu.  Everything is arranged so that BOTH operands of every product are K-major:
// next to Linv (lower) its transpose U = Linv^T (upper) is maintained, products are formed so that the output is
// the operand the next stage needs, and the epilogue writes the hi/lo split (and the transposed split) directly.
//
//   Cholesky outer update   A[r, c >= ce] -= P P^T            A = B = P (panel rows, hi/lo copy)     RMW epilogue
//   inverse, level b        Tt  = U11 * L21^T                 A = U rows, B = L rows    k >= column tile
//                           X21 = -Linv22 * Tt^T              A = Linv rows, B = Tt rows k <= row tile
//                                 -> Linv (fp32 + hi/lo) and U = X21^T (hi/lo)
//   K^-1 = U U^T            lower tiles, k >= row tile        -> Kinv fp32
// (gpytorch's backward through the Cholesky MLL, HEBO/hebo/models/gp/gp.py:115, as explicit dense algebra.)
#include <vector>

#include "gemm_core.cuh"
#include "kernels.h"
#include "tcgemm.h"

namespace hb {

// tables live in device memory: the current device is part of the key (a process may drive more than one GPU)
static inline TcTableKey table_key(int op, int64_t np, int64_t p1, int64_t p2, const Batch &bt) {
  int dev = 0;
  cudaGetDevice(&dev);
  return TcTableKey{dev, op, np, p1, p2, bt.nout};
}

// ------------------------------------------------------------------------------------------ Cholesky outer update
int launch_chol_outer_update_tc(float *A, int64_t np, int64_t cb, int64_t ce, const TcBuffers &tc, cudaStream_t st,
                                const Batch &bt) {
  const int64_t K = ce - cb;
  // hi/lo copy of the finished panel rows [ce, np) x [cb, ce) -> P[r][c - cb], leading dimension K
  int s = launch_split_region(A + ce * np + cb, np, tc.P_hi + ce * K, tc.P_lo + ce * K, K, np - ce, K, st, bt);
  if (s != HB_OK) return s;
  int ntiles = 0;
  const TcTableKey key = table_key(1, np, cb, ce, bt);
  const TcTile *tiles = tc_table_lookup(key, &ntiles);
  if (!tiles) {
    std::vector<TcTile> host;
    for (int64_t c0 = ce; c0 < np; c0 += 256)          // widest (longest) tile columns first
      for (int64_t r0 = (c0 / GT) * GT; r0 < np; r0 += GT) {
        if (c0 >= r0 + GT) continue;                    // tile entirely above the diagonal
        host.push_back(TcTile{(int)r0, 0, (int)c0, 0, 0, (int)K, (int)r0, (int)c0});
      }
    tiles = tc_table_store(key, host, &ntiles);
    if (!tiles) return HB_ERR_CUDA;
  }
  TcOperand P{tc.P_hi, tc.P_lo, (uint64_t)np, (uint64_t)K, (uint64_t)K};
  TcEpilogue epi{};
  epi.mode = TC_EPI_RMW_SUB;
  epi.C = A;
  epi.ldc = np;
  epi.r0 = (int)ce;
  epi.ncols = (int)np;
  return launch_tcgemm(P, P, 256, tiles, ntiles, epi, st, bt);
}

// ------------------------------------------------------------------------------------------ triangular inverse
// base case: triinv_base2_kernel (cholesky.cu) inverts the 128x128 diagonal blocks into Linv (fp32 + hi/lo) and U (hi/lo)
int launch_tri_inverse_tc(const float *L, int64_t np, float *Linv, const TcBuffers &tc, bool zero_fill, cudaStream_t st,
                          const Batch &bt) {
  if (np <= 0 || np % GT != 0) return HB_ERR_INVALID;
  const size_t bytes = (size_t)np * np * sizeof(float);
  if (zero_fill) {   // the triangular complements are never written afterwards: once per workspace is enough
    HB_CUDA(memset_slices(Linv, 0, bytes, bt, st));
    HB_CUDA(memset_slices(tc.Linv_hi, 0, bytes, bt, st));
    HB_CUDA(memset_slices(tc.Linv_lo, 0, bytes, bt, st));
    HB_CUDA(memset_slices(tc.U_hi, 0, bytes, bt, st));
    HB_CUDA(memset_slices(tc.U_lo, 0, bytes, bt, st));
  }
  int s = launch_split_region(L, np, tc.L_hi, tc.L_lo, np, np, np, st, bt);
  if (s != HB_OK) return s;
  s = launch_triinv_base2(L, np, Linv, tc.Linv_hi, tc.Linv_lo, tc.U_hi, tc.U_lo, st, bt);
  if (s != HB_OK) return s;
  TcOperand opL{tc.L_hi, tc.L_lo, (uint64_t)np, (uint64_t)np, (uint64_t)np};
  TcOperand opU{tc.U_hi, tc.U_lo, (uint64_t)np, (uint64_t)np, (uint64_t)np};
  TcOperand opLinv{tc.Linv_hi, tc.Linv_lo, (uint64_t)np, (uint64_t)np, (uint64_t)np};
  TcOperand opT{tc.T_hi, tc.T_lo, (uint64_t)np, (uint64_t)np, (uint64_t)np};
  for (int64_t b = GT; b < np; b *= 2) {
    const int bn = b >= 256 ? 256 : 128;
    for (int phase = 0; phase < 2; ++phase) {
      int ntiles = 0;
      const TcTableKey key = table_key(2 + phase, np, b, 0, bt);
      const TcTile *tiles = tc_table_lookup(key, &ntiles);
      if (!tiles) {
        std::vector<TcTile> host;
        for (int64_t s0 = 0; s0 + b < np; s0 += 2 * b) {
          const int64_t s2 = (np - s0 - b) < b ? (np - s0 - b) : b;
          if (phase == 0) {
            // Tt[c][r] = sum_{k >= c} U[s0+c][s0+k] * L[s0+b+r][s0+k]
            for (int64_t c = 0; c < b; c += GT)
              for (int64_t r = 0; r < s2; r += bn)
                host.push_back(TcTile{(int)(s0 + c), (int)s0, (int)(s0 + b + r), (int)s0, (int)c, (int)b,
                                      (int)(s0 + c), (int)(s0 + b + r)});
          } else {
            // X21[r][c] = -sum_{k <= r} Linv[s0+b+r][s0+b+k] * Tt[s0+c][s0+b+k]
            for (int64_t r = s2 - GT; r >= 0; r -= GT)      // longest k ranges first
              for (int64_t c = 0; c < b; c += bn) {
                const int64_t kend = (r + GT) < s2 ? (r + GT) : s2;
                host.push_back(TcTile{(int)(s0 + b + r), (int)(s0 + b), (int)(s0 + c), (int)(s0 + b), 0, (int)kend,
                                      (int)(s0 + b + r), (int)(s0 + c)});
              }
          }
        }
        tiles = tc_table_store(key, host, &ntiles);
        if (!tiles) return HB_ERR_CUDA;
      }
      TcEpilogue epi{};
      epi.mode = TC_EPI_STORE;
      epi.ldc = np;
      epi.ldct = np;
      epi.ncols = (int)np;
      if (phase == 0) {
        epi.sign = 1.0f;
        epi.C_hi = tc.T_hi;
        epi.C_lo = tc.T_lo;
        s = launch_tcgemm(opU, opL, bn, tiles, ntiles, epi, st, bt);
      } else {
        epi.sign = -1.0f;
        epi.C = Linv;
        epi.C_hi = tc.Linv_hi;
        epi.C_lo = tc.Linv_lo;
        epi.Ct_hi = tc.U_hi;
        epi.Ct_lo = tc.U_lo;
        s = launch_tcgemm(opLinv, opT, bn, tiles, ntiles, epi, st, bt);
      }
      if (s != HB_OK) return s;
    }
  }
  return HB_OK;
}

// ------------------------------------------------------------------------------------------ K^-1 = U U^T
int launch_kinv_tc(int64_t np, float *Kinv, const TcBuffers &tc, cudaStream_t st, const Batch &bt) {
  if (np <= 0 || np % GT != 0) return HB_ERR_INVALID;
  int ntiles = 0;
  const TcTableKey key = table_key(4, np, 0, 0, bt);
  const TcTile *tiles = tc_table_lookup(key, &ntiles);
  if (!tiles) {
    std::vector<TcTile> host;
    for (int64_t r0 = 0; r0 < np; r0 += GT)                 // small r0 = long k range first
      for (int64_t c0 = 0; c0 < r0 + GT; c0 += 256)
        host.push_back(TcTile{(int)r0, 0, (int)c0, 0, (int)r0, (int)np, (int)r0, (int)c0});
    tiles = tc_table_store(key, host, &ntiles);
    if (!tiles) return HB_ERR_CUDA;
  }
  TcOperand opU{tc.U_hi, tc.U_lo, (uint64_t)np, (uint64_t)np, (uint64_t)np};
  TcEpilogue epi{};
  epi.mode = TC_EPI_STORE;
  epi.sign = 1.0f;
  epi.C = Kinv;
  epi.ldc = np;
  epi.ncols = (int)np;
  return launch_tcgemm(opU, opU, 256, tiles, ntiles, epi, st, bt);
}

}  // namespace hb
