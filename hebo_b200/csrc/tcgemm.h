// Interface of the generic 3xTF32 tensor-core GEMM (tcgemm.cu).
#pragma once
#include <stdint.h>

#include <vector>

#include "common.cuh"

namespace hb {

struct TcTile {       // one 128 x BN output tile
  int a_row, a_k0;    // A box: rows [a_row, a_row+128), columns a_k0 + k
  int b_row, b_k0;    // B box: rows [b_row, b_row+BN),  columns b_k0 + k
  int kbeg, kend;     // k range (multiples of 32, kend > kbeg)
  int c_row, c_col;   // output tile origin
};

enum { TC_EPI_STORE = 0, TC_EPI_RMW_SUB = 1 };

struct TcEpilogue {
  int mode;
  float sign;               // STORE: C = sign * acc
  float *C;                 // fp32 output (STORE: optional; RMW_SUB: in/out)
  float *C_hi, *C_lo;       // optional 3xTF32 split of the output, leading dimension ldc
  float *Ct_hi, *Ct_lo;     // optional split of the TRANSPOSED output, leading dimension ldct
  int64_t ldc, ldct;
  int r0;                   // RMW_SUB: rows / columns below r0 are left untouched
  int ncols;                // columns >= ncols are never written (tile overhang)
};

struct TcOperand {          // K-major fp32 matrix given as a hi/lo pair
  const float *hi, *lo;
  uint64_t rows, cols, ld;
};

const TcTile *tc_table_lookup(uint64_t key, int *count);
const TcTile *tc_table_store(uint64_t key, const std::vector<TcTile> &host, int *count);
int launch_tcgemm(const TcOperand &A, const TcOperand &B, int bn, const TcTile *tiles, int ntiles, const TcEpilogue &epi,
                  cudaStream_t st);
int launch_split_region(const float *x, int64_t ldx, float *hi, float *lo, int64_t ldo, int64_t rows, int64_t cols,
                        cudaStream_t st);

}  // namespace hb
