// Interface of the generic 3xTF32 tensor-core GEMM (tcgemm.cu).
#pragma once
#include <stdint.h>

#include <vector>

#include "kernels.h"

namespace hb {

struct TcTile {       // one 128 x BN output tile
  int a_row, a_k0;    // A box: rows [a_row, a_row+128), columns a_k0 + k
  int b_row, b_k0;    // B box: rows [b_row, b_row+BN),  columns b_k0 + k
  int kbeg, kend;     // k range (multiples of 32, kend > kbeg)
  int c_row, c_col;   // output tile origin
  int out;            // output of the batch (kernels.h Batch): every operand and C are read / written in its slice
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

// Tile tables are built once per (device, operation, padded size, operation parameters, outputs) and cached on the device.
struct TcTableKey {
  int dev, op;
  int64_t np, p1, p2;
  int nout;
  bool operator<(const TcTableKey &o) const {
    if (dev != o.dev) return dev < o.dev;
    if (op != o.op) return op < o.op;
    if (np != o.np) return np < o.np;
    if (p1 != o.p1) return p1 < o.p1;
    if (p2 != o.p2) return p2 < o.p2;
    return nout < o.nout;
  }
};
const TcTile *tc_table_lookup(const TcTableKey &key, int *count);
// `host` lists the tiles of one output; the stored table repeats each of them for outputs 0 .. nout-1 in turn, so the
// outputs' tiles are interleaved and the table keeps its longest-first order
const TcTile *tc_table_store(const TcTableKey &key, const std::vector<TcTile> &host, int *count);
// one persistent launch over the tiles of every output; the operands' TMA maps are 3-D with the output outermost (stride
// bt.ws bytes), the epilogue offsets C by the tile's output times bt.ws
int launch_tcgemm(const TcOperand &A, const TcOperand &B, int bn, const TcTile *tiles, int ntiles, const TcEpilogue &epi,
                  cudaStream_t st, const Batch &bt);
int launch_split_region(const float *x, int64_t ldx, float *hi, float *lo, int64_t ldo, int64_t rows, int64_t cols,
                        cudaStream_t st, const Batch &bt);

}  // namespace hb
