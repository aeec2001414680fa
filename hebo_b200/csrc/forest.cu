// Random-forest surrogate (HEBO/hebo/models/rf/rf.py:19-56 over sklearn's RandomForestRegressor with its defaults):
// exact CART growth of every tree of every output in one launch, and forest scoring of candidates.
//
// Fit.  rf_prep_kernel lists each output's finite-y rows; rf_sort_kernel sorts every numeric column once by (value, row)
// (one CTA per column, a bitonic sort of 64-bit keys in shared memory); one-hot columns need no sort, since the stable
// order of a 0/1 column is its 0 rows then its 1 rows, each in row order.  rf_grow_kernel then runs one CTA per tree slot
// (trees beyond RF_SLOTS wait for a free slot).  A tree grows level by level on the device: every in-bag row carries its
// node, and for each feature a warp filters the presorted order into per-node segments (stable: a warp walks the order 32
// rows at a time and ranks rows of the same node with __match_any_sync), then each lane scans whole segments of its nodes
// sequentially in fp64, left to right, evaluating every valid cut.  Every sum has that one order; the cross-warp arg-max
// is a maximum under a total order (proxy, then lowest feature, then lowest cut), so a fit is bit-identical run to run.
// The only atomics are integer increments of the bootstrap counts.
//
// Predict.  One thread per (candidate, output) walks the trees in index order, twice: the first walk sums the leaf values
// sequentially (sklearn's forest mean) and pairwise (numpy's mean inside np.var), the second sums the squared deviations
// pairwise.  Thresholds are compared in fp32 as RD32(t), which takes exactly the decisions of the fp64 comparison.
#include <float.h>

#include <algorithm>
#include <vector>

#include "kernels.h"

namespace hb {

constexpr int RF_THREADS = 256;
constexpr int RF_WARPS = RF_THREADS / 32;
constexpr int RF_SLOTS = 264;            // concurrent tree CTAs (two per SM of a 132-SM H100); fixes the workspace size
constexpr int RF_SORT_THREADS = 1024;
constexpr int RF_PRED_THREADS = 128;
constexpr uint32_t RF_PHILOX_TAG = 0x52460000u;   // word 3 of the bootstrap counter ("RF")
constexpr double RF_FEATURE_THRESHOLD = 1e-7;     // sklearn _splitter.pyx FEATURE_THRESHOLD

// ------------------------------------------------------------------------------------------------ forest layout
// [header int32 x 8][uniq int32 [ne] | oh int32 [woh]][ncount int32 [B T]][nodes int4 [B T cap]][thr64 [B T cap]]
// [val64 [B T cap]], every block 256-byte aligned.  header = {cap, B, T, woh, ne, 0, 0, 0}.
struct RfForest {
  int cap, B, T, woh, ne;
  int32_t *uniq, *oh, *ncount;
  int4 *nodes;
  double *thr64, *val64;
};

__host__ __device__ inline int64_t rf_align(int64_t b) { return (b + 255) / 256 * 256; }

__host__ __device__ inline int64_t rf_forest_carve(unsigned char *base, int cap, int B, int T, int ne, int woh,
                                                   RfForest *f) {
  int64_t o = 256;
  const int64_t o_tab = o;
  o += rf_align(4 * (int64_t)(ne + woh));
  const int64_t o_cnt = o;
  o += rf_align(4 * (int64_t)B * T);
  const int64_t nn = (int64_t)B * T * cap;
  const int64_t o_nodes = o;
  o += rf_align(16 * nn);
  const int64_t o_thr = o;
  o += rf_align(8 * nn);
  const int64_t o_val = o;
  o += rf_align(8 * nn);
  if (f) {
    f->cap = cap;
    f->B = B;
    f->T = T;
    f->woh = woh;
    f->ne = ne;
    f->uniq = (int32_t *)(base + o_tab);
    f->oh = f->uniq + ne;
    f->ncount = (int32_t *)(base + o_cnt);
    f->nodes = (int4 *)(base + o_nodes);
    f->thr64 = (double *)(base + o_thr);
    f->val64 = (double *)(base + o_val);
  }
  return o;
}

__device__ inline RfForest rf_forest_view(unsigned char *base) {
  const int32_t *h = (const int32_t *)base;
  RfForest f;
  rf_forest_carve(base, h[0], h[1], h[2], h[4], h[3], &f);
  return f;
}

// value of feature f of row i: numeric column f < dc, else one-hot column f - dc = category (code & 4095) of column code >> 12
__device__ __forceinline__ float rf_x(const float *Xc, const int32_t *Xe, int dc, int ne, const int32_t *oh, int64_t i,
                                      int f) {
  if (f < dc) return Xc[i * dc + f];
  const int code = oh[f - dc];
  return Xe[i * ne + (code >> 12)] == (code & 4095) ? 1.0f : 0.0f;
}

// leaf value of tree node table `nodes` at input row i
__device__ __forceinline__ double rf_tree_value(const int4 *nodes, const float *Xc, const int32_t *Xe, int dc, int ne,
                                                const int32_t *oh, int64_t i) {
  int4 nd = nodes[0];
  while (nd.x >= 0) {
    const float x = rf_x(Xc, Xe, dc, ne, oh, i, nd.x);
    nd = nodes[x <= __int_as_float(nd.y) ? nd.z : nd.w];
  }
  return __hiloint2double(nd.w, nd.z);
}

// numpy's pairwise_sum (numpy/_core/src/umath/loops_utils.h.src) of a[i0 .. i0 + n - 1], a[i] = f(i), visiting the
// elements in index order: n < 8 sequentially from 0; n <= 128 eight strided accumulators combined as
// ((r0 + r1) + (r2 + r3)) + ((r4 + r5) + (r6 + r7)), then the tail; above 128 the halves n2 = n / 2 - (n / 2) % 8, n - n2.
// D bounds the recursion depth: n <= 8192 needs 7 levels.
template <int D, class F>
__device__ __noinline__ double rf_pairwise(F &f, int i0, int n) {
  if (n < 8) {
    double r = 0.0;
    for (int i = 0; i < n; ++i) r += f(i0 + i);
    return r;
  }
  if (D == 0 || n <= 128) {
    double r[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) r[j] = f(i0 + j);
    int i = 8;
    for (; i < n - (n % 8); i += 8) {
#pragma unroll
      for (int j = 0; j < 8; ++j) r[j] += f(i0 + i + j);
    }
    double res = ((r[0] + r[1]) + (r[2] + r[3])) + ((r[4] + r[5]) + (r[6] + r[7]));
    for (; i < n; ++i) res += f(i0 + i);
    return res;
  }
  if constexpr (D > 0) {
    int n2 = n / 2;
    n2 -= n2 % 8;
    const double a = rf_pairwise<D - 1>(f, i0, n2);
    return a + rf_pairwise<D - 1>(f, i0 + n2, n - n2);
  }
  return 0.0;
}
constexpr int RF_PW_DEPTH = 8;

// ------------------------------------------------------------------------------------------------ fit workspace
struct RfSlot {
  int32_t *w, *nid, *ncnt, *oidx, *openk, *segoff, *cursor, *bfeat, *bcnt, *fw;
  float *fv, *fy;
  double *nW, *nS, *nQ, *bprox, *bthr, *bWL, *bSL, *bQL, *fwy;
};

__host__ __device__ inline int64_t rf_slot_carve(unsigned char *base, int n, RfSlot *s) {
  const int64_t cap = 2 * (int64_t)n - 1, nw = (int64_t)RF_WARPS * n;
  int64_t o = 0;
  auto take = [&](int64_t bytes) {
    unsigned char *p = base ? base + o : nullptr;
    o += rf_align(bytes);
    return p;
  };
  RfSlot t;
  t.w = (int32_t *)take(4 * (int64_t)n);
  t.nid = (int32_t *)take(4 * (int64_t)n);
  t.ncnt = (int32_t *)take(4 * cap);
  t.oidx = (int32_t *)take(4 * cap);
  t.openk = (int32_t *)take(4 * (int64_t)n);
  t.segoff = (int32_t *)take(4 * (int64_t)n);
  t.cursor = (int32_t *)take(4 * nw);
  t.bfeat = (int32_t *)take(4 * nw);
  t.bcnt = (int32_t *)take(4 * nw);
  t.fw = (int32_t *)take(4 * nw);
  t.fv = (float *)take(4 * nw);
  t.fy = (float *)take(4 * nw);
  t.nW = (double *)take(8 * cap);
  t.nS = (double *)take(8 * cap);
  t.nQ = (double *)take(8 * cap);
  t.bprox = (double *)take(8 * nw);
  t.bthr = (double *)take(8 * nw);
  t.bWL = (double *)take(8 * nw);
  t.bSL = (double *)take(8 * nw);
  t.bQL = (double *)take(8 * nw);
  t.fwy = (double *)take(8 * nw);
  if (s) *s = t;
  return o;
}

// [ord int32 [dc, n]][sval float [dc, n]][kept int32 [B, n]][nkept int32 [B]][sq double [B, n]][RF_SLOTS slots]
struct RfGlobal {
  int32_t *ord, *kept, *nkept;
  float *sval;
  double *sq;
  unsigned char *slots;
  int64_t slot_bytes;
  int nslots;
};

static int64_t rf_ws_carve(unsigned char *base, int n, int dc, int B, int T, RfGlobal *g) {
  int64_t o = 0;
  auto take = [&](int64_t bytes) {
    unsigned char *p = base ? base + o : nullptr;
    o += rf_align(bytes);
    return p;
  };
  RfGlobal t;
  t.ord = (int32_t *)take(4 * (int64_t)dc * n);
  t.sval = (float *)take(4 * (int64_t)dc * n);
  t.kept = (int32_t *)take(4 * (int64_t)B * n);
  t.nkept = (int32_t *)take(4 * (int64_t)B);
  t.sq = (double *)take(8 * (int64_t)B * n);
  t.slot_bytes = rf_slot_carve(nullptr, n, nullptr);
  t.nslots = (int)std::min<int64_t>((int64_t)B * T, RF_SLOTS);
  t.slots = take(t.slot_bytes * t.nslots);
  if (g) *g = t;
  return o;
}

// spec -> (dc, ne, woh, host tables uniq ++ oh); false outside the envelope
static bool rf_layout(const hb_rf_spec_t *s, int &dc, int &ne, int &woh, std::vector<int32_t> *tab) {
  if (!s || s->num_cont < 0 || s->num_enum < 0 || s->num_cont + s->num_enum <= 0) return false;
  if (s->num_enum > 0 && !s->num_uniqs) return false;
  if (s->num_cont > HB_RF_MAX_WIDTH || s->num_enum > HB_RF_MAX_WIDTH) return false;
  dc = s->num_cont;
  ne = s->num_enum;
  int64_t w = 0;
  for (int c = 0; c < ne; ++c) {
    if (s->num_uniqs[c] < 1 || s->num_uniqs[c] > HB_RF_MAX_WIDTH) return false;
    w += s->num_uniqs[c];
  }
  if (dc + w > HB_RF_MAX_WIDTH) return false;
  woh = (int)w;
  if (tab) {
    tab->clear();
    for (int c = 0; c < ne; ++c) tab->push_back(s->num_uniqs[c]);
    for (int c = 0; c < ne; ++c)
      for (int u = 0; u < s->num_uniqs[c]; ++u) tab->push_back((c << 12) | u);
  }
  return true;
}

// ------------------------------------------------------------------------------------------------ fit kernels
// kept[b] = the rows with finite y[:, b], in row order (filter_nan(..., 'all') per output column, util.py)
__global__ void rf_prep_kernel(const float *__restrict__ y, int n, int B, int32_t *kept, int32_t *nkept) {
  const int b = blockIdx.x, lane = threadIdx.x;
  int c = 0;
  for (int base = 0; base < n; base += 32) {
    const int i = base + lane;
    const bool ok = i < n && isfinite(y[(int64_t)i * B + b]);
    const unsigned bal = __ballot_sync(0xffffffffu, ok);
    if (ok) kept[(int64_t)b * n + c + __popc(bal & ((1u << lane) - 1))] = i;
    c += __popc(bal);
  }
  if (lane == 0) nkept[b] = c;
}

// stable order of numeric column f by (value, row): -0 sorts as +0; ord [dc, n] rows, sval [dc, n] their values
__global__ void __launch_bounds__(RF_SORT_THREADS) rf_sort_kernel(const float *__restrict__ Xc, int n, int dc,
                                                                  int32_t *ord, float *sval) {
  extern __shared__ unsigned long long keys[];
  const int f = blockIdx.x;
  int N = 1;
  while (N < n) N <<= 1;
  for (int i = threadIdx.x; i < N; i += blockDim.x) {
    unsigned long long k = ~0ull;
    if (i < n) {
      float v = Xc[(int64_t)i * dc + f];
      if (v == 0.0f) v = 0.0f;
      uint32_t u = __float_as_uint(v);
      u = (u & 0x80000000u) ? ~u : (u | 0x80000000u);
      k = ((unsigned long long)u << 32) | (uint32_t)i;
    }
    keys[i] = k;
  }
  __syncthreads();
  for (int size = 2; size <= N; size <<= 1) {
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      for (int i = threadIdx.x; i < N; i += blockDim.x) {
        const int j = i ^ stride;
        if (j > i) {
          const bool up = (i & size) == 0;
          const unsigned long long a = keys[i], c = keys[j];
          if ((a > c) == up) {
            keys[i] = c;
            keys[j] = a;
          }
        }
      }
      __syncthreads();
    }
  }
  for (int p = threadIdx.x; p < n; p += blockDim.x) {
    const unsigned long long k = keys[p];
    const int i = (int)(uint32_t)k;
    float v = Xc[(int64_t)i * dc + f];
    if (v == 0.0f) v = 0.0f;
    ord[(int64_t)f * n + p] = i;
    sval[(int64_t)f * n + p] = v;
  }
}

struct RfFitArgs {
  const float *Xc, *y;
  const int32_t *Xe, *counts;
  int n, dc, ne, width, B, T;
  uint64_t seed;
  RfGlobal g;
  unsigned char *forest;
};

__device__ __forceinline__ void rf_write_leaf(const RfForest &F, int64_t base, int k, double value) {
  F.nodes[base + k] = make_int4(-2, 0, __double2loint(value), __double2hiint(value));
  F.thr64[base + k] = -2.0;
  F.val64[base + k] = value;
}

__global__ void __launch_bounds__(RF_THREADS) rf_grow_kernel(const __grid_constant__ RfFitArgs a) {
  const int n = a.n, tid = threadIdx.x, warp = tid / 32, lane = tid % 32, dc = a.dc, ne = a.ne;
  RfSlot s;
  rf_slot_carve(a.g.slots + (int64_t)blockIdx.x * a.g.slot_bytes, n, &s);
  const RfForest F = rf_forest_view(a.forest);
  const int cap = F.cap;
  __shared__ int s_nopen, s_next;
  const unsigned lt = (1u << lane) - 1;
  for (int tt = blockIdx.x; tt < a.B * a.T; tt += gridDim.x) {
    const int b = tt / a.T, t = tt % a.T;
    const int64_t nb0 = (int64_t)tt * cap;
    // bootstrap weights: w_i = times row i is drawn among n_b draws with replacement from output b's kept rows
    for (int i = tid; i < n; i += blockDim.x) {
      int w = 0;
      if (a.counts && isfinite(a.y[(int64_t)i * a.B + b])) w = max(0, a.counts[(int64_t)tt * n + i]);
      s.w[i] = w;
      s.nid[i] = 0;
    }
    __syncthreads();
    if (!a.counts) {
      const int nb = a.g.nkept[b];
      const int32_t *kept = a.g.kept + (int64_t)b * n;
      for (int q = tid; 4 * q < nb; q += blockDim.x) {
        uint32_t c[4] = {(uint32_t)q, (uint32_t)t, (uint32_t)b, RF_PHILOX_TAG};
        philox4x32_10(c, a.seed);
#pragma unroll
        for (int j = 0; j < 4; ++j)
          if (4 * q + j < nb) atomicAdd(&s.w[kept[__umulhi(c[j], (uint32_t)nb)]], 1);
      }
      __syncthreads();
    }
    // root totals, in row order
    if (tid == 0) {
      double W = 0.0, S = 0.0, Q = 0.0;
      int cnt = 0;
      for (int i = 0; i < n; ++i) {
        const int w = s.w[i];
        if (w > 0) {
          const double yi = (double)a.y[(int64_t)i * a.B + b], wy = (double)w * yi;
          W += (double)w;
          S += wy;
          Q = __dadd_rn(Q, __dmul_rn(wy, yi));
          ++cnt;
        }
      }
      s.nW[0] = W;
      s.nS[0] = S;
      s.nQ[0] = Q;
      s.ncnt[0] = cnt;
      s_next = 1;
    }
    __syncthreads();
    int lo = 0, hi = 1;
    while (lo < hi) {
      // A: leaf test of the level's nodes; open nodes get an index o and a segment of the filter buffers
      if (tid == 0) {
        int no = 0, acc = 0;
        for (int k = lo; k < hi; ++k) {
          const double W = s.nW[k], S = s.nS[k], mean = S / W, imp = __dsub_rn(s.nQ[k] / W, __dmul_rn(mean, mean));
          s.oidx[k] = -1;
          if (s.ncnt[k] < 2 || imp <= DBL_EPSILON) {
            rf_write_leaf(F, nb0, k, mean);
          } else {
            s.oidx[k] = no;
            s.openk[no] = k;
            s.segoff[no] = acc;
            acc += s.ncnt[k];
            ++no;
          }
        }
        s_nopen = no;
      }
      __syncthreads();
      const int nopen = s_nopen;
      if (nopen == 0) break;
      // B: per warp, features warp, warp + RF_WARPS, ...: stable filter into node segments, then lane-sequential scans
      int32_t *cur = s.cursor + (int64_t)warp * n;
      const int64_t wb = (int64_t)warp * n;
      for (int o = lane; o < nopen; o += 32) {
        s.bprox[wb + o] = -INFINITY;
        s.bfeat[wb + o] = INT_MAX;
      }
      for (int f = warp; f < a.width; f += RF_WARPS) {
        for (int o = lane; o < nopen; o += 32) cur[o] = 0;
        __syncwarp();
        const int len = f < dc ? n : 2 * n;
        for (int base = 0; base < len; base += 32) {
          const int p = base + lane;
          int o = -1, i = 0;
          float v = 0.0f;
          if (p < len) {
            if (f < dc) {
              i = a.g.ord[(int64_t)f * n + p];
              v = a.g.sval[(int64_t)f * n + p];
            } else {
              const int pass = p >= n;
              i = p - pass * n;
              v = rf_x(a.Xc, a.Xe, dc, ne, F.oh, i, f);
              if (v != (float)pass) i = -1;
            }
            if (i >= 0 && s.w[i] > 0) {
              const int k = s.nid[i];
              if (k >= lo && k < hi) o = s.oidx[k];
            }
          }
          const unsigned peers = __match_any_sync(0xffffffffu, o);
          const int c = o >= 0 ? cur[o] : 0;
          __syncwarp();
          if (o >= 0) {
            const int pos = s.segoff[o] + c + __popc(peers & lt);
            const int w = s.w[i];
            const float yi = a.y[(int64_t)i * a.B + b];
            s.fv[wb + pos] = v;
            s.fw[wb + pos] = w;
            s.fy[wb + pos] = yi;
            s.fwy[wb + pos] = (double)w * (double)yi;
            if (lane == __ffs(peers) - 1) cur[o] = c + __popc(peers);
          }
          __syncwarp();
        }
        for (int o = lane; o < nopen; o += 32) {
          const int k = s.openk[o], s0 = s.segoff[o], L = s.ncnt[k];
          const double W = s.nW[k], S = s.nS[k];
          double best = s.bprox[wb + o], WL = 0.0, SL = 0.0, QL = 0.0;
          bool improved = false;
          double bthr = 0.0, bWL = 0.0, bSL = 0.0, bQL = 0.0;
          int bcnt = 0;
          float vprev = 0.0f;
          for (int j = 0; j < L; ++j) {
            const int64_t q = wb + s0 + j;
            const float v = s.fv[q];
            if (j > 0 && (double)v > (double)vprev + RF_FEATURE_THRESHOLD) {
              const double SR = S - SL, proxy = __dadd_rn(__dmul_rn(SL, SL) / WL, __dmul_rn(SR, SR) / (W - WL));
              if (proxy > best) {
                best = proxy;
                improved = true;
                double th = (double)vprev / 2.0 + (double)v / 2.0;
                if (th == (double)v || isinf(th)) th = (double)vprev;
                bthr = th;
                bWL = WL;
                bSL = SL;
                bQL = QL;
                bcnt = j;
              }
            }
            const double wy = s.fwy[q];
            WL += (double)s.fw[q];
            SL += wy;
            QL = __dadd_rn(QL, __dmul_rn(wy, (double)s.fy[q]));
            vprev = v;
          }
          if (improved) {
            s.bprox[wb + o] = best;
            s.bfeat[wb + o] = f;
            s.bthr[wb + o] = bthr;
            s.bWL[wb + o] = bWL;
            s.bSL[wb + o] = bSL;
            s.bQL[wb + o] = bQL;
            s.bcnt[wb + o] = bcnt;
          }
        }
        __syncwarp();
      }
      __syncthreads();
      // C: per open node, the best split over warps (highest proxy, then lowest feature), into warp 0's slots
      for (int o = tid; o < nopen; o += blockDim.x) {
        int bw = 0;
        for (int w = 1; w < RF_WARPS; ++w) {
          const int64_t q = (int64_t)w * n + o, r = (int64_t)bw * n + o;
          if (s.bprox[q] > s.bprox[r] || (s.bprox[q] == s.bprox[r] && s.bfeat[q] < s.bfeat[r])) bw = w;
        }
        if (bw) {
          const int64_t q = (int64_t)bw * n + o;
          s.bprox[o] = s.bprox[q];
          s.bfeat[o] = s.bfeat[q];
          s.bthr[o] = s.bthr[q];
          s.bWL[o] = s.bWL[q];
          s.bSL[o] = s.bSL[q];
          s.bQL[o] = s.bQL[q];
          s.bcnt[o] = s.bcnt[q];
        }
      }
      __syncthreads();
      // D: children in breadth-first order: the split nodes of the level in index order, left then right
      if (tid == 0) {
        int nx = hi;
        for (int o = 0; o < nopen; ++o) {
          const int k = s.openk[o];
          const double W = s.nW[k], S = s.nS[k], Q = s.nQ[k];
          if (s.bprox[o] == -INFINITY) {
            s.oidx[k] = -1;
            rf_write_leaf(F, nb0, k, S / W);
            continue;
          }
          const int l = nx, r = nx + 1;
          nx += 2;
          const double th = s.bthr[o];
          F.nodes[nb0 + k] = make_int4(s.bfeat[o], __float_as_int(__double2float_rd(th)), l, r);
          F.thr64[nb0 + k] = th;
          F.val64[nb0 + k] = S / W;
          const double WL = s.bWL[o], SL = s.bSL[o], QL = s.bQL[o];
          s.nW[l] = WL;
          s.nS[l] = SL;
          s.nQ[l] = QL;
          s.ncnt[l] = s.bcnt[o];
          s.nW[r] = W - WL;
          s.nS[r] = S - SL;
          s.nQ[r] = Q - QL;
          s.ncnt[r] = s.ncnt[k] - s.bcnt[o];
        }
        s_next = nx;
      }
      __syncthreads();
      // E: every in-bag row of a split node moves to its child
      for (int i = tid; i < n; i += blockDim.x) {
        if (s.w[i] <= 0) continue;
        const int k = s.nid[i];
        if (k < lo || k >= hi || s.oidx[k] < 0) continue;
        const int4 nd = F.nodes[nb0 + k];
        const float x = rf_x(a.Xc, a.Xe, dc, ne, F.oh, i, nd.x);
        s.nid[i] = x <= __int_as_float(nd.y) ? nd.z : nd.w;
      }
      __syncthreads();
      lo = hi;
      hi = s_next;
    }
    if (tid == 0) F.ncount[tt] = s_next;
    __syncthreads();
  }
}

// est_noise (rf.py:42-43): sq[b, j] = (forest mean at kept row j - y)^2 in fp64, the mean summed sequentially in tree order
__global__ void rf_train_sq_kernel(const float *__restrict__ Xc, const int32_t *__restrict__ Xe, const float *__restrict__ y,
                                   int n, int dc, int ne, int B, int T, const int32_t *kept, const int32_t *nkept,
                                   unsigned char *forest, double *sq) {
  const int b = blockIdx.y, j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= nkept[b]) return;
  const RfForest F = rf_forest_view(forest);
  const int i = kept[(int64_t)b * n + j];
  double sum = 0.0;
  for (int t = 0; t < T; ++t) sum += rf_tree_value(F.nodes + ((int64_t)b * T + t) * F.cap, Xc, Xe, dc, ne, F.oh, i);
  const double d = sum / T - (double)y[(int64_t)i * B + b];
  sq[(int64_t)b * n + j] = __dmul_rn(d, d);
}

// noise[b] = fp32(np.mean(sq[b, :n_b])): numpy's pairwise sum, then the division
__global__ void rf_noise_kernel(const double *sq, int n, const int32_t *nkept, float *noise) {
  const int b = threadIdx.x;
  const double *a = sq + (int64_t)b * n;
  auto f = [a](int i) { return a[i]; };
  const int nb = nkept[b];
  noise[b] = (float)(rf_pairwise<RF_PW_DEPTH>(f, 0, nb) / (double)nb);
}

// ------------------------------------------------------------------------------------------------ predict
struct RfPredArgs {
  const float *Xc;
  const int32_t *Xe;
  int64_t m;
  int dc, ne, B, T, nsamp;
  const float *noise;
  float *mean, *var, *samp;
  uint64_t seed, counter;
  unsigned char *forest;
};

__global__ void __launch_bounds__(RF_PRED_THREADS) rf_predict_kernel(const __grid_constant__ RfPredArgs a) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= a.m * a.B) return;
  const int64_t r = idx / a.B;
  const int b = (int)(idx % a.B);
  const RfForest F = rf_forest_view(a.forest);
  bool ok = F.B == a.B && F.T == a.T && F.ne == a.ne;
  for (int c = 0; ok && c < a.ne; ++c) {
    const int u = a.Xe[r * a.ne + c];
    ok = u >= 0 && u < F.uniq[c];
  }
  float py = __int_as_float(0x7fffffff), ps2 = py;
  if (ok) {
    const int4 *trees = F.nodes + (int64_t)b * a.T * F.cap;
    const int cap = F.cap, dc = a.dc, ne = a.ne;
    const float *Xc = a.Xc;
    const int32_t *Xe = a.Xe, *oh = F.oh;
    double seq = 0.0;
    auto leaf = [&](int t) {
      const double v = rf_tree_value(trees + (int64_t)t * cap, Xc, Xe, dc, ne, oh, r);
      seq += v;
      return v;
    };
    const double mnp = rf_pairwise<RF_PW_DEPTH>(leaf, 0, a.T) / a.T;
    auto dev2 = [&](int t) {
      const double d = rf_tree_value(trees + (int64_t)t * cap, Xc, Xe, dc, ne, oh, r) - mnp;
      return __dmul_rn(d, d);
    };
    const double v64 = rf_pairwise<RF_PW_DEPTH>(dev2, 0, a.T) / a.T;
    py = (float)(seq / a.T);
    ps2 = __fadd_rn((float)v64, a.noise[b]);
  }
  a.mean[idx] = py;
  a.var[idx] = ps2;
  const float ps = __fsqrt_rn(ps2);
  for (int t = 0; t < a.nsamp; ++t) {
    const int64_t q = ((int64_t)t * a.m + r) * a.B + b;
    float z0, z1;
    philox_normal2(a.seed, (uint64_t)(q >> 1), a.counter, z0, z1);
    a.samp[q] = __fadd_rn(py, __fmul_rn(ps, (q & 1) ? z1 : z0));
  }
}

// ------------------------------------------------------------------------------------------------ load
struct RfLoadArgs {
  const int32_t *left, *right, *feature, *ncount;
  const double *thr, *val;
  int T, cap;
  unsigned char *forest;
};

__global__ void rf_load_kernel(const __grid_constant__ RfLoadArgs a) {
  const int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= (int64_t)a.T * a.cap) return;
  const RfForest F = rf_forest_view(a.forest);
  const int t = (int)(q / a.cap), k = (int)(q % a.cap);
  if (k == 0) F.ncount[t] = a.ncount[t];
  if (k >= a.ncount[t]) return;
  const double v = a.val[q];
  if (a.left[q] < 0 || a.feature[q] < 0) {
    rf_write_leaf(F, 0, (int)q, v);
    return;
  }
  const double th = a.thr[q];
  F.nodes[q] = make_int4(a.feature[q], __float_as_int(__double2float_rd(th)), a.left[q], a.right[q]);
  F.thr64[q] = th;
  F.val64[q] = v;
}

// ------------------------------------------------------------------------------------------------ launchers
static int rf_write_header(unsigned char *forest, int cap, int B, int T, int ne, int woh, const std::vector<int32_t> &tab,
                           cudaStream_t st) {
  RfForest f;
  rf_forest_carve(forest, cap, B, T, ne, woh, &f);
  const int32_t h[8] = {cap, B, T, woh, ne, 0, 0, 0};
  HB_CUDA(cudaMemcpyAsync(forest, h, sizeof(h), cudaMemcpyHostToDevice, st));
  if (!tab.empty())
    HB_CUDA(cudaMemcpyAsync(f.uniq, tab.data(), tab.size() * sizeof(int32_t), cudaMemcpyHostToDevice, st));
  HB_CUDA(cudaStreamSynchronize(st));   // the header and tables come from host locals
  return HB_OK;
}

int64_t rf_forest_bytes(const hb_rf_spec_t *spec, int64_t max_nodes, int64_t B, int64_t T) {
  int dc, ne, woh;
  if (!rf_layout(spec, dc, ne, woh, nullptr) || max_nodes < 1 || max_nodes > 2 * (int64_t)HB_RF_MAX_ROWS - 1 || B < 1 ||
      B > HB_MAX_OUTPUTS || T < 1 || T > HB_RF_MAX_TREES)
    return -1;
  return rf_forest_carve(nullptr, (int)max_nodes, (int)B, (int)T, ne, woh, nullptr);
}

int64_t rf_fit_ws_query(int64_t n, const hb_rf_spec_t *spec, int64_t B, int64_t T) {
  int dc, ne, woh;
  if (!rf_layout(spec, dc, ne, woh, nullptr) || n < 1 || n > HB_RF_MAX_ROWS || B < 1 || B > HB_MAX_OUTPUTS || T < 1 ||
      T > HB_RF_MAX_TREES)
    return -1;
  return rf_ws_carve(nullptr, (int)n, dc, (int)B, (int)T, nullptr);
}

int launch_rf_fit(const float *Xc, const int32_t *Xe, const float *y, int64_t n, const hb_rf_spec_t *spec, int64_t B,
                  int64_t T, const int32_t *counts, uint64_t seed, void *forest, float *noise, void *ws, int64_t ws_bytes,
                  cudaStream_t st) {
  int dc, ne, woh;
  std::vector<int32_t> tab;
  const int64_t need = rf_fit_ws_query(n, spec, B, T);
  if (need < 0 || !rf_layout(spec, dc, ne, woh, &tab)) return HB_ERR_INVALID;
  if (!y || !forest || !noise || !ws || ws_bytes < need || (dc > 0 && !Xc) || (ne > 0 && !Xe)) return HB_ERR_INVALID;
  const int cap = (int)(2 * n - 1);
  int s = rf_write_header((unsigned char *)forest, cap, (int)B, (int)T, ne, woh, tab, st);
  if (s != HB_OK) return s;
  RfFitArgs a{};
  rf_ws_carve((unsigned char *)ws, (int)n, dc, (int)B, (int)T, &a.g);
  a.Xc = Xc;
  a.Xe = Xe;
  a.y = y;
  a.counts = counts;
  a.n = (int)n;
  a.dc = dc;
  a.ne = ne;
  a.width = dc + woh;
  a.B = (int)B;
  a.T = (int)T;
  a.seed = seed;
  a.forest = (unsigned char *)forest;
  rf_prep_kernel<<<(unsigned)B, 32, 0, st>>>(y, (int)n, (int)B, a.g.kept, a.g.nkept);
  HB_LAUNCH_CHECK("rf_prep_kernel");
  if (dc > 0) {
    int N = 1;
    while (N < n) N <<= 1;
    const size_t smem = (size_t)N * sizeof(unsigned long long);
    HB_CUDA(cudaFuncSetAttribute(rf_sort_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    rf_sort_kernel<<<(unsigned)dc, RF_SORT_THREADS, smem, st>>>(Xc, (int)n, dc, a.g.ord, a.g.sval);
    HB_LAUNCH_CHECK("rf_sort_kernel");
  }
  rf_grow_kernel<<<(unsigned)a.g.nslots, RF_THREADS, 0, st>>>(a);
  HB_LAUNCH_CHECK("rf_grow_kernel");
  rf_train_sq_kernel<<<dim3((unsigned)ceil_div(n, 128), (unsigned)B), 128, 0, st>>>(
      Xc, Xe, y, (int)n, dc, ne, (int)B, (int)T, a.g.kept, a.g.nkept, (unsigned char *)forest, a.g.sq);
  HB_LAUNCH_CHECK("rf_train_sq_kernel");
  rf_noise_kernel<<<1, (unsigned)B, 0, st>>>(a.g.sq, (int)n, a.g.nkept, noise);
  HB_LAUNCH_CHECK("rf_noise_kernel");
  count_launches(dc > 0 ? 5 : 4);
  return HB_OK;
}

int launch_rf_predict(const float *Xc, const int32_t *Xe, int64_t m, const hb_rf_spec_t *spec, const void *forest,
                      int64_t B, int64_t T, const float *noise, float *mean, float *var, int64_t n_samples, uint64_t seed,
                      uint64_t counter, float *samples, cudaStream_t st) {
  int dc, ne, woh;
  if (!rf_layout(spec, dc, ne, woh, nullptr) || B < 1 || B > HB_MAX_OUTPUTS || T < 1 || T > HB_RF_MAX_TREES || m < 0 ||
      m > (int64_t(1) << 31) || n_samples < 0 || n_samples > (int64_t(1) << 31))
    return HB_ERR_INVALID;
  if (!forest || !noise || !mean || !var || (dc > 0 && !Xc) || (ne > 0 && !Xe) || (n_samples > 0 && !samples))
    return HB_ERR_INVALID;
  if (m == 0) return HB_OK;
  RfPredArgs a{};
  a.Xc = Xc;
  a.Xe = Xe;
  a.m = m;
  a.dc = dc;
  a.ne = ne;
  a.B = (int)B;
  a.T = (int)T;
  a.nsamp = (int)n_samples;
  a.noise = noise;
  a.mean = mean;
  a.var = var;
  a.samp = samples;
  a.seed = seed;
  a.counter = counter;
  a.forest = (unsigned char *)forest;
  rf_predict_kernel<<<(unsigned)ceil_div(m * B, RF_PRED_THREADS), RF_PRED_THREADS, 0, st>>>(a);
  count_launches(1);
  HB_LAUNCH_CHECK("rf_predict_kernel");
  return HB_OK;
}

int launch_rf_load(const int32_t *left, const int32_t *right, const int32_t *feature, const double *thr,
                   const double *value, const int32_t *node_counts, const hb_rf_spec_t *spec, int64_t T, int64_t max_nodes,
                   void *forest, cudaStream_t st) {
  int dc, ne, woh;
  std::vector<int32_t> tab;
  if (rf_forest_bytes(spec, max_nodes, 1, T) < 0 || !rf_layout(spec, dc, ne, woh, &tab)) return HB_ERR_INVALID;
  if (!left || !right || !feature || !thr || !value || !node_counts || !forest) return HB_ERR_INVALID;
  int s = rf_write_header((unsigned char *)forest, (int)max_nodes, 1, (int)T, ne, woh, tab, st);
  if (s != HB_OK) return s;
  RfLoadArgs a{left, right, feature, node_counts, thr, value, (int)T, (int)max_nodes, (unsigned char *)forest};
  rf_load_kernel<<<(unsigned)ceil_div(T * max_nodes, 256), 256, 0, st>>>(a);
  count_launches(1);
  HB_LAUNCH_CHECK("rf_load_kernel");
  return HB_OK;
}

}  // namespace hb
