// Monte-Carlo expected hypervolume improvement of GeneralBO's selection (HEBO/hebo/optimizers/general.py:107-158), bit for
// bit with the host hypervolume (hebo_b200/general.py: hypervolume / _hv / _nondominated):
//
//     base_hv = hypervolume(front, ref)
//     ehvi[j] = (sum_k (hypervolume(vstack([front, samples[k, j]]), ref) - base_hv)) / n_mc      (sum from 0.0, k ascending)
//
// One round has m n_mc + 1 hypervolumes (the last one is base_hv); each is one work item of one thread, so every sum keeps
// the host's sequential order.  The host recursion, for the rows strictly below ref in every coordinate:
//
//     hv(Y, ref[:D]):  D == 1: ref[0] - min(Y[:, 0])
//                      else:   Y stably sorted by column D-1;  vol = 0
//                              for i: hi = Y[i+1, D-1] (or ref[D-1] after the last row)
//                                     if hi > Y[i, D-1]: vol += hv(nondominated(Y[:i+1, :D-1]), ref[:D-1]) * (hi - Y[i, D-1])
//
// is restated level by level without changing a value or the order of an operation:
//  - ehvi_front_kernel drops the front rows not below ref (NaN rows fall out there) and sorts the rest stably by the last
//    column once per round; every item reads that sorted front (from shared memory when it fits).  A sample below ref is
//    the last row of its stack, so it goes after every front row whose last coordinate is <= its own.
//  - nondominated(prefix) of level D is kept incrementally as rows arrive in the level's order: a row dominated by a member
//    is not added, otherwise it drops the members it dominates.  Dominance is transitive, so the set equals the host's
//    nondominated(prefix) after every row; duplicates dominate nothing and both stay.  The set is kept ordered by the next
//    level's sort key (column D-2), ties in arrival order, which is exactly the host's stable argsort of nondominated(prefix)
//    in the parent's order, so the next level needs no sort.
//  - At D == 2, min over the nondominated prefix is min over the prefix: the leaf keeps a running minimum.
//  - Every fp64 operation is __dadd_rn / __dsub_rn / __dmul_rn / __ddiv_rn: no FMA contraction, and +-inf follow the host's
//    IEEE path (a -inf coordinate below ref gives inf, +inf is never below ref).
// Each thread carves its K - 2 level sets of n + 1 row ids from the workspace, interleaved across the resident threads so a
// warp's accesses at the same position coalesce; the number of resident threads is capped, so any n works.
// Cost is exponential in K, as on the host: the level-D loop runs the level-(D-1) loop once per slice.
#include <algorithm>

#include "kernels.h"

namespace hb {

constexpr int EHVI_THREADS = 32;                // one warp per CTA spreads a round's few thousand items over many SMs
constexpr int64_t EHVI_MAX_SLOTS = 65536;       // resident items (threads) of the grid-stride loop
constexpr int64_t EHVI_STAGE_BYTES = 16 * 1024; // the sorted front is staged in shared memory up to this size

struct EhviLayout {
  int64_t items, slots, hv, F, nf, lists, total;
};

static int64_t ehvi_layout(int64_t n, int64_t K, int64_t m, int64_t n_mc, EhviLayout *L) {
  if (K < 2 || K > HB_MAX_OBJ || n < 0 || m < 0 || n_mc < 1) return -1;
  if (n > INT32_MAX - 2 || n_mc > ((int64_t)1 << 40) || m > ((int64_t)1 << 40) / n_mc) return -1;   // int32 row ids
  L->items = m * n_mc + 1;
  L->slots = round_up(std::min(L->items, EHVI_MAX_SLOTS), EHVI_THREADS);
  int64_t off = 0;
  L->hv = off;    off += round_up(L->items * (int64_t)sizeof(double), 256);
  L->F = off;     off += round_up(n * K * (int64_t)sizeof(double), 256);
  L->nf = off;    off += 256;
  L->lists = off; off += round_up((K - 2) * (n + 1) * L->slots * (int64_t)sizeof(int32_t), 256);
  L->total = off;
  return off;
}

int64_t ehvi_ws_query(int64_t n, int64_t K, int64_t m, int64_t n_mc) {
  EhviLayout L;
  return ehvi_layout(n, K, m, n_mc, &L);
}

// the filtered front, stably sorted by its last column: row r below ref goes to its rank among those rows
__global__ void ehvi_front_kernel(const double *__restrict__ front, int64_t n, int K, const double *__restrict__ ref,
                                  double *__restrict__ F, int32_t *__restrict__ nf) {
  const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n) return;
  auto below = [&](int64_t q) {
    for (int c = 0; c < K; ++c)
      if (!(front[q * K + c] < ref[c])) return false;
    return true;
  };
  if (!below(r)) return;
  const double key = front[r * K + K - 1];
  int64_t rank = 0;
  for (int64_t q = 0; q < n; ++q) {
    if (!below(q)) continue;
    const double kq = front[q * K + K - 1];
    rank += kq < key || (kq == key && q < r);
  }
  for (int c = 0; c < K; ++c) F[rank * K + c] = front[r * K + c];
  atomicAdd(nf, 1);
}

// the rows of one hypervolume: the sorted front (row ids 0..nf-1) and the sample (row id nf)
template <int K>
struct HvItem {
  const double *F;
  int nf;
  double s[K], ref[K];
  __device__ __forceinline__ double v(int row, int c) const { return row == nf ? s[c] : F[(int64_t)row * K + c]; }
};

// level K's rows: the sorted front with the sample inserted at position p (p = nf when the sample is not below ref)
struct TopRows {
  int p, nf;
  __device__ __forceinline__ int operator()(int i) const { return i < p ? i : (i == p ? nf : i - 1); }
};
// a lower level's rows: the parent's nondominated set, element i at S[i * stride]
struct ListRows {
  const int32_t *S;
  int64_t stride;
  __device__ __forceinline__ int operator()(int i) const { return S[i * stride]; }
};

// does row q dominate the point a in the first C coordinates (<= in all, < in one)
template <int C, int K>
__device__ __forceinline__ bool dominates(const HvItem<K> &it, int q, const double (&a)[K]) {
  bool le = true, lt = false;
#pragma unroll
  for (int c = 0; c < C; ++c) {
    const double x = it.v(q, c);
    le = le && x <= a[c];
    lt = lt || x < a[c];
  }
  return le && lt;
}
template <int C, int K>
__device__ __forceinline__ bool dominated_by(const HvItem<K> &it, int q, const double (&a)[K]) {
  bool le = true, lt = false;
#pragma unroll
  for (int c = 0; c < C; ++c) {
    const double x = it.v(q, c);
    le = le && a[c] <= x;
    lt = lt || a[c] < x;
  }
  return le && lt;
}

// hv of the n rows `rows` (sorted by column D-1) in the first D coordinates; S: this level's nondominated set (n ids)
template <int D, int K, class Rows>
__device__ double hv_level(const HvItem<K> &it, const Rows &rows, int n, int32_t *S, int64_t stride, int64_t cap) {
  double vol = 0.0;
  if (n == 0) return vol;
  if constexpr (D == 2) {
    int r = rows(0);
    double mn = it.v(r, 0), y = it.v(r, 1);
    for (int i = 0; i < n; ++i) {
      const double x0 = it.v(r, 0);
      mn = x0 < mn ? x0 : mn;
      int rn = r;
      double hi = it.ref[1];
      if (i + 1 < n) {
        rn = rows(i + 1);
        hi = it.v(rn, 1);
      }
      if (hi > y) vol = __dadd_rn(vol, __dmul_rn(__dsub_rn(it.ref[0], mn), __dsub_rn(hi, y)));
      r = rn;
      y = hi;
    }
  } else {
    int s = 0;
    int r = rows(0);
    for (int i = 0; i < n; ++i) {
      double a[K];
#pragma unroll
      for (int c = 0; c < D; ++c) a[c] = it.v(r, c);
      bool dominated = false;
      for (int t = 0; t < s && !dominated; ++t) dominated = dominates<D - 1>(it, S[t * stride], a);
      if (!dominated) {
        int w = 0;
        for (int t = 0; t < s; ++t) {
          const int q = S[t * stride];
          if (!dominated_by<D - 1>(it, q, a)) S[w++ * stride] = q;
        }
        int pos = w;   // after every member whose column D-2 is <= the new row's
        while (pos > 0) {
          const int q = S[(pos - 1) * stride];
          if (!(it.v(q, D - 2) > a[D - 2])) break;
          S[pos * stride] = q;
          --pos;
        }
        S[pos * stride] = r;
        s = w + 1;
      }
      int rn = r;
      double hi = it.ref[D - 1];
      if (i + 1 < n) {
        rn = rows(i + 1);
        hi = it.v(rn, D - 1);
      }
      const double y = a[D - 1];
      if (hi > y) {
        const double sub = hv_level<D - 1>(it, ListRows{S, stride}, s, S + cap * stride, stride, cap);
        vol = __dadd_rn(vol, __dmul_rn(sub, __dsub_rn(hi, y)));
      }
      r = rn;
    }
  }
  return vol;
}

// hv[t] for the items t = k m + j (samples[k, j] stacked under the front) and t = m n_mc (the front alone)
template <int K>
__global__ void __launch_bounds__(EHVI_THREADS) ehvi_hv_kernel(const double *__restrict__ Fg, const int32_t *__restrict__ nf_p,
                                                               const double *__restrict__ samples, int64_t items,
                                                               const double *__restrict__ ref, int stage,
                                                               int32_t *__restrict__ lists, int64_t slots, int64_t cap,
                                                               double *__restrict__ hv) {
  extern __shared__ double Fs[];
  HvItem<K> it;
  it.nf = *nf_p;
  it.F = Fg;
  if (stage) {
    for (int64_t e = threadIdx.x; e < (int64_t)it.nf * K; e += blockDim.x) Fs[e] = Fg[e];
    __syncthreads();
    it.F = Fs;
  }
#pragma unroll
  for (int c = 0; c < K; ++c) it.ref[c] = ref[c];
  const int64_t slot = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  for (int64_t t = slot; t < items; t += slots) {
    bool keep = t != items - 1;
    if (keep) {
#pragma unroll
      for (int c = 0; c < K; ++c) {
        it.s[c] = samples[t * K + c];
        keep = keep && it.s[c] < it.ref[c];
      }
    }
    int p = it.nf, N = it.nf;
    if (keep) {   // upper bound of the sample's last coordinate in the sorted front
      int lo = 0, hi = it.nf;
      while (lo < hi) {
        const int mid = (lo + hi) / 2;
        if (it.F[(int64_t)mid * K + K - 1] <= it.s[K - 1]) lo = mid + 1;
        else hi = mid;
      }
      p = lo;
      N = it.nf + 1;
    }
    hv[t] = hv_level<K>(it, TopRows{p, it.nf}, N, lists + slot, slots, cap);
  }
}

__global__ void ehvi_mean_kernel(const double *__restrict__ hv, int64_t m, int64_t n_mc, double *__restrict__ base_hv,
                                 double *__restrict__ ehvi) {
  const int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const double base = hv[m * n_mc];
  if (j == 0) *base_hv = base;
  if (j >= m) return;
  double acc = 0.0;
  for (int64_t k = 0; k < n_mc; ++k) acc = __dadd_rn(acc, __dsub_rn(hv[k * m + j], base));
  ehvi[j] = __ddiv_rn(acc, (double)n_mc);
}

int launch_ehvi(const double *front, int64_t n, int64_t K, const double *samples, int64_t m, int64_t n_mc, const double *ref,
                double *base_hv, double *ehvi, void *ws, int64_t ws_bytes, cudaStream_t st) {
  EhviLayout L;
  const int64_t need = ehvi_layout(n, K, m, n_mc, &L);
  if (need < 0 || ws_bytes < need) return HB_ERR_INVALID;
  if (m == 0) return HB_OK;
  char *w = static_cast<char *>(ws);
  double *hv = reinterpret_cast<double *>(w + L.hv), *F = reinterpret_cast<double *>(w + L.F);
  int32_t *nf = reinterpret_cast<int32_t *>(w + L.nf), *lists = reinterpret_cast<int32_t *>(w + L.lists);
  HB_CUDA(cudaMemsetAsync(nf, 0, sizeof(int32_t), st));
  int launches = 2;
  if (n > 0) {
    ehvi_front_kernel<<<(unsigned)ceil_div(n, 128), 128, 0, st>>>(front, n, (int)K, ref, F, nf);
    ++launches;
  }
  const int64_t fbytes = n * K * (int64_t)sizeof(double);
  const int stage = fbytes <= EHVI_STAGE_BYTES;
  const size_t smem = stage ? (size_t)fbytes : 0;
  const unsigned grid = (unsigned)(L.slots / EHVI_THREADS);
  auto run = [&](auto kk) {
    ehvi_hv_kernel<decltype(kk)::value><<<grid, EHVI_THREADS, smem, st>>>(F, nf, samples, L.items, ref, stage, lists, L.slots,
                                                                          n + 1, hv);
  };
  switch (K) {
    case 2: run(std::integral_constant<int, 2>{}); break;
    case 3: run(std::integral_constant<int, 3>{}); break;
    case 4: run(std::integral_constant<int, 4>{}); break;
    case 5: run(std::integral_constant<int, 5>{}); break;
    case 6: run(std::integral_constant<int, 6>{}); break;
    case 7: run(std::integral_constant<int, 7>{}); break;
    default: run(std::integral_constant<int, 8>{}); break;
  }
  ehvi_mean_kernel<<<(unsigned)ceil_div(m, 128), 128, 0, st>>>(hv, m, n_mc, base_hv, ehvi);
  count_launches(launches);
  HB_LAUNCH_CHECK("ehvi");
  return HB_OK;
}

}  // namespace hb
