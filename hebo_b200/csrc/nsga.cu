// Device-resident NSGA-II for the acquisition optimiser (SURVEY 8f-1): the role pymoo's NSGA2 + MixedVariableMating play in
// HEBO/hebo/acq_optimizers/evolution_optimizer.py:107-160 (pop 100, `iters` generations, Real -> SBX + polynomial
// mutation, Integer -> the same + rounding repair, Choice -> uniform crossover + random-resample mutation, duplicate
// elimination, rank-and-crowding survival; variable typing as evolution_optimizer.py:26-41).  pymoo is a third-party
// dependency that is not installed here: the operators follow the published algorithms (Deb et al. 2002; Deb & Agrawal
// SBX eta = 15, pair probability 0.9, per-variable 0.5; Deb & Goyal PM eta = 20, per-variable min(0.5, 1/D)) -- pymoo's
// random stream is not reproduced.  The population never leaves the device: one generation = mate (1 launch) -> fused
// posterior + MACE on the offspring (the C-ABI call the Sobol path uses) -> survive (1 launch), no host synchronisation.
//
// Layout: X [P, D] fp32 in the optimisation space (numeric columns first, then the categorical indices as floats);
// kind[D]: 0 real, 1 integer, 2 choice; lb / ub [D]; fixed[D] (NaN = free, else the value of a `fix_input` column).
#include <cooperative_groups.h>

#include <algorithm>

#include "kernels.h"

namespace hb {

__device__ __forceinline__ void philox4(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3, uint64_t seed, float (&u)[4]) {
  uint32_t c[4] = {c0, c1, c2, c3};
  uint32_t k0 = (uint32_t)seed, k1 = (uint32_t)(seed >> 32);
  const uint32_t M0 = 0xD2511F53u, M1 = 0xCD9E8D57u;
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const uint32_t hi0 = __umulhi(M0, c[0]), lo0 = M0 * c[0];
    const uint32_t hi1 = __umulhi(M1, c[2]), lo1 = M1 * c[2];
    const uint32_t n0 = hi1 ^ c[1] ^ k0, n1 = lo1, n2 = hi0 ^ c[3] ^ k1, n3 = lo0;
    c[0] = n0; c[1] = n1; c[2] = n2; c[3] = n3;
    k0 += 0x9E3779B9u;
    k1 += 0xBB67AE85u;
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) u[i] = ((float)c[i] + 0.5f) * 2.3283064365386963e-10f;   // (0, 1)
}

__device__ __forceinline__ float repair(float v, int kind, float lo, float hi, float fixed) {
  if (!isnan(fixed)) return fixed;
  if (kind != 0) v = rintf(v);
  return fminf(fmaxf(v, lo), hi);
}

// split a float row of the optimisation space into the model's inputs: Xc [d] fp32, Xe [e] int32
__device__ __forceinline__ void split_row(const float *row, int d, int e, float *xc, int32_t *xe) {
  for (int k = 0; k < d; ++k) xc[k] = row[k];
  for (int k = 0; k < e; ++k) xe[k] = (int32_t)rintf(row[d + k]);
}

// initial population: uniform in the box (evolution_optimizer.py:44-55 with the default sobol_init flag samples
// uniformly), typed repair, row 0.. = the initial suggestions (prepended, :56-57)
__global__ void nsga_init_kernel(float *__restrict__ X, int P, int D, int d, const int32_t *__restrict__ kind,
                                 const float *__restrict__ lb, const float *__restrict__ ub, const float *__restrict__ fixed,
                                 const float *__restrict__ init, int n_init, uint64_t seed, float *__restrict__ Xc,
                                 int32_t *__restrict__ Xe) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= P) return;
  float *row = X + (int64_t)p * D;
  for (int k = 0; k < D; k += 4) {
    float u[4];
    philox4((uint32_t)p, 0xFFFFFFFFu, (uint32_t)k, 1u, seed, u);
    for (int j = 0; j < 4 && k + j < D; ++j) {
      const int c = k + j;
      float v = (p < n_init) ? init[(int64_t)p * D + c] : lb[c] + (ub[c] - lb[c]) * u[j];
      if (kind[c] == 2 && p >= n_init) v = floorf(lb[c] + (ub[c] - lb[c] + 1.0f) * u[j]);   // categories equally likely
      row[c] = repair(v, kind[c], lb[c], ub[c], fixed[c]);
    }
  }
  split_row(row, d, D - d, Xc + (int64_t)p * d, Xe + (int64_t)p * (D - d));
}

// one thread per mating: two random parents -> two children (rows 2t, 2t + 1 of the offspring buffers)
__global__ void nsga_mate_kernel(const float *__restrict__ X, int P, int D, int d, const int32_t *__restrict__ kind,
                                 const float *__restrict__ lb, const float *__restrict__ ub, const float *__restrict__ fixed,
                                 uint64_t seed, int gen, float pm_prob, float *__restrict__ C, float *__restrict__ Cc,
                                 int32_t *__restrict__ Ce) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (2 * t >= P) return;
  const float sbx_eta = 15.0f, sbx_prob = 0.9f, sbx_var = 0.5f, pm_eta = 20.0f;
  float u[4];
  philox4((uint32_t)t, (uint32_t)gen, 0xFFFFFFF0u, 2u, seed, u);
  const int pa = min((int)(u[0] * P), P - 1), pb = min((int)(u[1] * P), P - 1);
  const bool do_pair = u[2] < sbx_prob;
  const float *A = X + (int64_t)pa * D, *B = X + (int64_t)pb * D;
  float *c1 = C + (int64_t)(2 * t) * D, *c2 = C + (int64_t)min(2 * t + 1, P - 1) * D;
  const bool second = 2 * t + 1 < P;
  for (int k = 0; k < D; ++k) {
    float v[4], w[4];
    philox4((uint32_t)t, (uint32_t)gen, (uint32_t)k, 3u, seed, v);
    philox4((uint32_t)t, (uint32_t)gen, (uint32_t)k, 4u, seed, w);
    const float lo = lb[k], hi = ub[k];
    float x1 = A[k], x2 = B[k];
    if (kind[k] == 2) {                                   // Choice: uniform crossover, random-resample mutation
      if (do_pair && v[0] < 0.5f) { const float s = x1; x1 = x2; x2 = s; }
      if (v[1] < pm_prob) x1 = floorf(lo + (hi - lo + 1.0f) * v[2]);
      if (w[1] < pm_prob) x2 = floorf(lo + (hi - lo + 1.0f) * w[2]);
    } else {
      // ---- SBX with bounds
      const float y1 = fminf(x1, x2), y2 = fmaxf(x1, x2), diff = y2 - y1;
      if (do_pair && v[0] < sbx_var && diff > 1e-14f) {
        const float uu = v[1], ex = 1.0f / (sbx_eta + 1.0f);
        auto betaq = [&](float beta) {
          const float alpha = 2.0f - powf(beta, -(sbx_eta + 1.0f));
          const float inner = (uu <= 1.0f / alpha) ? uu * alpha : 1.0f / fmaxf(2.0f - uu * alpha, 1e-30f);
          return powf(inner, ex);
        };
        float a = 0.5f * ((y1 + y2) - betaq(1.0f + 2.0f * (y1 - lo) / diff) * diff);
        float b = 0.5f * ((y1 + y2) + betaq(1.0f + 2.0f * (hi - y2) / diff) * diff);
        if (v[2] < 0.5f) { const float s = a; a = b; b = s; }
        x1 = a;
        x2 = b;
      }
      // ---- polynomial mutation
      const float span = hi - lo, mp = 1.0f / (pm_eta + 1.0f);
      auto pm = [&](float x, float um) {
        const float d1 = (x - lo) / span, d2 = (hi - x) / span;
        const float dq = um < 0.5f ? powf(2.0f * um + (1.0f - 2.0f * um) * powf(1.0f - d1, pm_eta + 1.0f), mp) - 1.0f
                                   : 1.0f - powf(2.0f * (1.0f - um) + 2.0f * (um - 0.5f) * powf(1.0f - d2, pm_eta + 1.0f), mp);
        return x + dq * span;
      };
      if (span > 0.0f) {
        x1 = fminf(fmaxf(x1, lo), hi);
        x2 = fminf(fmaxf(x2, lo), hi);
        if (v[3] < pm_prob) x1 = pm(x1, w[0]);
        if (w[3] < pm_prob) x2 = pm(x2, w[1]);
      }
    }
    c1[k] = repair(x1, kind[k], lo, hi, fixed[k]);
    if (second) c2[k] = repair(x2, kind[k], lo, hi, fixed[k]);
  }
  split_row(c1, d, D - d, Cc + (int64_t)(2 * t) * d, Ce + (int64_t)(2 * t) * (D - d));
  if (second) split_row(c2, d, D - d, Cc + (int64_t)(2 * t + 1) * d, Ce + (int64_t)(2 * t + 1) * (D - d));
}

// ---- rank-and-crowding survival of the merged population (pop rows 0..P-1, offspring rows P..2P-1).
// Both survival kernels below (one CTA for 2P <= 512, the cooperative multi-CTA one for 512 < 2P <= 32768) give the
// same result, bit for bit:
//  * sanitising: every objective component that is not finite becomes +inf, one component at a time;
//  * duplicates (pymoo MixedVariableDuplicateElimination): child i is a duplicate when |o[k] - me[k]| <= 1e-16f for every
//    k against ANY earlier merged row j < i (population rows first, then earlier children, duplicates included); its three
//    objectives become +inf;
//  * ranks: fast non-dominated sort (j dominates i: all <=, one <), fronts peeled until the cumulative count reaches P;
//    whole fronts below the cut front survive;
//  * cut front: fp32 crowding distance, objective k = 0, 1, 2 in that order: members ordered by f_k with ties by merged
//    index, the two end positions become +inf, an interior member adds (f[next] - f[prev]) / (fmax - fmin) when
//    fmax > fmin and fmax - fmin is finite; the `need` members with the largest crowding survive, ties by lower index;
//  * output: survivors in ascending merged-row order, F_next holds the sanitised (duplicate -> +inf) objectives.
// With a constraint column G (hb_nsga2_survive_cv; pymoo's survival with infeasible filtering as EvolutionOpt runs it
// with n_constr = 1, evolution_optimizer.py:82,105,135-140 -- recalled, not checked against pymoo):
//  * a merged row is feasible iff G <= 0; a non-finite G becomes +inf; a duplicate child gets G = +inf as well;
//  * nf >= P feasible rows: only the feasible rows enter the rank-and-crowding survival above, unchanged;
//  * nf < P: every feasible row survives, the other P - nf slots go to infeasible rows in ascending G, ties by the lower
//    merged index;
//  * output order as above; G_next holds the survivors' sanitised G.
// Without G (hb_nsga2_survive_ex) every row is feasible with G = 0, duplicates included, which is the rule above.  G = 0
// everywhere gives the same survivors unless the cut reaches the front of all-+inf rows that holds a duplicate child:
// with G the duplicate is infeasible and leaves that front.
// Both kernels are templates on the objective count K (2 <= K <= HB_MAX_OBJ, hb_nsga2_survive_k): everything above holds
// with K objectives in place of three, and crowding adds objective k = 0 .. K-1 in that order.  hb_nsga2_survive_ex / _cv
// are the K = 3 instances.
__device__ __forceinline__ float sanitize_obj(float v) { return isfinite(v) ? v : INFINITY; }

// a dominates b (minimisation): all <=, at least one <
template <int K>
__device__ __forceinline__ bool dominates(const float *a, const float *b) {
  bool le = true, lt = false;
#pragma unroll
  for (int k = 0; k < K; ++k) {
    le = le && a[k] <= b[k];
    lt = lt || a[k] < b[k];
  }
  return le && lt;
}

// (same_row, common.cuh: the duplicate predicate, shared with hb_sample_y_batch)

// (fj, j) before (fi, i) in ascending f order, ties by index; in descending crowding order, ties by index
__device__ __forceinline__ bool before_asc(float fj, int j, float fi, int i) { return fj < fi || (fj == fi && j < i); }
__device__ __forceinline__ bool before_desc(float cj, int j, float ci, int i) { return cj > ci || (cj == ci && j < i); }

// the crowding term of an interior member of the cut front along one objective
__device__ __forceinline__ float crowd_interior(float acc, float fprev, float fnext, float fmin, float fmax) {
  return (fmax > fmin && isfinite(fmax - fmin)) ? acc + (fnext - fprev) / (fmax - fmin) : acc;
}

__device__ __forceinline__ const float *merged_row(const float *X, const float *C, int P, int D, int j) {
  return j < P ? X + (int64_t)j * D : C + (int64_t)(j - P) * D;
}

// merged row i (a child, i >= P) equals an earlier merged row j < i: the duplicate test of the single-CTA kernels
__device__ __forceinline__ bool dup_of_earlier(const float *X, const float *C, int P, int D, int i) {
  const float *me = C + (int64_t)(i - P) * D;
  bool dup = false;
  for (int j = 0; j < i && !dup; ++j) dup = same_row(merged_row(X, C, P, D, j), me, D);
  return dup;
}

constexpr int NSGA_MAX = 512;
template <int K>
__global__ void __launch_bounds__(NSGA_MAX) nsga_survive_kernel(const float *__restrict__ X, const float *__restrict__ F,
                                                                const float *__restrict__ G, const float *__restrict__ C,
                                                                const float *__restrict__ FC, const float *__restrict__ GC,
                                                                int P, int D, int d, float *__restrict__ Xn,
                                                                float *__restrict__ Fn, float *__restrict__ Gn,
                                                                float *__restrict__ Xcn, int32_t *__restrict__ Xen) {
  __shared__ float f[NSGA_MAX][K], g[NSGA_MAX];
  __shared__ int ndom[NSGA_MAX], rank[NSGA_MAX], order[NSGA_MAX];
  __shared__ float crowd[NSGA_MAX];
  __shared__ unsigned char infront[NSGA_MAX], keep[NSGA_MAX];
  __shared__ int cnt, cum, r_cut, need;
  const int N = 2 * P, i = threadIdx.x;
  const bool on = i < N;
  if (on) {
    const float *src = i < P ? F + (int64_t)i * K : FC + (int64_t)(i - P) * K;
    for (int k = 0; k < K; ++k) f[i][k] = sanitize_obj(src[k]);   // NaN / inf objectives never survive (evolution_optimizer.py:104 F)
    g[i] = G ? sanitize_obj(i < P ? G[i] : GC[i - P]) : 0.0f;      // evolution_optimizer.py:105 G
    rank[i] = -1;
    keep[i] = 0;
    infront[i] = 0;
  }
  __syncthreads();
  if (on && i >= P) {
    // duplicate elimination: a child equal to a population member or to an earlier child is discarded
    if (dup_of_earlier(X, C, P, D, i)) {
      for (int k = 0; k < K; ++k) f[i][k] = INFINITY;
      if (G) g[i] = INFINITY;
    }
  }
  // ---- stable compaction of the kept rows into the next population
  auto compact = [&]() {
    if (on && keep[i]) {
      int dst = 0;
      for (int j = 0; j < i; ++j) dst += keep[j];
      const float *src = merged_row(X, C, P, D, i);
      float *row = Xn + (int64_t)dst * D;
      for (int k = 0; k < D; ++k) row[k] = src[k];
      for (int k = 0; k < K; ++k) Fn[(int64_t)dst * K + k] = f[i][k];
      if (Gn) Gn[dst] = g[i];
      split_row(src, d, D - d, Xcn + (int64_t)dst * d, Xen + (int64_t)dst * (D - d));
    }
  };
  const bool live = on && g[i] <= 0.0f;   // feasible
  const int nf = __syncthreads_count(live);
  if (nf < P) {
    // ---- too few feasible rows: all of them survive, then the least infeasible ones (ascending G, ties by index)
    if (on) {
      int better = 0;
      if (!live)
        for (int j = 0; j < N; ++j) better += (!(g[j] <= 0.0f) && before_asc(g[j], j, g[i], i)) ? 1 : 0;
      keep[i] = (live || better < P - nf) ? 1 : 0;
    }
    __syncthreads();
    compact();
    return;
  }
  if (live) {
    int c = 0;
    for (int j = 0; j < N; ++j) c += (g[j] <= 0.0f && dominates<K>(f[j], f[i])) ? 1 : 0;
    ndom[i] = c;
  }
  if (i == 0) { cum = 0; r_cut = -1; need = 0; }
  __syncthreads();
  // ---- front peeling of the feasible rows until P survivors are covered
  for (int r = 0; r < N; ++r) {
    if (i == 0) cnt = 0;
    __syncthreads();
    if (live && rank[i] < 0 && ndom[i] == 0) {
      infront[i] = 1;
      atomicAdd(&cnt, 1);
    }
    __syncthreads();
    const int c = cnt;
    if (c == 0) break;
    if (on && infront[i]) rank[i] = r;
    if (i == 0) {
      if (r_cut < 0 && cum + c >= P) { r_cut = r; need = P - cum; }
      cum += c;
    }
    __syncthreads();
    if (r_cut >= 0) break;
    if (live && rank[i] < 0) {
      int sub = 0;
      for (int j = 0; j < N; ++j)
        if (infront[j]) sub += dominates<K>(f[j], f[i]) ? 1 : 0;
      ndom[i] -= sub;
    }
    __syncthreads();
    if (on) infront[i] = 0;
    __syncthreads();
  }
  // ---- whole fronts below the cut survive; the cut front is truncated by descending crowding distance
  const int rc = r_cut;
  if (on) {
    keep[i] = (rc >= 0 && rank[i] >= 0 && rank[i] < rc) ? 1 : 0;
    crowd[i] = 0.0f;
  }
  __syncthreads();
  const bool mine = on && rc >= 0 && rank[i] == rc;
  for (int k = 0; k < K; ++k) {
    // position of i inside the cut front along objective k (counting sort, ties by index), then its neighbours
    int pos = 0, m = 0;
    float fmin = INFINITY, fmax = -INFINITY;
    if (mine) {
      for (int j = 0; j < N; ++j)
        if (rank[j] == rc) {
          ++m;
          pos += before_asc(f[j][k], j, f[i][k], i) ? 1 : 0;
          fmin = fminf(fmin, f[j][k]);
          fmax = fmaxf(fmax, f[j][k]);
        }
      order[pos] = i;
    }
    __syncthreads();
    if (mine) {
      if (pos == 0 || pos == m - 1) crowd[i] = INFINITY;
      else crowd[i] = crowd_interior(crowd[i], f[order[pos - 1]][k], f[order[pos + 1]][k], fmin, fmax);
    }
    __syncthreads();
  }
  if (mine) {
    int better = 0;
    for (int j = 0; j < N; ++j)
      if (rank[j] == rc) better += before_desc(crowd[j], j, crowd[i], i) ? 1 : 0;
    if (better < need) keep[i] = 1;
  }
  __syncthreads();
  compact();
}

// ---- multi-CTA survival for 512 < 2P <= 32768 merged rows: one persistent cooperative kernel (grid sized by occupancy,
// every phase separated by a grid barrier), so a call is one launch and never reads anything back to the host whatever
// the number of fronts.  Same rules and results as nsga_survive_kernel (see above); how it gets there:
//  * duplicates: rows are hashed into a bucket table.  The key of a coordinate is 0 for |v| < 2^-20 and its bit pattern
//    otherwise; the fp32 spacing above 2^-20 exceeds 1e-16, so two rows the predicate calls equal always share a bucket.
//    A child then tests the exact predicate against the lower merged indices of its bucket only.  Bucket chains are
//    built with atomicExch, so their order varies from run to run; the answer (does an equal earlier row exist) does not;
//  * ranks: the N^2 dominance counts are tiled through shared memory, one 8-lane team per row.  Fronts are appended to
//    one list in peeling order (front r at [start_r, start_r + cnt_r)); a round subtracts front r's dominance from every
//    unranked row and appends the rows whose count reaches zero to front r + 1.  One grid barrier per front: the cost
//    grows linearly with the number of fronts peeled (P of them when the objectives are totally ordered);
//  * cut front: each member's position along f_k (counting, ties by index) gives the sorted order, the members then add
//    their crowding terms for k = 0, 1, 2 in that order, and a second count against the cut front ranks the crowding;
//  * output: a per-CTA count + exclusive scan maps survivors to ascending rows, then a coalesced copy;
//  * constraints: every CTA counts the feasible rows it sanitised (population) or de-duplicated (children), and after
//    the barrier every CTA adds the per-CTA counts in CTA order, so all of them take the same branch.  Infeasible rows get
//    rank -2 and NaN objectives as sweep columns (NaN never dominates); with fewer than P feasible rows one tiled count
//    of (G, index) among the infeasible rows replaces phases 3-7.
// Only integer atomics are used and every float is computed by one thread in a fixed order: outputs are bit-identical
// from run to run.
constexpr int NSGA_LARGE_MAX_POP = 16384;
constexpr int NSGA_LT = 512;                       // threads per CTA
constexpr int NSGA_TEAM = 8;                       // lanes per row in the tiled sweeps
constexpr int NSGA_ROWS = NSGA_LT / NSGA_TEAM;     // rows per CTA pass
constexpr int NSGA_TJ = 1024;                      // shared-memory tile of the swept set
constexpr int NSGA_GRID_MAX = 1024;

template <int K>
struct SweepEntryK {
  float v[K];
  int id;
};
using SweepEntry = SweepEntryK<3>;

struct SurviveWs {
  float *f;       // [K][N] sanitised objectives (duplicates -> +inf)
  float *g;       // [N] sanitised constraint (0 without one; duplicates -> +inf with one)
  int *ndom;      // [N] dominator count; phase 1 parks the bucket index here
  int *rank;      // [N] front index, -1 = not yet ranked
  int *list;      // [N] the fronts in peeling order
  int *cnt;       // [N + 2] size of front r
  int *head;      // [H] bucket -> last inserted merged row
  int *next;      // [N] bucket chains
  int *pos;       // [K][N] position of cut-front member a along f_k
  int *order;     // [K][N] cut-front members sorted along f_k
  float *crowd;   // [N] crowding of cut-front member a
  int *keep;      // [N]
  int *sel;       // [P] survivor r -> merged row
  int *bsum;      // [NSGA_GRID_MAX] survivors per CTA
  int *fsum;      // [NSGA_GRID_MAX] feasible rows per CTA
  int H;          // bucket count (power of two)
};

static int64_t nsga_buckets(int64_t P) {
  int64_t H = 1;
  while (H < 4 * P) H <<= 1;
  return H;
}

// K objectives per merged row (the single-objective GA survivals carve the K = 3 layout)
size_t nsga_survive_ws_bytes(int64_t P, int64_t K = 3) {
  const int64_t N = 2 * P;
  const int64_t words[] = {K * N, N, N, N, N, N + 2, nsga_buckets(P), N, K * N, K * N, N, N, P, NSGA_GRID_MAX, NSGA_GRID_MAX};
  size_t total = 0;
  for (int64_t w : words) total += (size_t)round_up(w * 4, 256);
  return total;
}

static SurviveWs nsga_carve(void *ws, int64_t P, int64_t K = 3) {
  const int64_t N = 2 * P, H = nsga_buckets(P);
  char *p = (char *)ws;
  auto take = [&](int64_t words) {
    char *q = p;
    p += round_up(words * 4, 256);
    return q;
  };
  SurviveWs w;
  w.f = (float *)take(K * N);
  w.g = (float *)take(N);
  w.ndom = (int *)take(N);
  w.rank = (int *)take(N);
  w.list = (int *)take(N);
  w.cnt = (int *)take(N + 2);
  w.head = (int *)take(H);
  w.next = (int *)take(N);
  w.pos = (int *)take(K * N);
  w.order = (int *)take(K * N);
  w.crowd = (float *)take(N);
  w.keep = (int *)take(N);
  w.sel = (int *)take(P);
  w.bsum = (int *)take(NSGA_GRID_MAX);
  w.fsum = (int *)take(NSGA_GRID_MAX);
  w.H = (int)H;
  return w;
}

__device__ __forceinline__ uint32_t row_bucket(const float *row, int D, int H) {
  uint32_t h = 0x811C9DC5u;
  for (int k = 0; k < D; ++k) {
    const float v = row[k];
    const uint32_t key = fabsf(v) < 0x1p-20f ? 0u : __float_as_uint(v);   // -0, +0 and everything within 2^-20 of 0 agree
    h = (h ^ key) * 0x01000193u;
    h ^= h >> 15;
  }
  h ^= h >> 16;
  h *= 0x85EBCA6Bu;
  h ^= h >> 13;
  h *= 0xC2B2AE35u;
  h ^= h >> 16;
  return h & (uint32_t)(H - 1);
}

// Steps shared by the multi-CTA survivals.  bucket_rows puts every merged row into its bucket (the bucket index is parked
// in w.ndom); after a grid barrier dup_in_bucket tests child i with the exact predicate against the lower merged indices
// of its bucket.
__device__ __forceinline__ void bucket_rows(const float *X, const float *C, int P, int D, const SurviveWs &w, int gtid, int gsz) {
  for (int i = gtid; i < 2 * P; i += gsz) {
    const int b = (int)row_bucket(merged_row(X, C, P, D, i), D, w.H);
    w.ndom[i] = b;
    w.next[i] = atomicExch(&w.head[b], i);
  }
}

__device__ __forceinline__ bool dup_in_bucket(const float *X, const float *C, int P, int D, const SurviveWs &w, int i) {
  const float *me = C + (int64_t)(i - P) * D;
  bool dup = false;
  for (int j = __ldcg(&w.head[__ldcg(&w.ndom[i])]); j >= 0 && !dup; j = __ldcg(&w.next[j]))
    dup = j < i && same_row(merged_row(X, C, P, D, j), me, D);
  return dup;
}

// coalesced copy of the survivors: output row r < total is merged row sel[r], with its Xc / Xe split
__device__ __forceinline__ void copy_survivors(const float *X, const float *C, int P, int D, int d, const int *sel, int total,
                                               float *Xn, float *Xcn, int32_t *Xen, int gtid, int gsz) {
  const int e = D - d;
  for (int64_t q = gtid; q < (int64_t)total * D; q += gsz) {
    const int r = (int)(q / D), k = (int)(q % D);
    Xn[q] = merged_row(X, C, P, D, __ldcg(sel + r))[k];
  }
  for (int64_t q = gtid; q < (int64_t)total * d; q += gsz) {
    const int r = (int)(q / d), k = (int)(q % d);
    Xcn[q] = merged_row(X, C, P, D, __ldcg(sel + r))[k];
  }
  for (int64_t q = gtid; q < (int64_t)total * e; q += gsz) {
    const int r = (int)(q / e), k = (int)(q % e);
    Xen[q] = (int32_t)rintf(merged_row(X, C, P, D, __ldcg(sel + r))[d + k]);
  }
}

// Tiled count: for every row r < nr (one 8-lane team each), acc[0..K-1] = sums of test(me, entry) over the nc entries of
// the swept set, staged NSGA_TJ at a time in shared memory; out(r, me, acc) runs on the team's lane 0.  Every thread of
// the CTA must call it (it holds __syncthreads and warp shuffles).
template <int K, class Row, class Col, class Test, class Out>
__device__ __forceinline__ void team_sweep(SweepEntryK<K> *tile, int nr, int nc, Row row, Col col, Test test, Out out) {
  const int team = threadIdx.x / NSGA_TEAM, lane = threadIdx.x % NSGA_TEAM;
  for (int base = blockIdx.x * NSGA_ROWS; base < nr; base += gridDim.x * NSGA_ROWS) {
    const int r = base + team;
    SweepEntryK<K> me;
    const bool act = r < nr && row(r, me);
    int acc[K] = {};
    for (int c0 = 0; c0 < nc; c0 += NSGA_TJ) {
      const int ce = min(NSGA_TJ, nc - c0);
      __syncthreads();
      for (int t = threadIdx.x; t < ce; t += blockDim.x) tile[t] = col(c0 + t);
      __syncthreads();
      if (act)
        for (int t = lane; t < ce; t += NSGA_TEAM) test(me, tile[t], acc);
    }
#pragma unroll
    for (int o = NSGA_TEAM / 2; o > 0; o >>= 1)
#pragma unroll
      for (int k = 0; k < K; ++k) acc[k] += __shfl_xor_sync(0xFFFFFFFFu, acc[k], o);
    if (act && lane == 0) out(r, me, acc);
  }
}

template <int K>
__global__ void __launch_bounds__(NSGA_LT, 2) nsga_survive_large_kernel(const float *__restrict__ X, const float *__restrict__ F,
                                                                        const float *__restrict__ G, const float *__restrict__ C,
                                                                        const float *__restrict__ FC, const float *__restrict__ GC,
                                                                        int P, int D, int d, float *__restrict__ Xn,
                                                                        float *__restrict__ Fn, float *__restrict__ Gn,
                                                                        float *__restrict__ Xcn, int32_t *__restrict__ Xen,
                                                                        const SurviveWs w_arg) {
  namespace cg = cooperative_groups;
  using Entry = SweepEntryK<K>;
  SurviveWs w = w_arg;
  cg::grid_group grid = cg::this_grid();
  __shared__ Entry tile[NSGA_TJ];
  __shared__ int s_warp[NSGA_LT / 32], s_base, s_feas;
  const int N = 2 * P;
  const int gtid = blockIdx.x * blockDim.x + threadIdx.x, gsz = gridDim.x * blockDim.x;
  auto obj = [&](int j) {   // written in this kernel: read through L2 after a grid barrier
    Entry e;
#pragma unroll
    for (int k = 0; k < K; ++k) e.v[k] = __ldcg(w.f + k * N + j);
    e.id = j;
    return e;
  };
  auto feasible = [&](int j) { return __ldcg(w.g + j) <= 0.0f; };
  if (threadIdx.x == 0) s_feas = 0;
  __syncthreads();
  int nfeas = 0;   // feasible rows this thread sanitised (population) or de-duplicated (children)

  // ---- 0: sanitise, clear the bucket table and the front sizes
  for (int i = gtid; i < N; i += gsz) {
    const float *src = i < P ? F + (int64_t)i * K : FC + (int64_t)(i - P) * K;
#pragma unroll
    for (int k = 0; k < K; ++k) w.f[k * N + i] = sanitize_obj(src[k]);
    const float gi = G ? sanitize_obj(i < P ? G[i] : GC[i - P]) : 0.0f;
    w.g[i] = gi;
    nfeas += (i < P && gi <= 0.0f) ? 1 : 0;
  }
  for (int h = gtid; h < w.H; h += gsz) w.head[h] = -1;
  for (int r = gtid; r < N + 2; r += gsz) w.cnt[r] = 0;
  grid.sync();
  // ---- 1: bucket every merged row
  bucket_rows(X, C, P, D, w, gtid, gsz);
  grid.sync();
  // ---- 2: duplicate children
  for (int i = P + gtid; i < N; i += gsz) {
    const bool dup = dup_in_bucket(X, C, P, D, w, i);
    float gi = __ldcg(w.g + i);
    if (dup) {
#pragma unroll
      for (int k = 0; k < K; ++k) w.f[k * N + i] = INFINITY;
      if (G) w.g[i] = gi = INFINITY;
    }
    nfeas += gi <= 0.0f ? 1 : 0;
  }
  atomicAdd(&s_feas, nfeas);
  __syncthreads();
  if (threadIdx.x == 0) w.fsum[blockIdx.x] = s_feas;
  grid.sync();
  if (threadIdx.x == 0) {
    int nf = 0;
    for (int b = 0; b < (int)gridDim.x; ++b) nf += __ldcg(w.fsum + b);
    s_feas = nf;
  }
  __syncthreads();
  const int nf = s_feas;
  if (nf < P) {
    // ---- 3': too few feasible rows: all of them survive, then the P - nf least infeasible (ascending G, ties by index)
    auto cv_entry = [&](int j) {
      Entry e;
      e.v[0] = feasible(j) ? __int_as_float(0x7FC00000) : __ldcg(w.g + j);   // NaN: a feasible row is never counted
#pragma unroll
      for (int k = 1; k < K; ++k) e.v[k] = 0.0f;
      e.id = j;
      return e;
    };
    // feasible rows are kept here, the infeasible ones get their keep from the sweep below: disjoint writers, no barrier
    for (int i = gtid; i < N; i += gsz)
      if (feasible(i)) w.keep[i] = 1;
    team_sweep(
        tile, N, N,
        [&](int r, Entry &me) {
          if (feasible(r)) return false;
          me = cv_entry(r);
          return true;
        },
        cv_entry,
        [](const Entry &me, const Entry &o, int *acc) { acc[0] += before_asc(o.v[0], o.id, me.v[0], me.id) ? 1 : 0; },
        [&](int r, const Entry &, const int *acc) { w.keep[r] = acc[0] < P - nf ? 1 : 0; });
    grid.sync();
  } else {
    // ---- 3: dominator counts among the feasible rows; front 0
    auto live_entry = [&](int j) {
      Entry e = obj(j);
      if (!feasible(j))
#pragma unroll
        for (int k = 0; k < K; ++k) e.v[k] = __int_as_float(0x7FC00000);   // NaN never dominates
      return e;
    };
    team_sweep(
        tile, N, N,
        [&](int r, Entry &me) {
          if (!feasible(r)) {
            w.rank[r] = -2;
            return false;
          }
          me = obj(r);
          return true;
        },
        live_entry,
        [](const Entry &me, const Entry &o, int *acc) { acc[0] += dominates<K>(o.v, me.v) ? 1 : 0; },
        [&](int r, const Entry &, const int *acc) {
          w.ndom[r] = acc[0];
          w.rank[r] = acc[0] == 0 ? 0 : -1;
          if (acc[0] == 0) w.list[atomicAdd(&w.cnt[0], 1)] = r;
        });
    grid.sync();
    // ---- 4: peel fronts until P rows are covered (every CTA reads the same counts, so all leave at the same round)
    int start = 0, rc = -1, need = 0;
    for (int r = 0; r < N; ++r) {
      const int c = __ldcg(&w.cnt[r]);
      if (c == 0) break;
      if (start + c >= P) { rc = r; need = P - start; break; }
      const int nxt = start + c;
      team_sweep(
          tile, N, c,
          [&](int i, Entry &me) {
            if (__ldcg(&w.rank[i]) != -1) return false;   // ranked or infeasible
            me = obj(i);
            return true;
          },
          [&](int t) { return obj(__ldcg(&w.list[start + t])); },
          [](const Entry &me, const Entry &o, int *acc) { acc[0] += dominates<K>(o.v, me.v) ? 1 : 0; },
          [&](int i, const Entry &, const int *acc) {
            if (acc[0] == 0) return;
            const int nd = __ldcg(&w.ndom[i]) - acc[0];
            w.ndom[i] = nd;
            if (nd == 0) {
              w.rank[i] = r + 1;
              w.list[nxt + atomicAdd(&w.cnt[r + 1], 1)] = i;
            }
          });
      start = nxt;
      grid.sync();
    }
    const int m = rc >= 0 ? __ldcg(&w.cnt[rc]) : 0;
    const int *front = w.list + start;
    // ---- 5: cut front: positions along f_0 .. f_{K-1}; whole fronts below the cut survive
    for (int i = gtid; i < N; i += gsz) {
      const int rk = __ldcg(&w.rank[i]);
      w.keep[i] = (rc >= 0 && rk >= 0 && rk < rc) ? 1 : 0;
    }
    team_sweep(
        tile, m, m, [&](int a, Entry &me) { me = obj(__ldcg(front + a)); return true; },
        [&](int t) { return obj(__ldcg(front + t)); },
        [](const Entry &me, const Entry &o, int *acc) {
#pragma unroll
          for (int k = 0; k < K; ++k) acc[k] += before_asc(o.v[k], o.id, me.v[k], me.id) ? 1 : 0;
        },
        [&](int a, const Entry &me, const int *acc) {
#pragma unroll
          for (int k = 0; k < K; ++k) {
            w.pos[k * N + a] = acc[k];
            w.order[k * N + acc[k]] = me.id;
          }
        });
    grid.sync();
    // ---- 6: crowding, k = 0 .. K-1 in order, by the member itself
    for (int a = gtid; a < m; a += gsz) {
      float cr = 0.0f;
#pragma unroll
      for (int k = 0; k < K; ++k) {
        const float *fk = w.f + k * N;
        const int *ok = w.order + k * N;
        const int p = __ldcg(w.pos + k * N + a);
        if (p == 0 || p == m - 1) cr = INFINITY;
        else cr = crowd_interior(cr, __ldcg(fk + __ldcg(ok + p - 1)), __ldcg(fk + __ldcg(ok + p + 1)), __ldcg(fk + __ldcg(ok)),
                                 __ldcg(fk + __ldcg(ok + m - 1)));
      }
      w.crowd[a] = cr;
    }
    grid.sync();
    // ---- 7: the `need` members with the largest crowding survive
    auto crowd_entry = [&](int a) {
      Entry e;
      e.v[0] = __ldcg(w.crowd + a);
#pragma unroll
      for (int k = 1; k < K; ++k) e.v[k] = 0.0f;
      e.id = __ldcg(front + a);
      return e;
    };
    team_sweep(
        tile, m, m, [&](int a, Entry &me) { me = crowd_entry(a); return true; }, crowd_entry,
        [](const Entry &me, const Entry &o, int *acc) { acc[0] += before_desc(o.v[0], o.id, me.v[0], me.id) ? 1 : 0; },
        [&](int, const Entry &me, const int *acc) {
          if (acc[0] < need) w.keep[me.id] = 1;
        });
    grid.sync();
  }
  // ---- 8: survivors -> ascending output rows (CTA b owns merged rows [b * chunk, (b + 1) * chunk))
  const int chunk = (int)ceil_div(N, gridDim.x);
  const int r0 = blockIdx.x * chunk, r1 = min(N, r0 + chunk);
  int kept = 0;
  for (int t0 = r0; t0 < r1; t0 += blockDim.x) {
    const int i = t0 + threadIdx.x;
    kept += __syncthreads_count(i < r1 && __ldcg(w.keep + i));
  }
  if (threadIdx.x == 0) w.bsum[blockIdx.x] = kept;
  grid.sync();
  if (threadIdx.x == 0) {
    int b0 = 0;
    for (int b = 0; b < (int)blockIdx.x; ++b) b0 += __ldcg(w.bsum + b);
    s_base = b0;
  }
  __syncthreads();
  int base = s_base;
  const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;
  for (int t0 = r0; t0 < r1; t0 += blockDim.x) {
    const int i = t0 + threadIdx.x;
    const bool k = i < r1 && __ldcg(w.keep + i);
    const unsigned bal = __ballot_sync(0xFFFFFFFFu, k);
    if (lane == 0) s_warp[warp] = __popc(bal);
    __syncthreads();
    int off = base;
    for (int q = 0; q < warp; ++q) off += s_warp[q];
    if (k) w.sel[off + __popc(bal & ((1u << lane) - 1u))] = i;
    for (int q = 0; q < NSGA_LT / 32; ++q) base += s_warp[q];
    __syncthreads();
  }
  grid.sync();
  int total = 0;
  for (int b = 0; b < (int)gridDim.x; ++b) total += __ldcg(w.bsum + b);
  // ---- 9: coalesced copy of the survivors
  for (int64_t q = gtid; q < (int64_t)total * K; q += gsz) {
    const int r = (int)(q / K), k = (int)(q % K);
    Fn[q] = __ldcg(w.f + k * N + __ldcg(w.sel + r));
  }
  if (Gn)
    for (int q = gtid; q < total; q += gsz) Gn[q] = __ldcg(w.g + __ldcg(w.sel + q));
  copy_survivors(X, C, P, D, d, w.sel, total, Xn, Xcn, Xen, gtid, gsz);
}

// ---- single-objective survival (hb_ga_survive, hb_ga_survive_cv): pymoo's FitnessSurvival as MixedVariableGA runs it for
// a one-objective acquisition (evolution_optimizer.py:123-124,132-133).  The ordering rule is recalled from pymoo 0.6 --
// np.lexsort([F, cv]) then pop[S[:n_survive]] -- and was not checked against pymoo.  On the merged rows (population
// 0..P-1, offspring P..2P-1, one objective f each):
//  * sanitising: a non-finite f becomes +inf; with a constraint column (CV), cv = max(G, 0), a non-finite G becomes +inf;
//  * duplicates: the predicate of the NSGA-II survival above (|o[k] - me[k]| <= 1e-16f in every column against any
//    earlier merged row); a duplicate child gets f = +inf (and cv = +inf);
//  * survivors: the P merged rows first in ascending (f, merged index) order -- (cv, f, merged index) with CV -- written
//    in that order (row 0 = the best); F_next holds the sanitised f, G_next the sanitised cv.
// A row's output slot is its rank, the count of merged rows with a smaller key.  The keys are distinct, so the ranks are
// a permutation and a row with rank < P writes its slot directly: no scan, no float atomics, the same bytes from both
// kernels and from run to run.  With G = 0 everywhere the order is the unconstrained one, except among the f = +inf rows
// when one of them is a duplicate child (cv = +inf here).
__device__ __forceinline__ float sanitize_cv(float v) { return isfinite(v) ? (v > 0.0f ? v : 0.0f) : INFINITY; }

// (gj, fj, j) before (gi, fi, i) in ascending lexicographic order
__device__ __forceinline__ bool before_lex(float gj, float fj, int j, float gi, float fi, int i) {
  return gj < gi || (gj == gi && before_asc(fj, j, fi, i));
}

template <bool CV>
__global__ void __launch_bounds__(NSGA_MAX) ga_survive_kernel(const float *__restrict__ X, const float *__restrict__ F,
                                                              const float *__restrict__ G, const float *__restrict__ C,
                                                              const float *__restrict__ FC, const float *__restrict__ GC, int P,
                                                              int D, int d, float *__restrict__ Xn, float *__restrict__ Fn,
                                                              float *__restrict__ Gn, float *__restrict__ Xcn,
                                                              int32_t *__restrict__ Xen) {
  __shared__ float f[NSGA_MAX], g[CV ? NSGA_MAX : 1];
  const int N = 2 * P, i = threadIdx.x;
  const bool on = i < N;
  if (on) {
    f[i] = sanitize_obj(i < P ? F[i] : FC[i - P]);
    if (CV) g[i] = sanitize_cv(i < P ? G[i] : GC[i - P]);
    if (i >= P && dup_of_earlier(X, C, P, D, i)) {
      f[i] = INFINITY;
      if (CV) g[i] = INFINITY;
    }
  }
  __syncthreads();
  if (!on) return;
  int rank = 0;
  for (int j = 0; j < N; ++j) rank += (CV ? before_lex(g[j], f[j], j, g[i], f[i], i) : before_asc(f[j], j, f[i], i)) ? 1 : 0;
  if (rank >= P) return;
  const float *src = merged_row(X, C, P, D, i);
  float *row = Xn + (int64_t)rank * D;
  for (int k = 0; k < D; ++k) row[k] = src[k];
  Fn[rank] = f[i];
  if (CV) Gn[rank] = g[i];
  split_row(src, d, D - d, Xcn + (int64_t)rank * d, Xen + (int64_t)rank * (D - d));
}

// multi-CTA form for 512 < 2P <= 32768: duplicates through the bucket table, ranks by the tiled count, then the copy
template <bool CV>
__global__ void __launch_bounds__(NSGA_LT, 2) ga_survive_large_kernel(const float *__restrict__ X, const float *__restrict__ F,
                                                                      const float *__restrict__ G, const float *__restrict__ C,
                                                                      const float *__restrict__ FC, const float *__restrict__ GC,
                                                                      int P, int D, int d, float *__restrict__ Xn,
                                                                      float *__restrict__ Fn, float *__restrict__ Gn,
                                                                      float *__restrict__ Xcn, int32_t *__restrict__ Xen,
                                                                      const SurviveWs w_arg) {
  namespace cg = cooperative_groups;
  SurviveWs w = w_arg;
  cg::grid_group grid = cg::this_grid();
  __shared__ SweepEntry tile[NSGA_TJ];
  const int N = 2 * P;
  const int gtid = blockIdx.x * blockDim.x + threadIdx.x, gsz = gridDim.x * blockDim.x;
  // ---- 0: sanitise, clear the bucket table
  for (int i = gtid; i < N; i += gsz) {
    w.f[i] = sanitize_obj(i < P ? F[i] : FC[i - P]);
    if (CV) w.g[i] = sanitize_cv(i < P ? G[i] : GC[i - P]);
  }
  for (int h = gtid; h < w.H; h += gsz) w.head[h] = -1;
  grid.sync();
  // ---- 1: bucket every merged row
  bucket_rows(X, C, P, D, w, gtid, gsz);
  grid.sync();
  // ---- 2: duplicate children
  for (int i = P + gtid; i < N; i += gsz)
    if (dup_in_bucket(X, C, P, D, w, i)) {
      w.f[i] = INFINITY;
      if (CV) w.g[i] = INFINITY;
    }
  grid.sync();
  // ---- 3: rank = count of smaller keys; the survivors write their output slot
  auto key = [&](int j) {
    SweepEntry e;
    e.v[0] = __ldcg(w.f + j);
    e.v[1] = CV ? __ldcg(w.g + j) : 0.0f;
    e.v[2] = 0.0f;
    e.id = j;
    return e;
  };
  team_sweep(
      tile, N, N, [&](int r, SweepEntry &me) { me = key(r); return true; }, key,
      [](const SweepEntry &me, const SweepEntry &o, int *acc) {
        acc[0] += (CV ? before_lex(o.v[1], o.v[0], o.id, me.v[1], me.v[0], me.id) : before_asc(o.v[0], o.id, me.v[0], me.id)) ? 1 : 0;
      },
      [&](int r, const SweepEntry &, const int *acc) {
        if (acc[0] < P) w.sel[acc[0]] = r;
      });
  grid.sync();
  // ---- 4: coalesced copy of the survivors
  for (int q = gtid; q < P; q += gsz) {
    const int s = __ldcg(w.sel + q);
    Fn[q] = __ldcg(w.f + s);
    if (CV) Gn[q] = __ldcg(w.g + s);
  }
  copy_survivors(X, C, P, D, d, w.sel, P, Xn, Xcn, Xen, gtid, gsz);
}

// CTAs of a cooperative survival kernel: co-resident CTAs on the current device (at most 2 per SM, looked up once per
// device), no more than row passes of the N-row sweeps, and no more than the per-CTA counts the workspace holds
template <class Kernel>
static int survive_grid(Kernel kernel, PerDevice &once, int64_t P, int *grid) {
  bool fresh = false;
  const int dev = once.slot(&fresh);
  if (dev < 0) return HB_ERR_CUDA;
  if (fresh) {
    int sms = 0, per_sm = 0, coop = 0;
    HB_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    HB_CUDA(cudaDeviceGetAttribute(&coop, cudaDevAttrCooperativeLaunch, dev));
    HB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, NSGA_LT, 0));
    if (!coop || per_sm < 1) {
      set_error(cudaErrorNotSupported, "nsga_survive: cooperative launch unavailable");
      return HB_ERR_CUDA;
    }
    once.aux[dev] = sms * min(per_sm, 2);
    once.done[dev] = true;
  }
  *grid = (int)std::min<int64_t>({(int64_t)once.aux[dev], ceil_div(2 * P, NSGA_ROWS), (int64_t)NSGA_GRID_MAX});
  return HB_OK;
}
int launch_nsga_init(float *X, int64_t P, int64_t D, int64_t d, const int32_t *kind, const float *lb, const float *ub,
                     const float *fixed, const float *init, int64_t n_init, uint64_t seed, float *Xc, int32_t *Xe, cudaStream_t st) {
  if (P <= 0 || D <= 0 || d < 0 || d > D || n_init < 0 || n_init > P) return HB_ERR_INVALID;
  nsga_init_kernel<<<(int)ceil_div(P, 128), 128, 0, st>>>(X, (int)P, (int)D, (int)d, kind, lb, ub, fixed, init, (int)n_init, seed, Xc, Xe);
  count_launches(1);
  HB_LAUNCH_CHECK("nsga_init");
  return HB_OK;
}

int launch_nsga_mate(const float *X, int64_t P, int64_t D, int64_t d, const int32_t *kind, const float *lb, const float *ub,
                     const float *fixed, uint64_t seed, int gen, float *C, float *Cc, int32_t *Ce, cudaStream_t st) {
  if (P <= 0 || D <= 0 || d < 0 || d > D) return HB_ERR_INVALID;
  const float pm_prob = fminf(0.5f, 1.0f / (float)D);
  nsga_mate_kernel<<<(int)ceil_div((P + 1) / 2, 64), 64, 0, st>>>(X, (int)P, (int)D, (int)d, kind, lb, ub, fixed, seed, gen, pm_prob, C, Cc, Ce);
  count_launches(1);
  HB_LAUNCH_CHECK("nsga_mate");
  return HB_OK;
}

int64_t nsga_survive_ws_query(int64_t P, int64_t D, int64_t K) {
  if (P < 1 || P > NSGA_LARGE_MAX_POP || D < 1 || K < 2 || K > HB_MAX_OBJ) return -1;
  return (int64_t)nsga_survive_ws_bytes(P, K);
}

template <int K>
static int launch_nsga_survive_t(const float *X, const float *F, const float *G, const float *C, const float *FC, const float *GC,
                                 int64_t P, int64_t D, int64_t d, float *Xn, float *Fn, float *Gn, float *Xcn, int32_t *Xen,
                                 void *ws, int64_t ws_bytes, cudaStream_t st) {
  if (2 * P <= NSGA_MAX) {
    nsga_survive_kernel<K><<<1, NSGA_MAX, 0, st>>>(X, F, G, C, FC, GC, (int)P, (int)D, (int)d, Xn, Fn, Gn, Xcn, Xen);
    count_launches(1);
    HB_LAUNCH_CHECK("nsga_survive");
    return HB_OK;
  }
  if (!ws || ws_bytes < (int64_t)nsga_survive_ws_bytes(P, K)) return HB_ERR_INVALID;
  static PerDevice once;   // aux[dev] = co-resident CTAs of this cooperative survival kernel on that device
  int grid = 0;
  const int rc = survive_grid(nsga_survive_large_kernel<K>, once, P, &grid);
  if (rc != HB_OK) return rc;
  SurviveWs w = nsga_carve(ws, P, K);
  int Pi = (int)P, Di = (int)D, di = (int)d;
  void *args[] = {&X, &F, &G, &C, &FC, &GC, &Pi, &Di, &di, &Xn, &Fn, &Gn, &Xcn, &Xen, &w};
  HB_CUDA(cudaLaunchCooperativeKernel((const void *)nsga_survive_large_kernel<K>, dim3(grid), dim3(NSGA_LT), args, 0, st));
  count_launches(1);
  HB_LAUNCH_CHECK("nsga_survive_large");
  return HB_OK;
}

int launch_nsga_survive(const float *X, const float *F, const float *G, const float *C, const float *FC, const float *GC,
                        int64_t P, int64_t D, int64_t d, int64_t K, float *Xn, float *Fn, float *Gn, float *Xcn, int32_t *Xen,
                        void *ws, int64_t ws_bytes, cudaStream_t st) {
  if (P <= 0 || P > NSGA_LARGE_MAX_POP || D <= 0 || d < 0 || d > D) return HB_ERR_INVALID;
  if (!G != !GC || !G != !Gn) return HB_ERR_INVALID;
  switch (K) {
    case 2: return launch_nsga_survive_t<2>(X, F, G, C, FC, GC, P, D, d, Xn, Fn, Gn, Xcn, Xen, ws, ws_bytes, st);
    case 3: return launch_nsga_survive_t<3>(X, F, G, C, FC, GC, P, D, d, Xn, Fn, Gn, Xcn, Xen, ws, ws_bytes, st);
    case 4: return launch_nsga_survive_t<4>(X, F, G, C, FC, GC, P, D, d, Xn, Fn, Gn, Xcn, Xen, ws, ws_bytes, st);
    case 5: return launch_nsga_survive_t<5>(X, F, G, C, FC, GC, P, D, d, Xn, Fn, Gn, Xcn, Xen, ws, ws_bytes, st);
    case 6: return launch_nsga_survive_t<6>(X, F, G, C, FC, GC, P, D, d, Xn, Fn, Gn, Xcn, Xen, ws, ws_bytes, st);
    case 7: return launch_nsga_survive_t<7>(X, F, G, C, FC, GC, P, D, d, Xn, Fn, Gn, Xcn, Xen, ws, ws_bytes, st);
    case 8: return launch_nsga_survive_t<8>(X, F, G, C, FC, GC, P, D, d, Xn, Fn, Gn, Xcn, Xen, ws, ws_bytes, st);
    default: return HB_ERR_INVALID;
  }
}

template <bool CV>
static int launch_ga_survive_t(const float *X, const float *F, const float *G, const float *C, const float *FC, const float *GC,
                               int64_t P, int64_t D, int64_t d, float *Xn, float *Fn, float *Gn, float *Xcn, int32_t *Xen,
                               void *ws, int64_t ws_bytes, cudaStream_t st) {
  if (2 * P <= NSGA_MAX) {
    ga_survive_kernel<CV><<<1, (int)round_up(2 * P, 32), 0, st>>>(X, F, G, C, FC, GC, (int)P, (int)D, (int)d, Xn, Fn, Gn, Xcn, Xen);
    count_launches(1);
    HB_LAUNCH_CHECK("ga_survive");
    return HB_OK;
  }
  if (!ws || ws_bytes < (int64_t)nsga_survive_ws_bytes(P)) return HB_ERR_INVALID;
  static PerDevice once;   // aux[dev] = co-resident CTAs of this cooperative GA survival kernel on that device
  int grid = 0;
  const int rc = survive_grid(ga_survive_large_kernel<CV>, once, P, &grid);
  if (rc != HB_OK) return rc;
  SurviveWs w = nsga_carve(ws, P);
  int Pi = (int)P, Di = (int)D, di = (int)d;
  void *args[] = {&X, &F, &G, &C, &FC, &GC, &Pi, &Di, &di, &Xn, &Fn, &Gn, &Xcn, &Xen, &w};
  HB_CUDA(cudaLaunchCooperativeKernel((const void *)ga_survive_large_kernel<CV>, dim3(grid), dim3(NSGA_LT), args, 0, st));
  count_launches(1);
  HB_LAUNCH_CHECK("ga_survive_large");
  return HB_OK;
}

int launch_ga_survive(const float *X, const float *F, const float *G, const float *C, const float *FC, const float *GC, int64_t P,
                      int64_t D, int64_t d, float *Xn, float *Fn, float *Gn, float *Xcn, int32_t *Xen, void *ws, int64_t ws_bytes,
                      cudaStream_t st) {
  if (P <= 0 || P > NSGA_LARGE_MAX_POP || D <= 0 || d < 0 || d > D) return HB_ERR_INVALID;
  if (!G != !GC || !G != !Gn) return HB_ERR_INVALID;
  return G ? launch_ga_survive_t<true>(X, F, G, C, FC, GC, P, D, d, Xn, Fn, Gn, Xcn, Xen, ws, ws_bytes, st)
           : launch_ga_survive_t<false>(X, F, G, C, FC, GC, P, D, d, Xn, Fn, Gn, Xcn, Xen, ws, ws_bytes, st);
}

}  // namespace hb
