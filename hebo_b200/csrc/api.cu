// extern "C" entry points of libhebo_b200.so (declared in include/hebo_b200.h) and the native fit-loop
// runtime (the 100-epoch pSGLD loop of HEBO/hebo/models/gp/gp.py:96-135 without Python in the loop).
#include <stdio.h>
#include <string.h>

#include <atomic>
#include <vector>

#include "h16.cuh"
#include "kernels.h"

namespace hb {

static thread_local char g_err[512] = "";

void set_error(cudaError_t e, const char *where) {
  snprintf(g_err, sizeof(g_err), "%s: %s", where, cudaGetErrorString(e));
}

int check_launch(const char *where) {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_error(e, where);
    return HB_ERR_CUDA;
  }
  return HB_OK;
}

static std::atomic<long long> g_launches{0};
void count_launches(int n) { g_launches += n; }

// CUDA-event brackets around the dominant kernel (posterior variance contraction), recorded on the launching
// stream; enabled by bench.py through hb_profile_enable and read back with hb_profile_collect.
struct Prof {
  bool on = false;
  std::vector<cudaEvent_t> a, b;
  size_t used = 0;
};
static Prof g_prof;
void prof_begin(cudaStream_t st) {
  if (!g_prof.on) return;
  if (g_prof.used == g_prof.a.size()) {
    cudaEvent_t e0, e1;
    if (cudaEventCreate(&e0) != cudaSuccess || cudaEventCreate(&e1) != cudaSuccess) return;
    g_prof.a.push_back(e0);
    g_prof.b.push_back(e1);
  }
  cudaEventRecord(g_prof.a[g_prof.used], st);
}
void prof_end(cudaStream_t st) {
  if (!g_prof.on || g_prof.used >= g_prof.a.size()) return;
  cudaEventRecord(g_prof.b[g_prof.used], st);
  g_prof.used++;
}

// ---------------------------------------------------------------- fit workspace layout
constexpr int FIT_BATCH = 16;   // epochs replayed per host synchronisation (CUDA-graph fit loop)

struct FitWs {
  float *hyp, *grad, *sq, *loss;
  int32_t *info;          // [0] factorisation status, [1] epoch counter, [2] replay slot of the current batch (per output)
  double *scal;
  float *status;          // [FIT_BATCH][2]: (info, loss) of every epoch of a batch
  float *L, *Linv, *tmp, *alpha, *Zt, *cholws, *Linv_hi, *Linv_lo;
  float *Ets;             // = Zt + d * NP: embedding rows of the scaled feature matrix (mixed model)
  float *dZa, *dZb;       // [d, NP] d Zt / d a_k, d Zt / d b_k (warped model)
  float *tab_s;           // [T] embedding tables / embedding lengthscale (candidate side of the posterior)
  int32_t *meta, *Xe;     // categorical layout arrays (ModelSpec) and the training categories [n, e]
  TcBuffers tc;
  void *solvews, *gradws;
  size_t total;
};

static inline size_t al256(size_t x) { return (x + 255) / 256 * 256; }

// ---- ModelSpec from the C-ABI description; device arrays bound separately (they live in the fit workspace)
static bool build_spec(int64_t d, const hb_model_spec_t *c, ModelSpec &sp) {
  sp = ModelSpec();
  if (d < 0) return false;
  sp.d = (int)d;
  if (c) {
    sp.ard = c->ard_kernel ? 1 : 0;
    sp.warp = (sp.d > 0) ? c->warp : 0;
    if (sp.warp < 0 || sp.warp > 2) return false;
    sp.e = c->num_enum;
    if (sp.e < 0 || (sp.e > 0 && (!c->num_uniqs || !c->emb_sizes))) return false;
    for (int k = 0; k < sp.e; ++k) {
      if (c->num_uniqs[k] <= 0 || c->emb_sizes[k] <= 0) return false;
      sp.De += c->emb_sizes[k];
      sp.T += c->num_uniqs[k] * c->emb_sizes[k];
    }
  }
  return sp.dtot() > 0 && sp.dtot() <= HB_MAX_FEATURES;
}
static size_t meta_ints(const ModelSpec &sp) { return (size_t)2 * sp.De + 2 * sp.e + 3 * sp.T; }
static void bind_meta(ModelSpec &sp, const int32_t *meta, const int32_t *Xe) {
  if (sp.e <= 0) return;
  sp.q_col = meta;
  sp.q_loc = sp.q_col + sp.De;
  sp.tab_off = sp.q_loc + sp.De;
  sp.emb_size = sp.tab_off + sp.e;
  sp.ent_col = sp.emb_size + sp.e;
  sp.ent_u = sp.ent_col + sp.T;
  sp.ent_q = sp.ent_u + sp.T;
  sp.Xe = Xe;
}
static void fill_meta_host(const hb_model_spec_t *c, const ModelSpec &sp, std::vector<int32_t> &m) {
  m.assign(meta_ints(sp), 0);
  int32_t *q_col = m.data(), *q_loc = q_col + sp.De, *tab_off = q_loc + sp.De, *emb_size = tab_off + sp.e;
  int32_t *ent_col = emb_size + sp.e, *ent_u = ent_col + sp.T, *ent_q = ent_u + sp.T;
  int q = 0, t = 0;
  for (int k = 0; k < sp.e; ++k) {
    tab_off[k] = t;
    emb_size[k] = c->emb_sizes[k];
    for (int j = 0; j < c->emb_sizes[k]; ++j, ++q) {
      q_col[q] = k;
      q_loc[q] = j;
    }
    for (int u = 0; u < c->num_uniqs[k]; ++u)
      for (int j = 0; j < c->emb_sizes[k]; ++j, ++t) {   // nn.Embedding weight [num_uniq, emb_size], row-major
        ent_col[t] = k;
        ent_u[t] = u;
        ent_q[t] = j;
      }
  }
}

// The hi/lo companion buffers of the tensor-core stages, in this order: Linv_hi, Linv_lo, L_hi, L_lo, U_hi, U_lo, T_hi, T_lo
// ([NP, NP] each) and P_hi, P_lo ([NP, 512]), each block 256-byte aligned.  The fit workspace and the stand-alone
// tensor-core entry points (hb_tc_workspace_bytes) both carve them here, so the two layouts are one.
template <class Take> static TcBuffers carve_tc(Take &take, int64_t np) {
  const size_t sq = (size_t)np * np * 4, panel = (size_t)np * 512 * 4;
  TcBuffers tc;
  tc.Linv_hi = (float *)take(sq);
  tc.Linv_lo = (float *)take(sq);
  tc.L_hi = (float *)take(sq);
  tc.L_lo = (float *)take(sq);
  tc.U_hi = (float *)take(sq);
  tc.U_lo = (float *)take(sq);
  tc.T_hi = (float *)take(sq);
  tc.T_lo = (float *)take(sq);
  tc.P_hi = (float *)take(panel);
  tc.P_lo = (float *)take(panel);
  return tc;
}

// TcBuffers of a stand-alone tensor-core workspace at `base` (nullptr: only counts); `bytes` = its size
static TcBuffers carve_tc_ws(void *base, int64_t np, size_t &bytes) {
  unsigned char *p = reinterpret_cast<unsigned char *>(base);
  size_t off = 0;
  auto take = [&](size_t b) {
    void *r = p ? (void *)(p + off) : nullptr;
    off += al256(b);
    return r;
  };
  const TcBuffers tc = carve_tc(take, np);
  bytes = off;
  return tc;
}

static FitWs carve_fit(void *base, int64_t n, const ModelSpec &sp) {
  const int64_t np = round_up(n, TILE);
  const int64_t P = sp.P(), H = sp.H();
  unsigned char *p = reinterpret_cast<unsigned char *>(base);
  size_t off = 0;
  FitWs w;
  auto take = [&](size_t bytes) {
    void *r = p ? (void *)(p + off) : nullptr;
    off += al256(bytes);
    return r;
  };
  w.hyp = (float *)take(H * 4);
  w.grad = (float *)take(P * 4);
  w.sq = (float *)take(P * 4);
  w.loss = (float *)take(16);
  w.info = (int32_t *)take(16);
  w.scal = (double *)take(16);
  w.status = (float *)take(FIT_BATCH * 2 * sizeof(float));
  w.L = (float *)take((size_t)np * np * 4);
  w.Linv = (float *)take((size_t)np * np * 4);
  w.tmp = (float *)take((size_t)np * np * 4);
  w.tc = carve_tc(take, np);
  w.Linv_hi = w.tc.Linv_hi;
  w.Linv_lo = w.tc.Linv_lo;
  w.alpha = (float *)take((size_t)np * 4);
  w.Zt = (float *)take((size_t)sp.dtot() * np * 4);
  w.Ets = w.Zt ? w.Zt + (size_t)sp.d * np : nullptr;
  w.dZa = (float *)take(sp.warp ? (size_t)sp.d * np * 4 : 16);
  w.dZb = (float *)take(sp.warp ? (size_t)sp.d * np * 4 : 16);
  w.cholws = (float *)take((size_t)TILE * TILE * 4);
  w.solvews = take(solve_ws_bytes(np));
  w.gradws = take(grad_ws_bytes(np, sp));
  w.tab_s = (float *)take((size_t)(sp.T > 0 ? sp.T : 1) * 4);
  w.meta = (int32_t *)take((meta_ints(sp) + 1) * 4);
  w.Xe = (int32_t *)take(((size_t)n * sp.e + 1) * 4);
  w.total = off;
  return w;
}

struct HostStatus {
  int32_t info;
  float loss;
  int32_t set_epoch;
  int32_t pad;
  float batch[HB_MAX_OUTPUTS][FIT_BATCH * 2];   // per output: (info as float bits, loss) per replay slot
};
// host state of the fit on one DEVICE (the header allows one in-flight call per process and device): the pinned block the
// status words are read back into, and the stream an epoch is captured on
struct FitHost {
  HostStatus *status = nullptr;
  cudaStream_t capture = nullptr;
};
static int fit_host(FitHost *&h) {
  static PerDevice once;
  static FitHost per_dev[MAX_DEVICES];
  bool fresh = false;
  const int dev = once.slot(&fresh);
  if (dev < 0) return HB_ERR_CUDA;
  h = &per_dev[dev];
  if (fresh) {
    if (!h->status) HB_CUDA(cudaMallocHost(&h->status, sizeof(HostStatus)));
    HB_CUDA(cudaStreamCreateWithFlags(&h->capture, cudaStreamNonBlocking));
    once.done[dev] = true;
  }
  return HB_OK;
}

// conditional pSGLD (sgld.py:57-70): skipped on the device when the epoch's factorisation failed.  One block per output
// (Batch: raw rows P apart, Langevin draws num_epochs * P apart, the rest in the output's workspace slice).  The epoch
// index lives on the device (info[1], advanced on success only), so the same launch -- and a CUDA graph replay of it -- works
// for every epoch: the Langevin row is langevin[epoch] once epoch + 1 > pretrain (n_step is incremented first in the
// reference).  An output whose counter has reached num_epochs is done and never stepped again (the outputs of a batch
// advance independently).  (info, loss) of the attempt go to status[slot], slot = info[2]++.
__global__ void __launch_bounds__(256) psgld_guarded_kernel(float *__restrict__ raw, const float *__restrict__ grad,
                                                            float *__restrict__ sq, int p, float lr, float a, float eps,
                                                            float factor, const float *__restrict__ langevin, int pretrain,
                                                            int num_epochs, int32_t *__restrict__ info,
                                                            const float *__restrict__ loss, float *__restrict__ status,
                                                            const float *__restrict__ hyp, int nhyp, int frozen_begin,
                                                            int frozen_end, int64_t wss) {
  {
    const int b = blockIdx.x;
    raw += (int64_t)b * p;
    if (langevin) langevin += (int64_t)b * num_epochs * p;
    grad = slice(grad, wss, b);
    sq = slice(sq, wss, b);
    info = slice(info, wss, b);
    loss = slice(loss, wss, b);
    status = slice(status, wss, b);
    hyp = slice(hyp, wss, b);
  }
  // hopeless epoch: a constrained hyper-parameter is not finite or a lengthscale / outputscale has underflowed to zero
  // (pSGLD's Langevin step divides by sqrt(sqrt(v) + 1e-8): a parameter with a vanishing gradient random-walks in steps of
  // ~5 raw units, sgld.py:64-70).  K is then NaN, no jitter can repair it, and -- as in the reference, where the closure
  // raises before the optimiser updates anything (gp.py:111-126) -- no later epoch can change the parameters: status -1.
  __shared__ int bad;
  if (threadIdx.x == 0) bad = 0;
  __syncthreads();
  for (int i = threadIdx.x; i < nhyp; i += blockDim.x) {
    const float h = hyp[i];
    if (!isfinite(h) || (i != 1 && !(h > 0.0f))) bad = 1;
  }
  __syncthreads();
  const int ep = info[1], slot = info[2], ok = info[0] == 0 && !bad && ep < num_epochs;
  const float *xi = (langevin && (ep + 1) > pretrain) ? langevin + (int64_t)ep * p : nullptr;
  if (ok) {
    for (int i = threadIdx.x; i < p; i += blockDim.x) {
      if (i >= frozen_begin && i < frozen_end) continue;   // fixed (not learned) warp exponents are not optimiser parameters
      psgld_update(raw, grad, sq, i, lr, a, eps, factor, xi);
    }
  }
  __syncthreads();   // every thread has read the counters
  if (threadIdx.x == 0) {
    if (slot < FIT_BATCH) {
      status[2 * slot + 0] = __int_as_float(bad ? -1 : info[0]);
      status[2 * slot + 1] = loss[0];
    }
    info[2] = slot + 1;
    if (ok) info[1] = ep + 1;
  }
}

// gram -> cholesky at (hyp, jitter); info left on the device.  tc: the Cholesky's outer update on the tensor cores
// (nullptr: FP32 SIMT).  (mixed model: gathers the embedding features at the current tables / lengthscale first)
// bt: the outputs of a batch, w = the workspace of output 0, raw = its raw row.
static int factor_once(const float *Xt, int64_t n, int64_t np, const ModelSpec &sp, const float *raw, int kern,
                       const float *noise_diag, float jitter, FitWs &w, cudaStream_t st, const TcBuffers *tc,
                       const Batch &bt = Batch()) {
  HB_CUDA(memset_slices(w.info, 0, sizeof(int32_t), bt, st));
  int s = launch_emb_gather(raw + sp.i_tab(), sp, n, np, w.hyp, w.Ets, w.tab_s, st, bt);
  if (s != HB_OK) return s;
  if (sp.warp) {   // warped features (and their exponent derivatives) at the current a, b, lengthscales
    s = launch_scale_zt(Xt, np, sp, w.hyp, w.Zt, w.dZa, w.dZb, st, bt);
    if (s != HB_OK) return s;
  }
  s = launch_gram(sp.warp ? w.Zt : Xt, w.Ets, n, np, sp, w.hyp, kern, noise_diag, jitter, w.L, st, bt);
  if (s != HB_OK) return s;
  return launch_cholesky(w.L, np, w.cholws, w.info, st, tc, bt);
}

// one MLL forward + backward at `raw`: transform -> [gather] -> Gram -> Cholesky -> L^-1 -> alpha / log-det -> K^-1 ->
// gradient, into w.grad / w.loss (factorisation status in w.info).  tc: the GEMM stages on the 3xTF32 tensor cores, with
// zero_fill on the first use of the workspace in a fit (see launch_tri_inverse_tc); nullptr: FP32 SIMT.
// bt: all outputs of a batch (tensor-core path only), w / raw / y those of output 0.
static int enqueue_mll(const float *Xt, const float *y, int64_t n, int64_t np, const ModelSpec &sp, const float *raw, int kern,
                       const float *noise_diag, float noise_lb, float noise_guess, float jitter, FitWs &w, cudaStream_t st,
                       const TcBuffers *tc, bool zero_fill, const Batch &bt = Batch()) {
  if (!tc && bt.nout != 1) return HB_ERR_INVALID;
  int s = launch_transform_hypers(raw, sp, noise_lb, w.hyp, st, bt);
  if (s != HB_OK) return s;
  s = factor_once(Xt, n, np, sp, raw, kern, noise_diag, jitter, w, st, tc, bt);
  if (s != HB_OK) return s;
  s = tc ? launch_tri_inverse_tc(w.L, np, w.Linv, *tc, zero_fill, st, bt) : launch_tri_inverse(w.L, np, w.Linv, w.tmp, st);
  if (s != HB_OK) return s;
  s = launch_solve_logdet(w.L, w.Linv, y, n, np, w.hyp, w.alpha, w.scal, w.solvews, st, bt);
  if (s != HB_OK) return s;
  s = tc ? launch_kinv_tc(np, w.tmp, *tc, st, bt) : launch_kinv(w.Linv, np, w.tmp, st);
  if (s != HB_OK) return s;
  return launch_mll_grad(sp.warp ? w.Zt : Xt, w.Ets, n, np, sp, raw, w.hyp, kern, w.tmp, w.alpha, w.scal, noise_guess, w.grad,
                         w.loss, w.gradws, st, w.dZa, w.dZb, bt);
}

static float next_jitter(float j) { return j == 0.0f ? 1e-6f : j * 10.0f; }   // fp32 ladder of gp.py:104-110
constexpr float JITTER_MAX = 1e3f;                                             // 100 * (jitter <= 10), gp.py:121

// jitter ladder of gp.py:104-126: attempt(jitter, info) at jitter 0, 1e-6, 1e-5, .. until info is 0 (success) or -1 (hopeless,
// see psgld_guarded_kernel: no jitter can help).  HB_ERR_NOT_PD once the next jitter exceeds JITTER_MAX (`jitter` = that one).
template <class Attempt> static int jitter_ladder(Attempt &&attempt, float &jitter, int32_t &info) {
  for (jitter = 0.0f; jitter <= JITTER_MAX; jitter = next_jitter(jitter)) {
    const int s = attempt(jitter, info);
    if (s != HB_OK || info == 0 || info == -1) return s;
  }
  return HB_ERR_NOT_PD;
}

// start of every entry point that trains or factorises in a fit workspace of num_out slices: checks the shared arguments,
// builds the model description, carves slice 0 into w and uploads the categorical layout arrays + training categories into
// every slice (each slice is a complete workspace); sp is bound to slice 0's copy
static int open_fit_ws(const float *Xt, const int32_t *Xe, const float *y, int64_t n, int64_t d, const hb_model_spec_t *spec,
                       const float *raw, int32_t kern, void *ws, int64_t ws_bytes, int64_t num_out, cudaStream_t st,
                       ModelSpec &sp, FitWs &w) {
  if (!y || !raw || !ws || n <= 0 || !kern_known(kern) || !build_spec(d, spec, sp) || (sp.d > 0 && !Xt)) return HB_ERR_INVALID;
  w = carve_fit(ws, n, sp);
  if (ws_bytes / num_out < (int64_t)w.total) return HB_ERR_INVALID;
  if (sp.e <= 0) return HB_OK;
  if (!Xe) return HB_ERR_INVALID;
  std::vector<int32_t> m;
  fill_meta_host(spec, sp, m);
  for (int b = 0; b < num_out; ++b) {
    FitWs wb = carve_fit(slice(ws, (int64_t)w.total, b), n, sp);
    HB_CUDA(cudaMemcpyAsync(wb.meta, m.data(), m.size() * sizeof(int32_t), cudaMemcpyHostToDevice, st));
    HB_CUDA(cudaMemcpyAsync(wb.Xe, Xe, (size_t)n * sp.e * sizeof(int32_t), cudaMemcpyDeviceToDevice, st));
  }
  HB_CUDA(cudaStreamSynchronize(st));   // `m` is pageable host memory and dies with this frame
  bind_meta(sp, w.meta, w.Xe);
  return HB_OK;
}

// prediction state at `raw` in a carved and bound workspace: Gram + Cholesky through the jitter ladder (gp.py:140-157),
// L^-1 with one Newton refinement, its fp16 split, alpha / log-det, the scaled features.  Built ONCE per fit, so it stays on
// the FP32 SIMT pipe (round-to-nearest accumulation); the 3xTF32 tensor path (the tensor cores' fp32 accumulation is not
// RN) serves the gradient epochs only.  HB_ERR_NOT_PD: the ladder gave up.
static int factorize(const float *Xt, const float *y, int64_t n, const ModelSpec &sp, const float *raw, int kern,
                     const float *noise_diag, float noise_lb, FitWs &w, HostStatus *hs, float *jitter_used, cudaStream_t st) {
  const int64_t np = round_up(n, TILE);
  int s = launch_transform_hypers(raw, sp, noise_lb, w.hyp, st);
  if (s != HB_OK) return s;
  float jitter = 0.0f;
  s = jitter_ladder(
      [&](float j, int32_t &info) -> int {   // info: hs->info (pinned)
        const int r = factor_once(Xt, n, np, sp, raw, kern, noise_diag, j, w, st, nullptr);
        if (r != HB_OK) return r;
        HB_CUDA(cudaMemcpyAsync(&info, w.info, sizeof(int32_t), cudaMemcpyDeviceToHost, st));
        HB_CUDA(cudaStreamSynchronize(st));
        return HB_OK;
      },
      jitter, hs->info);
  if (jitter_used) *jitter_used = jitter;
  if (s != HB_OK) return s;
  s = launch_tri_inverse(w.L, np, w.Linv, w.tmp, st);
  if (s != HB_OK) return s;
  s = launch_linv_refine(w.L, w.Linv, np, w.tmp, w.tc.T_hi, st);   // Newton step, fp64 residual (scratch: tmp, T_hi)
  if (s != HB_OK) return s;
  // operands of the posterior's tensor-core contraction: two-level fp16 split (h0 in the Linv_hi buffer, h1 in the first
  // half of the Linv_lo buffer, the power-of-two scale right after it)
  s = launch_split_h16(w.Linv, np * np, reinterpret_cast<__half *>(w.Linv_hi), reinterpret_cast<__half *>(w.Linv_lo),
                       w.Linv_lo + np * np / 2, st);
  if (s != HB_OK) return s;
  s = launch_solve_logdet(w.L, w.Linv, y, n, np, w.hyp, w.alpha, w.scal, w.solvews, st);
  if (s != HB_OK) return s;
  return launch_scale_zt(Xt, np, sp, w.hyp, w.Zt, w.dZa, w.dZb, st);   // (embedding rows of Zt: filled by factor_once's gather)
}

}  // namespace hb

using namespace hb;

extern "C" {

int32_t hb_version(void) { return 200; }
const char *hb_last_error(void) { return g_err; }
int64_t hb_padded_n(int64_t n) { return round_up(n, TILE); }
int32_t hb_vnorm_operand_kind(void) { return 0; }

int64_t hb_launch_count(int32_t reset) {
  long long v = g_launches.load();
  if (reset) g_launches = 0;
  return (int64_t)v;
}

int32_t hb_profile_enable(int32_t on) {
  g_prof.on = on != 0;
  g_prof.used = 0;
  return HB_OK;
}

int32_t hb_profile_collect(double *total_ms, int32_t *n_launches) {
  if (!total_ms || !n_launches) return HB_ERR_INVALID;
  double tot = 0.0;
  for (size_t i = 0; i < g_prof.used; ++i) {
    float ms = 0.f;
    HB_CUDA(cudaEventSynchronize(g_prof.b[i]));
    HB_CUDA(cudaEventElapsedTime(&ms, g_prof.a[i], g_prof.b[i]));
    tot += ms;
  }
  *total_ms = tot;
  *n_launches = (int32_t)g_prof.used;
  g_prof.used = 0;
  return HB_OK;
}

int32_t hb_guard_stats(uint64_t *rows_flagged, int32_t reset) {
  if (!rows_flagged) return HB_ERR_INVALID;
  unsigned long long v[2] = {0, 0};
  const int s = guard_stats(v, reset);
  rows_flagged[0] = v[0];
  rows_flagged[1] = v[1];
  return s;
}

int64_t hb_num_params(int64_t d, const hb_model_spec_t *spec) {
  ModelSpec sp;
  if (!build_spec(d, spec, sp)) return -1;
  return sp.P();
}
int64_t hb_fit_workspace_bytes_ex(int64_t n, int64_t d, const hb_model_spec_t *spec) {
  ModelSpec sp;
  if (n <= 0 || !build_spec(d, spec, sp)) return -1;
  return (int64_t)carve_fit(nullptr, n, sp).total;
}
int64_t hb_fit_workspace_bytes(int64_t n, int64_t d) { return d <= 0 ? -1 : hb_fit_workspace_bytes_ex(n, d, nullptr); }
int64_t hb_posterior_workspace_bytes(int64_t n, int64_t d, int64_t m_chunk) {
  if (n <= 0 || d < 0 || m_chunk <= 0) return -1;
  return (int64_t)carve_posterior_ws(nullptr, round_up(n, TILE), m_chunk).bytes;
}
int64_t hb_pareto_workspace_bytes(int64_t m) {
  if (m <= 0) return -1;
  return (int64_t)pareto_ws_bytes(m);
}

int32_t hb_transform_hypers(const float *raw, int64_t d, float noise_lb, float *hyp, void *stream) {
  ModelSpec sp;
  if (!raw || !hyp || d <= 0 || !build_spec(d, nullptr, sp)) return HB_ERR_INVALID;
  return launch_transform_hypers(raw, sp, noise_lb, hyp, (cudaStream_t)stream);
}

int32_t hb_median_pdist(const float *Xt, int64_t n, int64_t d, const int32_t *idx, int64_t k, float clamp_min,
                        float *out, void *stream) {
  if (!Xt || !out || n <= 0) return HB_ERR_INVALID;
  return launch_median_pdist(Xt, round_up(n, TILE), d, idx, k, clamp_min, out, (cudaStream_t)stream);
}

int32_t hb_gram(const float *Xt, int64_t n, int64_t d, const float *hyp, int32_t kern, const float *noise_diag,
                float jitter, float *K, void *stream) {
  ModelSpec sp;
  if (!Xt || !hyp || !K || d <= 0 || !build_spec(d, nullptr, sp)) return HB_ERR_INVALID;
  return launch_gram(Xt, nullptr, n, round_up(n, TILE), sp, hyp, kern, noise_diag, jitter, K, (cudaStream_t)stream);
}

int32_t hb_cholesky(float *A, int64_t np, float *ws, int32_t *info, void *stream) {
  if (!A || !ws || !info) return HB_ERR_INVALID;
  return launch_cholesky(A, np, ws, info, (cudaStream_t)stream);
}

int32_t hb_tri_inverse(const float *L, int64_t np, float *Linv, float *tmp, void *stream) {
  if (!L || !Linv || !tmp) return HB_ERR_INVALID;
  return launch_tri_inverse(L, np, Linv, tmp, (cudaStream_t)stream);
}

int32_t hb_kinv(const float *Linv, int64_t np, float *Kinv, void *stream) {
  if (!Linv || !Kinv) return HB_ERR_INVALID;
  return launch_kinv(Linv, np, Kinv, (cudaStream_t)stream);
}

// the tensor-core twins: the same launchers the fit epoch runs (enqueue_mll with tc != nullptr), one stage at a time
static bool tc_np_ok(int64_t np) { return np > 0 && np % TILE == 0; }
static bool open_tc_ws(void *tc_ws, int64_t tc_ws_bytes, int64_t np, TcBuffers &tc) {
  if (!tc_ws || !tc_np_ok(np)) return false;
  size_t need = 0;
  tc = carve_tc_ws(tc_ws, np, need);
  return tc_ws_bytes >= 0 && (uint64_t)tc_ws_bytes >= need;
}

int64_t hb_tc_workspace_bytes(int64_t np) {
  if (!tc_np_ok(np)) return -1;
  size_t bytes = 0;
  carve_tc_ws(nullptr, np, bytes);
  return (int64_t)bytes;
}

int32_t hb_cholesky_tc(float *A, int64_t np, float *ws, int32_t *info, void *tc_ws, int64_t tc_ws_bytes, void *stream) {
  TcBuffers tc;
  if (!A || !ws || !info || !open_tc_ws(tc_ws, tc_ws_bytes, np, tc)) return HB_ERR_INVALID;
  return launch_cholesky(A, np, ws, info, (cudaStream_t)stream, &tc);
}

int32_t hb_tri_inverse_tc(const float *L, int64_t np, float *Linv, void *tc_ws, int64_t tc_ws_bytes, void *stream) {
  TcBuffers tc;
  if (!L || !Linv || !open_tc_ws(tc_ws, tc_ws_bytes, np, tc)) return HB_ERR_INVALID;
  return launch_tri_inverse_tc(L, np, Linv, tc, true, (cudaStream_t)stream, Batch());
}

int32_t hb_kinv_tc(int64_t np, float *Kinv, void *tc_ws, int64_t tc_ws_bytes, void *stream) {
  TcBuffers tc;
  if (!Kinv || !open_tc_ws(tc_ws, tc_ws_bytes, np, tc)) return HB_ERR_INVALID;
  return launch_kinv_tc(np, Kinv, tc, (cudaStream_t)stream, Batch());
}

int32_t hb_solve_logdet(const float *L, const float *Linv, const float *y, int64_t n, int64_t np, const float *hyp,
                        float *alpha, double *scal, void *ws, void *stream) {
  if (!L || !Linv || !y || !hyp || !alpha || !scal || !ws) return HB_ERR_INVALID;
  return launch_solve_logdet(L, Linv, y, n, np, hyp, alpha, scal, ws, (cudaStream_t)stream);
}

int32_t hb_mll_grad(const float *Xt, int64_t n, int64_t d, const float *raw, const float *hyp, int32_t kern,
                    const float *Kinv, const float *alpha, const double *scal, float noise_guess, float *grad,
                    float *loss, void *ws, void *stream) {
  ModelSpec sp;
  if (!Xt || !raw || !hyp || !Kinv || !alpha || !scal || !grad || !loss || !ws || d <= 0 || !build_spec(d, nullptr, sp))
    return HB_ERR_INVALID;
  return launch_mll_grad(Xt, nullptr, n, round_up(n, TILE), sp, raw, hyp, kern, Kinv, alpha, scal, noise_guess, grad, loss, ws,
                         (cudaStream_t)stream);
}

int32_t hb_psgld_step(float *raw, const float *grad, float *square_avg, int64_t p, float lr, float rms_alpha,
                      float rms_eps, float factor, const float *xi, void *stream) {
  if (!raw || !grad || !square_avg) return HB_ERR_INVALID;
  return launch_psgld(raw, grad, square_avg, p, lr, rms_alpha, rms_eps, factor, xi, (cudaStream_t)stream);
}

int32_t hb_fit_state_ex(void *ws, int64_t n, int64_t d, const hb_model_spec_t *spec, hb_fit_state_t *out) {
  ModelSpec sp;
  if (!ws || !out || n <= 0 || !build_spec(d, spec, sp)) return HB_ERR_INVALID;
  FitWs w = carve_fit(ws, n, sp);
  out->hyp = w.hyp;
  out->L = w.L;
  out->Linv = w.Linv;
  out->alpha = w.alpha;
  out->Zt = w.Zt;
  out->scal = w.scal;
  out->Linv_hi = w.Linv_hi;
  out->Linv_lo = w.Linv_lo;
  out->tab_s = w.tab_s;
  out->emb_meta = w.meta;
  out->grad = w.grad;
  out->loss = w.loss;
  return HB_OK;
}
int32_t hb_fit_state(void *ws, int64_t n, int64_t d, hb_fit_state_t *out) {
  return d <= 0 ? HB_ERR_INVALID : hb_fit_state_ex(ws, n, d, nullptr, out);
}

int32_t hb_factorize_ex(const float *Xt, const int32_t *Xe, const float *y, int64_t n, int64_t d, const hb_model_spec_t *spec,
                        const float *raw, int32_t kern, const float *noise_diag, float noise_lb, float *jitter_used, void *ws,
                        int64_t ws_bytes, void *stream) {
  ModelSpec sp;
  FitWs w;
  int s = open_fit_ws(Xt, Xe, y, n, d, spec, raw, kern, ws, ws_bytes, 1, (cudaStream_t)stream, sp, w);
  if (s != HB_OK) return s;
  FitHost *fh = nullptr;
  s = fit_host(fh);
  if (s != HB_OK) return s;
  return factorize(Xt, y, n, sp, raw, kern, noise_diag, noise_lb, w, fh->status, jitter_used, (cudaStream_t)stream);
}
int32_t hb_factorize(const float *Xt, const float *y, int64_t n, int64_t d, const float *raw, int32_t kern,
                     const float *noise_diag, float noise_lb, float *jitter_used, void *ws, int64_t ws_bytes,
                     void *stream) {
  if (d <= 0) return HB_ERR_INVALID;
  return hb_factorize_ex(Xt, nullptr, y, n, d, nullptr, raw, kern, noise_diag, noise_lb, jitter_used, ws, ws_bytes, stream);
}

// one MLL forward + backward at `raw` (SURVEY 8b `hb_mll_fwd_bwd`) with FP32 SIMT GEMM stages.  Results stay on the device
// (fit-state grad / loss, `info`).
int32_t hb_mll_fwd_bwd(const float *Xt, const int32_t *Xe, const float *y, int64_t n, int64_t d, const hb_model_spec_t *spec,
                       const float *raw, int32_t kern, const float *noise_diag, float noise_lb, float noise_guess, float jitter,
                       float *grad, float *loss, int32_t *info, void *ws, int64_t ws_bytes, void *stream) {
  if (!grad || !loss || !info) return HB_ERR_INVALID;
  cudaStream_t st = (cudaStream_t)stream;
  ModelSpec sp;
  FitWs w;
  int s = open_fit_ws(Xt, Xe, y, n, d, spec, raw, kern, ws, ws_bytes, 1, st, sp, w);
  if (s != HB_OK) return s;
  s = enqueue_mll(Xt, y, n, round_up(n, TILE), sp, raw, kern, noise_diag, noise_lb, noise_guess, jitter, w, st, nullptr, false);
  if (s != HB_OK) return s;
  HB_CUDA(cudaMemcpyAsync(grad, w.grad, sp.P() * sizeof(float), cudaMemcpyDeviceToDevice, st));
  HB_CUDA(cudaMemcpyAsync(loss, w.loss, sizeof(float), cudaMemcpyDeviceToDevice, st));
  HB_CUDA(cudaMemcpyAsync(info, w.info, sizeof(int32_t), cudaMemcpyDeviceToDevice, st));
  return HB_OK;
}

int64_t hb_fit_multi_workspace_bytes(int64_t n, int64_t d, const hb_model_spec_t *spec, int64_t num_out) {
  if (num_out < 1 || num_out > HB_MAX_OUTPUTS) return -1;
  const int64_t one = hb_fit_workspace_bytes_ex(n, d, spec);
  return one < 0 ? -1 : one * num_out;
}

int32_t hb_fit_multi_ex(const float *Xt, const int32_t *Xe, const float *Y, int64_t n, int64_t d, const hb_model_spec_t *spec,
                        int64_t num_out, float *raw, int32_t kern, const float *noise_diag, float noise_lb, float noise_guess,
                        float lr, int32_t num_epochs, const float *langevin, float *losses, int32_t *status, void *ws,
                        int64_t ws_bytes, void *stream) {
  if (!status || num_epochs < 0 || num_out < 1 || num_out > HB_MAX_OUTPUTS) return HB_ERR_INVALID;
  cudaStream_t st = (cudaStream_t)stream;
  ModelSpec sp;
  FitWs w;                                  // output 0; output b's workspace starts b * stride bytes later
  int s = open_fit_ws(Xt, Xe, Y, n, d, spec, raw, kern, ws, ws_bytes, num_out, st, sp, w);
  if (s != HB_OK) return s;
  FitHost *fh = nullptr;
  s = fit_host(fh);
  if (s != HB_OK) return s;
  HostStatus *hs = fh->status;
  const int B = (int)num_out;
  const int64_t stride = (int64_t)w.total;
  const Batch all{B, stride};
  const int64_t np = round_up(n, TILE);
  const int64_t P = sp.P();
  HB_CUDA(memset_slices(w.sq, 0, P * sizeof(float), all, st));
  HB_CUDA(memset_slices(w.info, 0, 4 * sizeof(int32_t), all, st));   // status, epoch counter, replay slot
  bool zeroed = false;                           // triangular complements of Linv / U zero-filled once per fit
  const int pretrain = num_epochs / 10;          // gp.py:99 pretrain_step = num_epochs // 10
  const float factor = 1.0f / (float)n;          // gp.py:99 factor = 1 / y.shape[0]

  // one epoch of outputs [b0, b0 + bt.nout) = MLL forward + backward on the tensor cores -> guarded pSGLD step
  auto enqueue_epoch = [&](float jitter, cudaStream_t s_, int b0, const Batch &bt) -> int {
    FitWs wb = carve_fit(slice(ws, stride, b0), n, sp);
    const int s = enqueue_mll(Xt, Y + b0 * n, n, np, sp, raw + b0 * P, kern, noise_diag, noise_lb, noise_guess, jitter, wb, s_,
                              &wb.tc, !zeroed, bt);
    zeroed = true;
    if (s != HB_OK) return s;
    psgld_guarded_kernel<<<bt.nout, 256, 0, s_>>>(raw + b0 * P, wb.grad, wb.sq, (int)P, lr, 0.99f, 1e-8f, factor,
                                                 langevin ? langevin + (int64_t)b0 * num_epochs * P : nullptr, pretrain,
                                                 num_epochs, wb.info, wb.loss, wb.status, wb.hyp, sp.H(),
                                                 sp.warp == 2 ? sp.i_wa() : 0, sp.warp == 2 ? sp.i_wa() + sp.n_w() : 0, stride);
    count_launches(1);
    HB_LAUNCH_CHECK("psgld_guarded");
    return HB_OK;
  };
  // per-output host state: next epoch, and whether the output stopped on a hopeless epoch (from which epoch)
  std::vector<int> ep(B, 0), hopeless_from(B, -1);
  auto active = [&](int b) { return hopeless_from[b] < 0 && ep[b] < num_epochs; };
  auto loss_out = [&](int b, int e, float v) {
    if (losses) losses[(int64_t)b * num_epochs + e] = v;
  };
  // epoch ep[b] of output b through the jitter ladder on its own slice, one host synchronisation per attempt; the other
  // outputs are not touched
  const Batch one{1, stride};
  auto slow_epoch = [&](int b) -> int {
    FitWs wb = carve_fit(slice(ws, stride, b), n, sp);
    float jitter = 0.0f;
    int32_t info = 0;
    const int s = jitter_ladder(
        [&](float j, int32_t &inf) -> int {
          HB_CUDA(cudaMemsetAsync(wb.info + 2, 0, sizeof(int32_t), st));   // replay slot 0
          const int r = enqueue_epoch(j, st, b, one);
          if (r != HB_OK) return r;
          HB_CUDA(cudaMemcpyAsync(hs->batch[b], wb.status, 2 * sizeof(float), cudaMemcpyDeviceToHost, st));
          HB_CUDA(cudaStreamSynchronize(st));
          memcpy(&inf, &hs->batch[b][0], sizeof(inf));
          return HB_OK;
        },
        jitter, info);
    if (s != HB_OK && s != HB_ERR_NOT_PD) return s;
    if (s == HB_OK && info == -1) {   // hopeless (see psgld_guarded_kernel): this and every later epoch is given up
      hopeless_from[b] = ep[b];
      return HB_OK;
    }
    // trained, or "jitter is too large, give up fitting GP": epoch skipped, gp.py:121-122
    loss_out(b, ep[b]++, s == HB_OK ? hs->batch[b][1] : INFINITY);
    if (s == HB_OK) return HB_OK;
    hs->set_epoch = ep[b];   // the device counter only advances on success
    HB_CUDA(cudaMemcpyAsync(wb.info + 1, &hs->set_epoch, sizeof(int32_t), cudaMemcpyHostToDevice, st));
    HB_CUDA(cudaStreamSynchronize(st));
    return HB_OK;
  };
  // R epochs of every active output at jitter 0 -- replays of the captured graph, or enqueued directly when there is none
  // -- then one status read-back.  A failed factorisation leaves that output's hypers, RMS state and device epoch counter
  // untouched (the pSGLD kernel is guarded), so the rest of the batch fails the same way for it; the host then runs that
  // epoch through the output's ladder.  The other outputs are unaffected: each has its own counter and replay slots.
  cudaGraphExec_t exec = nullptr;
  long long launches_per_epoch = 0;
  auto run_epochs = [&](int R, int &failed) -> int {
    HB_CUDA(memset_slices(w.info + 2, 0, sizeof(int32_t), all, st));
    for (int r = 0; r < R; ++r) {
      if (exec) HB_CUDA(cudaGraphLaunch(exec, st));
      else if (const int s = enqueue_epoch(0.0f, st, 0, all); s != HB_OK) return s;
    }
    if (exec) count_launches(launches_per_epoch * R);
    HB_CUDA(cudaMemcpy2DAsync(hs->batch, sizeof(hs->batch[0]), w.status, (size_t)stride, (size_t)R * 2 * sizeof(float), B,
                              cudaMemcpyDeviceToHost, st));
    HB_CUDA(cudaStreamSynchronize(st));
    failed = 0;
    for (int b = 0; b < B; ++b) {
      if (!active(b)) continue;
      const int need = R < num_epochs - ep[b] ? R : num_epochs - ep[b];
      int done = 0;
      for (; done < need; ++done) {
        int32_t info;
        memcpy(&info, &hs->batch[b][2 * done], sizeof(info));
        if (info != 0) break;
        loss_out(b, ep[b] + done, hs->batch[b][2 * done + 1]);
      }
      ep[b] += done;
      if (done < need) {
        failed = 1;
        const int s = slow_epoch(b);
        if (s != HB_OK) return s;
      }
    }
    return HB_OK;
  };

  int failed = 0;
  if (num_epochs > 0) {   // enqueued directly: the first epoch also builds every lazily created table / attribute
    s = run_epochs(1, failed);
    if (s != HB_OK) return s;
  }
  if (num_epochs - 1 >= 4) {   // capture ONE epoch of all outputs into a CUDA graph for the remaining epochs
    HB_CUDA(cudaStreamSynchronize(st));
    cudaGraph_t graph = nullptr;
    const long long before = g_launches.load();
    if (cudaStreamBeginCapture(fh->capture, cudaStreamCaptureModeThreadLocal) == cudaSuccess) {
      const int r = enqueue_epoch(0.0f, fh->capture, 0, all);
      const cudaError_t e = cudaStreamEndCapture(fh->capture, &graph);
      if (r == HB_OK && e == cudaSuccess && graph && cudaGraphInstantiate(&exec, graph, 0) == cudaSuccess) {
        launches_per_epoch = g_launches.load() - before;
      } else {
        exec = nullptr;
      }
      if (graph) cudaGraphDestroy(graph);
    }
    g_launches = before;       // nothing was launched by the capture itself
    (void)cudaGetLastError();  // a failed capture leaves the direct enqueues to run the epochs
  }
  int batch = FIT_BATCH;
  for (;;) {
    int left = 0;   // epochs the furthest-behind active output still needs
    for (int b = 0; b < B; ++b)
      if (active(b) && num_epochs - ep[b] > left) left = num_epochs - ep[b];
    if (left == 0) break;
    int R = batch < FIT_BATCH ? batch : FIT_BATCH;   // ramps 1, 2, 4, .. after a failure: a failing epoch wastes the rest
    if (R > left) R = left;                         // of its batch, and failures come in runs (gp.py:117-126 territory)
    s = run_epochs(R, failed);
    if (s != HB_OK) break;
    batch = failed ? 1 : (2 * batch > FIT_BATCH ? FIT_BATCH : 2 * batch);
  }
  if (exec) cudaGraphExecDestroy(exec);
  if (s != HB_OK) return s;
  // final prediction state of every output, once per fit
  for (int b = 0; b < B; ++b) {
    if (hopeless_from[b] >= 0)   // "jitter is too large, give up fitting GP" for that and every remaining epoch
      for (int e = hopeless_from[b]; e < num_epochs; ++e) loss_out(b, e, INFINITY);
    FitWs wb = carve_fit(slice(ws, stride, b), n, sp);
    s = factorize(Xt, Y + b * n, n, sp, raw + b * P, kern, noise_diag, noise_lb, wb, hs, nullptr, st);
    if (s != HB_OK && s != HB_ERR_NOT_PD) return s;
    status[b] = s;
  }
  return HB_OK;
}

int32_t hb_fit_ex(const float *Xt, const int32_t *Xe, const float *y, int64_t n, int64_t d, const hb_model_spec_t *spec,
                  float *raw, int32_t kern, const float *noise_diag, float noise_lb, float noise_guess, float lr,
                  int32_t num_epochs, const float *langevin, float *losses, void *ws, int64_t ws_bytes, void *stream) {
  int32_t status = HB_OK;
  const int32_t s = hb_fit_multi_ex(Xt, Xe, y, n, d, spec, 1, raw, kern, noise_diag, noise_lb, noise_guess, lr, num_epochs,
                                    langevin, losses, &status, ws, ws_bytes, stream);
  return s != HB_OK ? s : status;
}
int32_t hb_fit(const float *Xt, const float *y, int64_t n, int64_t d, float *raw, int32_t kern,
               const float *noise_diag, float noise_lb, float noise_guess, float lr, int32_t num_epochs,
               const float *langevin, float *losses, void *ws, int64_t ws_bytes, void *stream) {
  if (d <= 0) return HB_ERR_INVALID;
  return hb_fit_ex(Xt, nullptr, y, n, d, nullptr, raw, kern, noise_diag, noise_lb, noise_guess, lr, num_epochs, langevin, losses,
                   ws, ws_bytes, stream);
}

// The fitted-model arguments that hb_posterior_mace_ex, hb_posterior_grad_ex, hb_sample_y and hb_sample_y_batch share,
// validated and bound into `gp`; false: the call is invalid.  Xs / Xe_s are the candidates, checked here because which of
// them a call needs follows from the same spec.
static bool open_fitted(const float *Xs, const int32_t *Xe_s, int64_t n, int64_t d, const hb_model_spec_t *spec,
                        const int32_t *emb_meta, const float *tab_s, const float *x_mul, const float *x_add, const float *Zt,
                        const float *alpha, const float *Linv, const float *hyp, int32_t kern, float y_mean, float y_std,
                        int32_t pred_likeli, Fitted &gp) {
  ModelSpec sp;
  if (!build_spec(d, spec, sp) || n <= 0 || !kern_known(kern)) return false;
  if ((sp.d > 0 && (!Xs || !x_mul || !x_add)) || !Zt || !alpha || !Linv || !hyp) return false;
  if (sp.e > 0 && (!Xe_s || !emb_meta || !tab_s)) return false;
  bind_meta(sp, emb_meta, nullptr);
  gp = Fitted{sp, n, round_up(n, TILE), kern, Zt, alpha, Linv, hyp, tab_s, x_mul, x_add, y_mean, y_std, pred_likeli};
  return true;
}

int32_t hb_posterior_mace_ex(const float *Xs, const int32_t *Xe_s, int64_t m, int64_t rng_offset, int64_t n, int64_t d,
                             const hb_model_spec_t *spec,
                             const int32_t *emb_meta, const float *tab_s, const float *x_mul, const float *x_add,
                             const float *Zt, const float *alpha, const float *Linv, const float *Linv_hi,
                             const float *Linv_lo, const float *hyp, int32_t kern, float y_mean, float y_std, int32_t pred_likeli,
                             float tau, float kappa, float eps, const float *xi1, const float *xi2, uint64_t seed, float *F,
                             float *mu, float *var, void *ws, int64_t ws_bytes, int64_t m_chunk, void *stream) {
  Fitted gp;
  if (!open_fitted(Xs, Xe_s, n, d, spec, emb_meta, tab_s, x_mul, x_add, Zt, alpha, Linv, hyp, kern, y_mean, y_std, pred_likeli, gp))
    return HB_ERR_INVALID;
  if (!ws || (!F && !mu && !var)) return HB_ERR_INVALID;
  if ((Linv_hi == nullptr) != (Linv_lo == nullptr)) return HB_ERR_INVALID;
  return launch_posterior_mace(gp, Xs, Xe_s, m, rng_offset, Linv_hi, Linv_lo, tau, kappa, eps, xi1, xi2, seed, F, mu, var, ws,
                               ws_bytes, m_chunk, (cudaStream_t)stream);
}
int32_t hb_posterior_mace(const float *Xs, int64_t m, int64_t n, int64_t d, const float *x_mul, const float *x_add,
                          const float *Zt, const float *alpha, const float *Linv, const float *Linv_hi,
                          const float *Linv_lo, const float *hyp, int32_t kern, float y_mean, float y_std, int32_t pred_likeli, float tau, float kappa, float eps,
                          const float *xi1, const float *xi2, uint64_t seed, float *F, float *mu, float *var,
                          void *ws, int64_t ws_bytes, int64_t m_chunk, void *stream) {
  if (d <= 0) return HB_ERR_INVALID;
  return hb_posterior_mace_ex(Xs, nullptr, m, 0, n, d, nullptr, nullptr, nullptr, x_mul, x_add, Zt, alpha, Linv, Linv_hi, Linv_lo, hyp,
                              kern, y_mean, y_std, pred_likeli, tau, kappa, eps, xi1, xi2, seed, F, mu, var, ws, ws_bytes, m_chunk,
                              stream);
}

int32_t hb_posterior_grad_ex(const float *Xs, const int32_t *Xe_s, int64_t m, int64_t n, int64_t d, const hb_model_spec_t *spec,
                             const int32_t *emb_meta, const float *tab_s, const float *x_mul, const float *x_add,
                             const float *Zt, const float *alpha, const float *Linv, const float *hyp, int32_t kern, float y_mean,
                             float y_std, int32_t pred_likeli, float *mu, float *var, float *dmu, float *dvar, void *ws,
                             int64_t ws_bytes, int64_t m_chunk, void *stream) {
  // post_grad_kernel differentiates through x_mul / l only: a warp is the caller's, in front of this call
  if ((spec && spec->warp != 0) || d <= 0) return HB_ERR_INVALID;
  Fitted gp;
  if (!open_fitted(Xs, Xe_s, n, d, spec, emb_meta, tab_s, x_mul, x_add, Zt, alpha, Linv, hyp, kern, y_mean, y_std, pred_likeli, gp))
    return HB_ERR_INVALID;
  if (!ws || !mu || !var || !dmu || !dvar) return HB_ERR_INVALID;
  return launch_posterior_grad(gp, Xs, Xe_s, m, mu, var, dmu, dvar, ws, ws_bytes, m_chunk, (cudaStream_t)stream);
}
int32_t hb_posterior_grad(const float *Xs, int64_t m, int64_t n, int64_t d, const float *x_mul, const float *x_add,
                          const float *Zt, const float *alpha, const float *Linv, const float *hyp, int32_t kern, float y_mean,
                          float y_std, int32_t pred_likeli, float *mu, float *var, float *dmu, float *dvar, void *ws,
                          int64_t ws_bytes, int64_t m_chunk, void *stream) {
  return hb_posterior_grad_ex(Xs, nullptr, m, n, d, nullptr, nullptr, nullptr, x_mul, x_add, Zt, alpha, Linv, hyp, kern, y_mean, y_std,
                              pred_likeli, mu, var, dmu, dvar, ws, ws_bytes, m_chunk, stream);
}

int64_t hb_sample_workspace_bytes(int64_t n, int64_t d, const hb_model_spec_t *spec, int64_t m) {
  ModelSpec sp;
  if (n <= 0 || m <= 0 || !build_spec(d, spec, sp)) return -1;
  return (int64_t)sample_ws_bytes(round_up(n, TILE), sp.dtot(), m);
}

int32_t hb_sample_y(const float *Xs, const int32_t *Xe_s, int64_t m, int64_t n, int64_t d, const hb_model_spec_t *spec,
                    const int32_t *emb_meta, const float *tab_s, const float *x_mul, const float *x_add, const float *Zt,
                    const float *alpha, const float *Linv, const float *hyp, const float *hyp_host, int32_t kern, float y_mean,
                    float y_std, int32_t pred_likeli, const float *z, int32_t n_samples, float *out, float *jitter_used, void *ws,
                    int64_t ws_bytes, void *stream) {
  Fitted gp;
  if (!open_fitted(Xs, Xe_s, n, d, spec, emb_meta, tab_s, x_mul, x_add, Zt, alpha, Linv, hyp, kern, y_mean, y_std, pred_likeli, gp))
    return HB_ERR_INVALID;
  if (!ws || !hyp_host || !z || !out) return HB_ERR_INVALID;
  return launch_sample_y(gp, Xs, Xe_s, m, hyp_host, z, n_samples, out, jitter_used, ws, ws_bytes, (cudaStream_t)stream);
}

int32_t hb_sample_y_batch(const float *Xs, const int32_t *Xe_s, int64_t m, int64_t n, int64_t d, const hb_model_spec_t *spec,
                          const int32_t *emb_meta, const float *tab_s, const float *x_mul, const float *x_add, const float *Zt,
                          const float *alpha, const float *Linv, const float *hyp, int32_t kern, float y_mean, float y_std,
                          int32_t pred_likeli, const float *z, uint64_t seed, uint64_t counter, float *f, float *jitter,
                          int32_t *status, void *ws, int64_t ws_bytes, void *stream) {
  Fitted gp;
  if (!open_fitted(Xs, Xe_s, n, d, spec, emb_meta, tab_s, x_mul, x_add, Zt, alpha, Linv, hyp, kern, y_mean, y_std, pred_likeli, gp))
    return HB_ERR_INVALID;
  if (!ws || !f || !jitter || !status) return HB_ERR_INVALID;
  return launch_sample_y_batch(gp, Xs, Xe_s, m, z, seed, counter, f, jitter, status, ws, ws_bytes, (cudaStream_t)stream);
}

int32_t hb_mace_epilogue(const float *mu, const float *var, int64_t m, float noise_var, float tau, float kappa,
                         float eps, const float *xi1, const float *xi2, uint64_t seed, float *F, void *stream) {
  if (!mu || !var || !F) return HB_ERR_INVALID;
  return launch_mace_only(mu, var, m, noise_var, tau, kappa, eps, xi1, xi2, seed, F, (cudaStream_t)stream);
}

int32_t hb_acq1_epilogue(const float *mu, const float *var, int64_t m, int32_t mode, float kappa, float eta, float *f,
                         void *stream) {
  if (!mu || !var || !f) return HB_ERR_INVALID;
  return launch_acq1(mu, var, m, mode, kappa, eta, f, (cudaStream_t)stream);
}

int32_t hb_general_acq_epilogue(const float *mu, const float *var, int64_t m, int64_t num_obj, int64_t num_constr, float kappa,
                                float c_kappa, const float *noise_sd, const float *xi, uint64_t seed, uint64_t counter, float *Fo,
                                float *Fc, float *cv, void *stream) {
  if (!mu || !var || !Fo) return HB_ERR_INVALID;
  return launch_general_acq(mu, var, m, num_obj, num_constr, kappa, c_kappa, noise_sd, xi, seed, counter, Fo, Fc, cv,
                            (cudaStream_t)stream);
}

int32_t hb_mo_lcb_epilogue(const float *mu, const float *var, int64_t m, float noise_sd, float best_y, float kappa,
                           const float *xi, uint64_t seed, uint64_t counter, float *F, float *G, void *stream) {
  if (!mu || !var || !F || !G) return HB_ERR_INVALID;
  return launch_mo_lcb(mu, var, m, noise_sd, best_y, kappa, xi, seed, counter, F, G, (cudaStream_t)stream);
}

int32_t hb_pareto_front3(const float *F, int64_t m, int32_t *idx_out, int32_t *count, void *ws, int64_t ws_bytes,
                         void *stream) {
  if (!F || !idx_out || !count || !ws) return HB_ERR_INVALID;
  return launch_pareto_k(F, m, 3, idx_out, count, ws, ws_bytes, (cudaStream_t)stream);
}

int32_t hb_pareto_front_k(const float *F, int64_t m, int64_t num_obj, int32_t *idx_out, int32_t *count, void *ws, int64_t ws_bytes,
                          void *stream) {
  if (!F || !idx_out || !count || !ws || num_obj < 1 || num_obj > HB_MAX_OBJ) return HB_ERR_INVALID;
  return launch_pareto_k(F, m, num_obj, idx_out, count, ws, ws_bytes, (cudaStream_t)stream);
}

int64_t hb_front_merge_workspace_bytes(int64_t world, int64_t capacity) {
  if (world <= 0 || capacity <= 0) return -1;
  return (int64_t)front_merge_ws_bytes(world, capacity);
}

int32_t hb_front_pack(const float *F, const float *mu, const float *var, const int32_t *idx, const int32_t *count,
                      int64_t row_offset, int64_t capacity, float *out, void *stream) {
  if (!F || !idx || !count || !out) return HB_ERR_INVALID;
  return launch_front_pack(F, mu, var, idx, count, row_offset, capacity, out, (cudaStream_t)stream);
}

int32_t hb_front_merge(const float *all_buf, int64_t world, int64_t capacity, float *out, void *ws, int64_t ws_bytes,
                       void *stream) {
  if (!all_buf || !out || !ws) return HB_ERR_INVALID;
  return launch_front_merge(all_buf, world, capacity, out, ws, ws_bytes, (cudaStream_t)stream);
}

int32_t hb_nsga2_init(float *X, int64_t pop, int64_t D, int64_t d, const int32_t *kind, const float *lb, const float *ub,
                      const float *fixed, const float *init, int64_t n_init, uint64_t seed, float *Xc, int32_t *Xe, void *stream) {
  if (!X || !kind || !lb || !ub || !fixed || (n_init > 0 && !init) || (d > 0 && !Xc) || (D > d && !Xe)) return HB_ERR_INVALID;
  return launch_nsga_init(X, pop, D, d, kind, lb, ub, fixed, init, n_init, seed, Xc, Xe, (cudaStream_t)stream);
}

int32_t hb_nsga2_mate(const float *X, int64_t pop, int64_t D, int64_t d, const int32_t *kind, const float *lb, const float *ub,
                      const float *fixed, uint64_t seed, int32_t generation, float *C, float *Cc, int32_t *Ce, void *stream) {
  if (!X || !kind || !lb || !ub || !fixed || !C || (d > 0 && !Cc) || (D > d && !Ce)) return HB_ERR_INVALID;
  return launch_nsga_mate(X, pop, D, d, kind, lb, ub, fixed, seed, generation, C, Cc, Ce, (cudaStream_t)stream);
}

int32_t hb_nsga2_survive(const float *X, const float *F, const float *C, const float *FC, int64_t pop, int64_t D, int64_t d,
                         float *X_next, float *F_next, float *Xc_next, int32_t *Xe_next, void *stream) {
  if (!X || !F || !C || !FC || !X_next || !F_next || (d > 0 && !Xc_next) || (D > d && !Xe_next)) return HB_ERR_INVALID;
  if (pop > 256) return HB_ERR_INVALID;   // the workspace-free entry keeps the single-CTA limit
  return launch_nsga_survive(X, F, nullptr, C, FC, nullptr, pop, D, d, 3, X_next, F_next, nullptr, Xc_next, Xe_next, nullptr, 0,
                             (cudaStream_t)stream);
}

int64_t hb_nsga2_workspace_bytes(int64_t pop, int64_t D) { return nsga_survive_ws_query(pop, D, 3); }

int64_t hb_nsga2_workspace_bytes_k(int64_t pop, int64_t D, int64_t num_obj) { return nsga_survive_ws_query(pop, D, num_obj); }

int32_t hb_nsga2_survive_ex(const float *X, const float *F, const float *C, const float *FC, int64_t pop, int64_t D,
                            int64_t d, float *X_next, float *F_next, float *Xc_next, int32_t *Xe_next, void *ws,
                            int64_t ws_bytes, void *stream) {
  if (!X || !F || !C || !FC || !X_next || !F_next || (d > 0 && !Xc_next) || (D > d && !Xe_next)) return HB_ERR_INVALID;
  return launch_nsga_survive(X, F, nullptr, C, FC, nullptr, pop, D, d, 3, X_next, F_next, nullptr, Xc_next, Xe_next, ws, ws_bytes,
                             (cudaStream_t)stream);
}

int32_t hb_nsga2_survive_cv(const float *X, const float *F, const float *G, const float *C, const float *FC, const float *GC,
                            int64_t pop, int64_t D, int64_t d, float *X_next, float *F_next, float *G_next, float *Xc_next,
                            int32_t *Xe_next, void *ws, int64_t ws_bytes, void *stream) {
  if (!X || !F || !G || !C || !FC || !GC || !X_next || !F_next || !G_next || (d > 0 && !Xc_next) || (D > d && !Xe_next))
    return HB_ERR_INVALID;
  return launch_nsga_survive(X, F, G, C, FC, GC, pop, D, d, 3, X_next, F_next, G_next, Xc_next, Xe_next, ws, ws_bytes,
                             (cudaStream_t)stream);
}

int32_t hb_nsga2_survive_k(const float *X, const float *F, const float *G, const float *C, const float *FC, const float *GC,
                           int64_t pop, int64_t D, int64_t d, int64_t num_obj, float *X_next, float *F_next, float *G_next,
                           float *Xc_next, int32_t *Xe_next, void *ws, int64_t ws_bytes, void *stream) {
  if (!X || !F || !C || !FC || !X_next || !F_next || (d > 0 && !Xc_next) || (D > d && !Xe_next)) return HB_ERR_INVALID;
  if (!G != !GC || !G != !G_next) return HB_ERR_INVALID;
  return launch_nsga_survive(X, F, G, C, FC, GC, pop, D, d, num_obj, X_next, F_next, G_next, Xc_next, Xe_next, ws, ws_bytes,
                             (cudaStream_t)stream);
}

int32_t hb_ga_survive(const float *X, const float *F, const float *C, const float *FC, int64_t pop, int64_t D, int64_t d,
                      float *X_next, float *F_next, float *Xc_next, int32_t *Xe_next, void *ws, int64_t ws_bytes, void *stream) {
  if (!X || !F || !C || !FC || !X_next || !F_next || (d > 0 && !Xc_next) || (D > d && !Xe_next)) return HB_ERR_INVALID;
  return launch_ga_survive(X, F, nullptr, C, FC, nullptr, pop, D, d, X_next, F_next, nullptr, Xc_next, Xe_next, ws, ws_bytes,
                           (cudaStream_t)stream);
}

int32_t hb_ga_survive_cv(const float *X, const float *F, const float *G, const float *C, const float *FC, const float *GC, int64_t pop,
                         int64_t D, int64_t d, float *X_next, float *F_next, float *G_next, float *Xc_next, int32_t *Xe_next, void *ws,
                         int64_t ws_bytes, void *stream) {
  if (!X || !F || !G || !C || !FC || !GC || !X_next || !F_next || !G_next || (d > 0 && !Xc_next) || (D > d && !Xe_next))
    return HB_ERR_INVALID;
  return launch_ga_survive(X, F, G, C, FC, GC, pop, D, d, X_next, F_next, G_next, Xc_next, Xe_next, ws, ws_bytes,
                           (cudaStream_t)stream);
}

int64_t hb_embed_violation_workspace_bytes(int64_t m, int64_t e, int64_t D) { return embed_violation_ws_query(m, e, D); }

int32_t hb_embed_violation(const float *Y, int64_t m, int64_t e, const float *B, int64_t D, float *G, void *ws, int64_t ws_bytes,
                           void *stream) {
  if (!Y || !B || !G || !ws) return HB_ERR_INVALID;
  return launch_embed_violation(Y, m, e, B, D, G, ws, ws_bytes, (cudaStream_t)stream);
}

// deep_ensemble.py:34-61 / BaseNet :183-221: P of one member
int64_t hb_de_num_params(const hb_de_spec_t *spec) { return de_num_params(spec, DeVariant{}); }

int64_t hb_de_fit_workspace_bytes(const hb_de_spec_t *spec, int64_t E) { return de_fit_ws_query(spec, DeVariant{}, E); }

// deep_ensemble.py:71-93 (the member loop) and fit_one :151-181
int32_t hb_de_fit(const float *Xc, const int32_t *Xe, const float *y, int64_t n, const hb_de_spec_t *spec, int64_t E,
                  float *params, double lr, float l1, int64_t batch_size, int64_t num_epochs, const int32_t *perm,
                  uint64_t seed, float *losses, void *ws, int64_t ws_bytes, void *stream) {
  return launch_de_fit(Xc, Xe, y, n, spec, DeVariant{}, E, params, lr, l1, batch_size, num_epochs, perm, nullptr, seed, losses,
                       ws, ws_bytes, (cudaStream_t)stream);
}

// deep_ensemble.py:95-106 (predict) and :108-116 (sample_f, member >= 0)
int32_t hb_de_predict(const float *Xs, const int32_t *Xe, int64_t m, const hb_de_spec_t *spec, int64_t E,
                      const float *params, const float *x_mul, const float *x_add, const float *y_mean, const float *y_std,
                      int32_t member, float *mu, float *var, void *stream) {
  return launch_de_predict(Xs, Xe, m, spec, DeVariant{}, E, params, x_mul, x_add, y_mean, y_std, member, nullptr, 0, 0, mu, var,
                           nullptr, nullptr, nullptr, 0, (cudaStream_t)stream);
}

// autograd of deep_ensemble.py:95-106 with respect to Xc (the support_grad contract, base_model.py / test_base_model.py:94-108)
int32_t hb_de_predict_grad(const float *Xs, const int32_t *Xe, int64_t m, const hb_de_spec_t *spec, int64_t E,
                           const float *params, const float *x_mul, const float *x_add, const float *y_mean,
                           const float *y_std, float *mu, float *var, float *dmu, float *dvar, void *stream) {
  if (!dmu || !dvar) return HB_ERR_INVALID;
  return launch_de_predict(Xs, Xe, m, spec, DeVariant{}, E, params, x_mul, x_add, y_mean, y_std, -1, nullptr, 0, 0, mu, var,
                           dmu, dvar, nullptr, 0, (cudaStream_t)stream);
}

// deep_ensemble.py:71-93 for the ensembles of a MultiTaskModel (model_factory.py:60-92), all in one launch
int32_t hb_de_fit_batch(const float *Xc, const int32_t *Xe, const float *y, const int64_t *off, int64_t B,
                        const hb_de_spec_t *spec, int64_t E, float *params, double lr, float l1, int64_t batch_size,
                        int64_t num_epochs, const uint64_t *seeds, float *losses, void *ws, int64_t ws_bytes, void *stream) {
  return launch_de_fit_batch(Xc, Xe, y, off, B, spec, E, params, lr, l1, batch_size, num_epochs, seeds, losses, ws, ws_bytes,
                             (cudaStream_t)stream);
}

// deep_ensemble.py:95-106 for B ensembles, and BaseModel.sample_y (base_model.py:78-84)
int32_t hb_de_predict_batch(const float *Xs, const int32_t *Xe, int64_t m, const hb_de_spec_t *spec, int64_t B, int64_t E,
                            const float *params, const float *x_mul, const float *x_add, const float *y_mean,
                            const float *y_std, float *mu, float *var, int64_t n_samples, const float *xi, uint64_t seed,
                            uint64_t counter, float *y_samp, void *stream) {
  return launch_de_predict_batch(Xs, Xe, m, spec, B, E, params, x_mul, x_add, y_mean, y_std, mu, var, n_samples, xi, seed,
                                 counter, y_samp, (cudaStream_t)stream);
}

// The gated and Gumbel layouts depend on neither the gate's kind and temperatures nor predict's temperature: the
// queries, and the Gumbel fit (which anneals its own temperature), pass any valid one
static const hb_fe_gate_t ANY_GATE = {HB_FE_STG, 1.0f, 1.0, 0.1, 0.99, 0.1f};
static DeVariant gumbel_variant(int64_t reduced_dim, float temperature = 1.0f) {
  return {DeVariant::GUMBEL, nullptr, reduced_dim, temperature};
}

// fe_deep_ensemble.py: FeNet / FeDeepEnsemble, P of one gated member
int64_t hb_fe_num_params(const hb_de_spec_t *spec) { return de_num_params(spec, {DeVariant::GATED, &ANY_GATE}); }

int64_t hb_fe_fit_workspace_bytes(const hb_de_spec_t *spec, int64_t E) {
  return de_fit_ws_query(spec, {DeVariant::GATED, &ANY_GATE}, E);
}

// deep_ensemble.py:71-93 (the member loop) and FeDeepEnsemble.fit_one (fe_deep_ensemble.py:46-75)
int32_t hb_fe_fit(const float *Xc, const int32_t *Xe, const float *y, int64_t n, const hb_de_spec_t *spec,
                  const hb_fe_gate_t *gate, int64_t E, float *params, double lr, float l1, int64_t batch_size,
                  int64_t num_epochs, const int32_t *perm, const float *draws, uint64_t seed, float *losses, void *ws,
                  int64_t ws_bytes, void *stream) {
  return launch_de_fit(Xc, Xe, y, n, spec, {DeVariant::GATED, gate}, E, params, lr, l1, batch_size, num_epochs, perm, draws,
                       seed, losses, ws, ws_bytes, (cudaStream_t)stream);
}

// deep_ensemble.py:95-116 over FeNet members (fe_deep_ensemble.py:29-35), the gate in eval mode
int32_t hb_fe_predict(const float *Xs, const int32_t *Xe, int64_t m, const hb_de_spec_t *spec, const hb_fe_gate_t *gate,
                      int64_t E, const float *params, const float *x_mul, const float *x_add, const float *y_mean,
                      const float *y_std, int32_t member, const float *draws, uint64_t seed, uint64_t counter, float *mu,
                      float *var, void *stream) {
  return launch_de_predict(Xs, Xe, m, spec, {DeVariant::GATED, gate}, E, params, x_mul, x_add, y_mean, y_std, member, draws,
                           seed, counter, mu, var, nullptr, nullptr, nullptr, 0, (cudaStream_t)stream);
}

// gumbel_linear.py: GumbelNet / GumbelDeepEnsemble, P of one member
int64_t hb_gumbel_num_params(const hb_de_spec_t *spec, int64_t reduced_dim) {
  return de_num_params(spec, gumbel_variant(reduced_dim));
}

int64_t hb_gumbel_fit_workspace_bytes(const hb_de_spec_t *spec, int64_t reduced_dim, int64_t E) {
  return de_fit_ws_query(spec, gumbel_variant(reduced_dim), E);
}

// deep_ensemble.py:71-93 (the member loop) and GumbelDeepEnsemble.fit_one (gumbel_linear.py:69-100)
int32_t hb_gumbel_fit(const float *Xc, const int32_t *Xe, const float *y, int64_t n, const hb_de_spec_t *spec,
                      int64_t reduced_dim, int64_t E, float *params, double lr, float l1, int64_t batch_size,
                      int64_t num_epochs, const int32_t *perm, const float *draws, uint64_t seed, float *losses, void *ws,
                      int64_t ws_bytes, void *stream) {
  return launch_de_fit(Xc, Xe, y, n, spec, gumbel_variant(reduced_dim), E, params, lr, l1, batch_size, num_epochs, perm, draws,
                       seed, losses, ws, ws_bytes, (cudaStream_t)stream);
}

// deep_ensemble.py:95-116 over GumbelNet members (gumbel_linear.py:58-61)
int32_t hb_gumbel_predict(const float *Xs, const int32_t *Xe, int64_t m, const hb_de_spec_t *spec, int64_t reduced_dim,
                          float temperature, int64_t E, const float *params, const float *x_mul, const float *x_add,
                          const float *y_mean, const float *y_std, int32_t member, const float *draws, uint64_t seed,
                          uint64_t counter, float *mu, float *var, void *ws, int64_t ws_bytes, void *stream) {
  return launch_de_predict(Xs, Xe, m, spec, gumbel_variant(reduced_dim, temperature), E, params, x_mul, x_add, y_mean, y_std,
                           member, draws, seed, counter, mu, var, nullptr, nullptr, ws, ws_bytes, (cudaStream_t)stream);
}

// rf.py:19-56: RF over sklearn's RandomForestRegressor (forest.cu)
int64_t hb_rf_fit_workspace_bytes(int64_t n, const hb_rf_spec_t *spec, int64_t B, int64_t T) {
  return rf_fit_ws_query(n, spec, B, T);
}

int64_t hb_rf_forest_bytes(const hb_rf_spec_t *spec, int64_t max_nodes, int64_t B, int64_t T) {
  return rf_forest_bytes(spec, max_nodes, B, T);
}

// rf.py:37-43 (fit)
int32_t hb_rf_fit(const float *Xc, const int32_t *Xe, const float *y, int64_t n, const hb_rf_spec_t *spec, int64_t B,
                  int64_t T, const int32_t *counts, uint64_t seed, void *forest, float *noise, void *ws, int64_t ws_bytes,
                  void *stream) {
  return launch_rf_fit(Xc, Xe, y, n, spec, B, T, counts, seed, forest, noise, ws, ws_bytes, (cudaStream_t)stream);
}

// rf.py:49-56 (predict) and BaseModel.sample_y (base_model.py:78-84)
int32_t hb_rf_predict(const float *Xc, const int32_t *Xe, int64_t m, const hb_rf_spec_t *spec, const void *forest,
                      int64_t B, int64_t T, const float *noise, float *mean, float *var, int64_t n_samples, uint64_t seed,
                      uint64_t counter, float *samples, void *stream) {
  return launch_rf_predict(Xc, Xe, m, spec, forest, B, T, noise, mean, var, n_samples, seed, counter, samples,
                           (cudaStream_t)stream);
}

// a forest from per-tree node arrays (sklearn's tree_.children_left / children_right / feature / threshold / value)
int32_t hb_rf_load(const int32_t *left, const int32_t *right, const int32_t *feature, const double *threshold,
                   const double *value, const int32_t *node_counts, const hb_rf_spec_t *spec, int64_t T,
                   int64_t max_nodes, void *forest, void *stream) {
  return launch_rf_load(left, right, feature, threshold, value, node_counts, spec, T, max_nodes, forest,
                        (cudaStream_t)stream);
}

// general.py:116-140: the Monte-Carlo EHVI of one selection round (hypervolume.cu)
int64_t hb_ehvi_workspace_bytes(int64_t n, int64_t K, int64_t m, int64_t n_mc) { return ehvi_ws_query(n, K, m, n_mc); }

int32_t hb_ehvi(const double *front, int64_t n, int64_t K, const double *samples, int64_t m, int64_t n_mc, const double *ref,
                double *base_hv, double *ehvi, void *ws, int64_t ws_bytes, void *stream) {
  if ((n > 0 && !front) || !samples || !ref || !base_hv || !ehvi || !ws) return HB_ERR_INVALID;
  return launch_ehvi(front, n, K, samples, m, n_mc, ref, base_hv, ehvi, ws, ws_bytes, (cudaStream_t)stream);
}

}  // extern "C"
