// Deep-ensemble surrogate (HEBO/hebo/models/nn/deep_ensemble.py): the whole fit of every member in one launch, and the
// ensemble's predictive mean / variance and their input gradients.
//
// Fit: one CTA per member.  A member's parameters, gradient and Adam moments live in global memory (the parameters in the
// caller's array, the rest in the workspace), which stays L2-resident: the envelope's largest member (3 x 256 hidden units
// with a prior net) holds 1.5 MB of parameters, too much for one SM's shared memory.  The minibatch's activations and
// deltas live in shared memory.  Every output element of every stage is computed by one thread with a sequential loop, so
// each sum runs in a fixed order and a fit is bit-identical from run to run; there are no atomics.
#include "kernels.h"

namespace hb {

constexpr int DE_FIT_THREADS = 512;
constexpr int DE_PRED_THREADS = 256;
constexpr int DE_TM = 16;              // candidates per predict CTA

// One member's parameter layout, in BaseNet's registration order (deep_ensemble.py:183-221)
struct DeNet {
  int dc, ne, din, L, H, O, noise, prior, emb, P, prior0;
  int in_ld, h_ld;
  float noise_lb;
  int w[HB_DE_MAX_LAYERS], b[HB_DE_MAX_LAYERS];      // hidden.{2l}.weight / bias
  int mu_w, mu_b, sg_w, sg_b;                        // mu, sigma2.0
  int pw[HB_DE_MAX_LAYERS], pb[HB_DE_MAX_LAYERS];    // prior_net.{2l}
  int po_w, po_b;                                    // prior_net.prior_net_out
  short col_in[HB_DE_MAX_IN];                        // categorical column c: first input column (after the numeric ones)
  short col_w[HB_DE_MAX_IN];                         // its width (embedding size or categories)
  short in_col[HB_DE_MAX_IN];                        // input column dc + q -> categorical column
  int col_u[HB_DE_MAX_IN];                           // categories of column c
  int col_tab[HB_DE_MAX_IN];                         // offset of its embedding table
};

static bool de_layout(const hb_de_spec_t *s, DeNet &net) {
  if (!s || s->num_cont < 0 || s->num_enum < 0 || s->num_cont + s->num_enum <= 0) return false;
  if (s->num_layers < 1 || s->num_layers > HB_DE_MAX_LAYERS || s->num_hiddens < 1 || s->num_hiddens > HB_DE_MAX_HIDDEN)
    return false;
  if (s->num_out < 1 || s->num_out > HB_DE_MAX_OUT || !(s->noise_lb >= 0.0f)) return false;
  if (s->enum_trans != HB_DE_EMBEDDING && s->enum_trans != HB_DE_ONEHOT) return false;
  if (s->num_enum > 0 && !s->num_uniqs) return false;
  if (s->num_cont > HB_DE_MAX_IN || s->num_enum > HB_DE_MAX_IN) return false;
  net = DeNet{};
  net.dc = s->num_cont;
  net.ne = s->num_enum;
  net.L = s->num_layers;
  net.H = s->num_hiddens;
  net.O = s->num_out;
  net.noise = s->output_noise ? 1 : 0;
  net.prior = s->rand_prior ? 1 : 0;
  net.emb = s->enum_trans == HB_DE_EMBEDDING;
  net.noise_lb = s->noise_lb;
  int64_t p = 0, width = 0;
  for (int c = 0; c < net.ne; ++c) {
    const int u = s->num_uniqs[c];
    if (u < 1) return false;
    const int64_t wc = net.emb ? (u / 2 + 1 < 50 ? u / 2 + 1 : 50) : u;     // models/layers.py:19 / one-hot
    if (width + wc > HB_DE_MAX_IN) return false;
    net.col_in[c] = (short)width;
    net.col_w[c] = (short)wc;
    net.col_u[c] = u;
    for (int q = 0; q < wc; ++q) net.in_col[width + q] = (short)c;
    width += wc;
    if (net.emb) {
      net.col_tab[c] = (int)p;
      p += (int64_t)u * wc;
    }
  }
  net.din = net.dc + (int)width;
  if (net.din < 1 || net.din > HB_DE_MAX_IN) return false;
  int K = net.din;
  for (int l = 0; l < net.L; ++l) {
    net.w[l] = (int)p;
    p += (int64_t)net.H * K;
    net.b[l] = (int)p;
    p += net.H;
    K = net.H;
  }
  net.mu_w = (int)p;
  p += (int64_t)net.O * net.H;
  net.mu_b = (int)p;
  p += net.O;
  if (net.noise) {
    net.sg_w = (int)p;
    p += (int64_t)net.O * net.H;
    net.sg_b = (int)p;
    p += net.O;
  }
  net.prior0 = (int)p;
  if (net.prior) {
    K = net.din;
    for (int l = 0; l < net.L; ++l) {
      net.pw[l] = (int)p;
      p += (int64_t)net.H * K;
      net.pb[l] = (int)p;
      p += net.H;
      K = net.H;
    }
    net.po_w = (int)p;
    p += (int64_t)net.O * net.H;
    net.po_b = (int)p;
    p += net.O;
  }
  net.P = (int)p;
  net.in_ld = net.din | 1;
  net.h_ld = (net.H > net.din ? net.H : net.din) | 1;
  return true;
}

// floats of the per-row buffers of B rows (the envelope formula of include/hebo_b200.h) and the fixed scratch
static int64_t de_rows_floats(const DeNet &net, int64_t B) {
  return B * (net.in_ld + (int64_t)(net.L + 2) * net.h_ld + 5 * net.O + 1);
}
constexpr int DE_SCRATCH = 64;

struct DeSmem {
  float *xin, *act, *d0, *d1, *head, *dhead, *pri;
  int *rows;
  float *red;
};

__device__ __forceinline__ DeSmem de_carve(const DeNet &net, float *base, int B) {
  DeSmem s;
  s.xin = base;
  s.act = s.xin + B * net.in_ld;
  s.d0 = s.act + net.L * B * net.h_ld;
  s.d1 = s.d0 + B * net.h_ld;
  s.head = s.d1 + B * net.h_ld;
  s.dhead = s.head + 2 * B * net.O;
  s.pri = s.dhead + 2 * B * net.O;
  s.rows = (int *)(s.pri + B * net.O);
  s.red = (float *)(s.rows + B);
  return s;
}

// torch.nn.functional.softplus (beta 1, threshold 20) and its derivative
__device__ __forceinline__ float de_softplus(float z) { return z > 20.0f ? z : log1pf(expf(z)); }
__device__ __forceinline__ float de_softplus_d(float z) {
  if (z > 20.0f) return 1.0f;
  const float e = expf(z);
  return e / (e + 1.0f);
}

// y[p, j] = act(bias[j] + sum_k x[p, k] W[j, k]) (+ add[p, j]) for p < B, j < N; W [N, K] row-major (torch's layout);
// bias NULL: no bias term (F.linear(x, W)).  Lanes run over rows p, so W[j, k] is one broadcast load per warp.
__device__ void de_dense(const float *x, int ldx, int B, int K, const float *W, const float *bias, int N, float *y, int ldy,
                         bool relu, const float *add = nullptr, int ld_add = 0) {
  for (int idx = threadIdx.x; idx < B * N; idx += blockDim.x) {
    const int p = idx % B, j = idx / B;
    const float *xr = x + p * ldx;
    const float *wr = W + (size_t)j * K;
    float acc = 0.0f;
    for (int k = 0; k < K; ++k) acc = fmaf(xr[k], wr[k], acc);
    float v = bias ? acc + bias[j] : acc;
    if (relu) v = v < 0.0f ? 0.0f : v;
    if (add) v += add[p * ld_add + j];
    y[p * ldy + j] = v;
  }
}

// The input rows of s.rows: numeric columns (scaled as x * x_mul + x_add when x_mul is given), then the embedding rows
// or one-hot codes of the categorical columns.  A category outside 0 .. u - 1 loads NaN, so its row's outputs are NaN.
// MASK: every input column k is then multiplied by gmask[k] (a feature gate's eval mask, shared by all rows).
// Only columns k0 .. din - 1 are loaded (the Gumbel selection writes its columns 0 .. k0 - 1 itself).
template <bool MASK = false>
__device__ void de_load_inputs(const DeNet &net, const float *prm, const float *X, const int32_t *Xe, const float *x_mul,
                               const float *x_add, const DeSmem &s, int B, const float *gmask = nullptr, int k0 = 0) {
  const int w = net.din - k0;
  for (int idx = threadIdx.x; idx < B * w; idx += blockDim.x) {
    const int p = idx / w, k = k0 + idx % w;
    const int64_t r = s.rows[p];
    float v;
    if (k < net.dc) {
      v = X[r * net.dc + k];
      if (x_mul) v = __fadd_rn(__fmul_rn(x_mul[k], v), x_add[k]);
    } else {
      const int c = net.in_col[k - net.dc], q = k - net.dc - net.col_in[c];
      const int cat = Xe[r * net.ne + c];
      if (cat < 0 || cat >= net.col_u[c])
        v = __int_as_float(0x7fc00000);      // out of range: a NaN row, never a read outside the table
      else
        v = net.emb ? prm[net.col_tab[c] + (int64_t)cat * net.col_w[c] + q] : (cat == q ? 1.0f : 0.0f);
    }
    if constexpr (MASK) v = __fmul_rn(v, gmask[k]);
    s.xin[p * net.in_ld + k] = v;
  }
}

// BaseNet.forward (deep_ensemble.py:229-238) of the B rows in s.xin: prior net into s.pri (through d0 / d1), hidden
// activations into s.act, heads into s.head[p, 0:O] = mu (+ prior) and s.head[p, O:2O] = the sigma2 head's pre-softplus z.
// GATE (FeNet.forward, fe_deep_ensemble.py:29-35): the prior net is built but not evaluated.  DE_GUMBEL (GumbelNet,
// gumbel_linear.py:58-61) evaluates it on the selected inputs.
constexpr int DE_GUMBEL = 2 + HB_FE_HARD_CONCRETE;      // the GATE value of the Gumbel selection layer
template <int GATE = 0>
__device__ void de_forward(const DeNet &net, const float *prm, const DeSmem &s, int B) {
  const bool prior = (GATE == 0 || GATE == DE_GUMBEL) && net.prior;
  if (prior) {
    const float *src = s.xin;
    int ld = net.in_ld, K = net.din;
    for (int l = 0; l < net.L; ++l) {
      float *dst = (l & 1) ? s.d1 : s.d0;
      de_dense(src, ld, B, K, prm + net.pw[l], prm + net.pb[l], net.H, dst, net.h_ld, true);
      __syncthreads();
      src = dst;
      ld = net.h_ld;
      K = net.H;
    }
    de_dense(src, ld, B, K, prm + net.po_w, prm + net.po_b, net.O, s.pri, net.O, false);
    __syncthreads();
  }
  const float *src = s.xin;
  int ld = net.in_ld, K = net.din;
  for (int l = 0; l < net.L; ++l) {
    float *dst = s.act + l * B * net.h_ld;
    de_dense(src, ld, B, K, prm + net.w[l], prm + net.b[l], net.H, dst, net.h_ld, true);
    __syncthreads();
    src = dst;
    ld = net.h_ld;
    K = net.H;
  }
  de_dense(src, ld, B, K, prm + net.mu_w, prm + net.mu_b, net.O, s.head, 2 * net.O, false, prior ? s.pri : nullptr, net.O);
  if (net.noise) de_dense(src, ld, B, K, prm + net.sg_w, prm + net.sg_b, net.O, s.head + net.O, 2 * net.O, false);
  __syncthreads();
}

// From head seeds s.dhead[p, 0:O] (d/d mu) and s.dhead[p, O:2O] (d/d z) back to the hidden layers; cur holds the delta of
// layer l's output after each stage.  With g != nullptr the weight and bias gradients are written to g; with
// want_input the input delta of layer 0 goes to columns [k0, din) of the returned buffer.  Returns that buffer.
__device__ float *de_backward(const DeNet &net, const float *prm, const DeSmem &s, int B, float *g, bool want_input, int k0) {
  const int H = net.H, O = net.O, hl = net.h_ld;
  const float *aL = s.act + (net.L - 1) * B * hl;
  if (g) {
    for (int idx = threadIdx.x; idx < O * H; idx += blockDim.x) {
      const int o = idx / H, j = idx % H;
      float gm = 0.0f, gs = 0.0f;
      for (int p = 0; p < B; ++p) {
        gm = fmaf(s.dhead[p * 2 * O + o], aL[p * hl + j], gm);
        if (net.noise) gs = fmaf(s.dhead[p * 2 * O + O + o], aL[p * hl + j], gs);
      }
      g[net.mu_w + idx] = gm;
      if (net.noise) g[net.sg_w + idx] = gs;
    }
    for (int o = threadIdx.x; o < O; o += blockDim.x) {
      float gm = 0.0f, gs = 0.0f;
      for (int p = 0; p < B; ++p) {
        gm += s.dhead[p * 2 * O + o];
        gs += s.dhead[p * 2 * O + O + o];
      }
      g[net.mu_b + o] = gm;
      if (net.noise) g[net.sg_b + o] = gs;
    }
  }
  for (int idx = threadIdx.x; idx < B * H; idx += blockDim.x) {
    const int p = idx / H, j = idx % H;
    float acc = 0.0f;
    for (int o = 0; o < O; ++o) {
      acc = fmaf(s.dhead[p * 2 * O + o], prm[net.mu_w + o * H + j], acc);
      if (net.noise) acc = fmaf(s.dhead[p * 2 * O + O + o], prm[net.sg_w + o * H + j], acc);
    }
    s.d0[p * hl + j] = aL[p * hl + j] > 0.0f ? acc : 0.0f;
  }
  __syncthreads();
  float *cur = s.d0, *nxt = s.d1;
  for (int l = net.L - 1; l >= 0; --l) {
    const float *in = l == 0 ? s.xin : s.act + (l - 1) * B * hl;
    const int ldi = l == 0 ? net.in_ld : hl, K = l == 0 ? net.din : H;
    const float *W = prm + net.w[l];
    if (g) {
      for (int idx = threadIdx.x; idx < H * K; idx += blockDim.x) {
        const int j = idx / K, k = idx % K;
        float acc = 0.0f;
        for (int p = 0; p < B; ++p) acc = fmaf(cur[p * hl + j], in[p * ldi + k], acc);
        g[net.w[l] + idx] = acc;
      }
      for (int j = threadIdx.x; j < H; j += blockDim.x) {
        float acc = 0.0f;
        for (int p = 0; p < B; ++p) acc += cur[p * hl + j];
        g[net.b[l] + j] = acc;
      }
    }
    if (l > 0 || want_input) {
      const int kb = l > 0 ? 0 : k0;
      for (int idx = threadIdx.x; idx < B * (K - kb); idx += blockDim.x) {
        const int p = idx / (K - kb), k = kb + idx % (K - kb);
        float acc = 0.0f;
        for (int j = 0; j < H; ++j) acc = fmaf(cur[p * hl + j], W[(size_t)j * K + k], acc);
        nxt[p * hl + k] = (l == 0 || in[p * ldi + k] > 0.0f) ? acc : 0.0f;
      }
    }
    __syncthreads();
    float *t = cur;
    cur = nxt;
    nxt = t;
  }
  return cur;
}

// ------------------------------------------------------------------------------------------------ permutation
// Round r of the Feistel network on 2h bits: word 0 of the Philox block of (half, epoch, member, 0x44450000 + r).
__device__ __forceinline__ uint32_t de_feistel(uint32_t x, int h, uint64_t seed, uint32_t epoch, uint32_t member) {
  const uint32_t mask = (1u << h) - 1u;
  uint32_t L = x >> h, R = x & mask;
#pragma unroll
  for (int r = 0; r < 4; ++r) {
    uint32_t c[4] = {R, epoch, member, 0x44450000u + (uint32_t)r};
    philox4x32_10(c, seed);
    const uint32_t nR = L ^ (c[0] & mask);
    L = R;
    R = nR;
  }
  return (L << h) | R;
}

__device__ __forceinline__ int de_perm(int pos, int n, int h, uint64_t seed, int epoch, int member) {
  uint32_t x = (uint32_t)pos;
  do {
    x = de_feistel(x, h, seed, (uint32_t)epoch, (uint32_t)member);
  } while (x >= (uint32_t)n);
  return (int)x;
}

// ------------------------------------------------------------------------------------------------ selection
// A member's selection layer.  GATE = 0: none (BaseNet).  GATE = 1 + HB_FE_STG | HB_FE_CONCRETE | HB_FE_HARD_CONCRETE:
// FeNet's gate (fe_layers.py) on the input columns, one parameter theta per column, [din] after BaseNet's P: mu (stg) or
// logits (concrete layers).  GATE = DE_GUMBEL: GumbelNet's selection of the numeric columns (below).
struct DeSel {
  int off;               // first selection parameter (BaseNet's P); a member holds off + din (gate) or off + r dx floats
  float T;               // stg: its temperature throughout; concrete layers and Gumbel: predict's (the last epoch's)
  float mcoef;           // gate: fp32 (1 / (n num_out)) * mask_reg, 0 without numeric columns (no mask penalty)
  int gate;              // GATE
  double t0, t1, tb;     // gate: start_temp, end_temp, anneal_base of the concrete layers' schedule
  const float *draws;    // raw draws, or NULL: Philox.  Gate: fit [E, epochs, nb, B, din] / predict [E, din]; Gumbel:
                         // fit [E, epochs, nb, r, dx] / predict [E, r, dx] uniforms
  uint64_t seed, counter;      // predict's Philox key
  int dx, r, x_ld;       // Gumbel: numeric columns of the data, selected columns, leading dimension of the on-chip numeric rows
  float *w;              // Gumbel: [E, r, dx] each member's W of the current step (fit) or call (predict)
};

// ------------------------------------------------------------------------------------------------ feature gate
constexpr uint32_t FE_TAG_FIT = 0x46454654u;      // upper word of the Philox counter of the training draws ('FEFT')
constexpr uint32_t FE_TAG_EVAL = 0x46454556u;     // ... and of the eval draws ('FEEV')

// Raw draw `half` of the Philox block (row, stream): N(0, 1) by philox_normal2 for stg, U(0, 1] word for the concrete layers
template <int GATE>
__device__ __forceinline__ float fe_draw(uint64_t seed, uint64_t row, uint64_t stream, int half) {
  if constexpr (GATE == 1 + HB_FE_STG) {
    float z0, z1;
    philox_normal2(seed, row, stream, z0, z1);
    return half ? z1 : z0;
  } else {
    uint32_t c[4] = {(uint32_t)row, (uint32_t)(row >> 32), (uint32_t)stream, (uint32_t)(stream >> 32)};
    philox4x32_10(c, seed);
    return philox_uniform(c[half]);
  }
}

// sigmoid((logits + logit(u)) / T) with u clamped to [eps, 1 - eps] (ConcreteLayer.gumbel_sigmoid, fe_layers.py:44-50)
__device__ __forceinline__ float fe_concrete(float theta, float r, float T) {
  const float u = fminf(fmaxf(r, 1.1920928955078125e-07f), 0.99999988079071044921875f);
  const float ul = logf(__fdiv_rn(u, __fsub_rn(1.0f, u)));
  const float zt = __fdiv_rn(__fadd_rn(theta, ul), T);
  return __frcp_rn(__fadd_rn(1.0f, expf(-zt)));
}

// The gate's state st of one element (stg: the pre-clamp mu + 0.5 + T r; concrete layers: the sigmoid) and its mask
template <int GATE>
__device__ __forceinline__ float fe_state(float theta, float r, float T) {
  if constexpr (GATE == 1 + HB_FE_STG) return __fadd_rn(__fadd_rn(__fmul_rn(T, r), theta), 0.5f);
  else return fe_concrete(theta, r, T);
}
template <int GATE>
__device__ __forceinline__ float fe_mask(float st) {
  if constexpr (GATE == 1 + HB_FE_CONCRETE) return st;
  const float v = GATE == 1 + HB_FE_STG ? st : __fadd_rn(__fmul_rn(st, 1.2f), -0.1f);      // hard: stretch to [-0.1, 1.1]
  return fminf(fmaxf(v, 0.0f), 1.0f);
}
// d loss / d theta of one element from gm = d loss / d mask, through torch.clamp's pass-through (inclusive at both bounds)
template <int GATE>
__device__ __forceinline__ float fe_dtheta(float st, float gm, float T) {
  if constexpr (GATE == 1 + HB_FE_STG) return (st >= 0.0f && st <= 1.0f) ? gm : 0.0f;
  if constexpr (GATE == 1 + HB_FE_HARD_CONCRETE) {
    const float v = __fadd_rn(__fmul_rn(st, 1.2f), -0.1f);
    gm = (v >= 0.0f && v <= 1.0f) ? __fmul_rn(gm, 1.2f) : 0.0f;
  }
  return __fdiv_rn(__fmul_rn(__fmul_rn(gm, __fsub_rn(1.0f, st)), st), T);
}
// d mask_loss / d theta: mcoef d mask_norm / d theta, mask_norm = sum Phi((mu + 0.5) / T) (stg) or sum sigmoid(logits)
template <int GATE>
__device__ __forceinline__ float fe_dnorm(float theta, float mcoef, float T) {
  if constexpr (GATE == 1 + HB_FE_STG) {
    const float w = __fdiv_rn(__fdiv_rn(__fadd_rn(theta, 0.5f), T), 1.41421356237309515f);
    const float g = __fmul_rn(__fmul_rn(mcoef, 0.5f), __fmul_rn(1.12837916709551257f, expf(-__fmul_rn(w, w))));
    return __fdiv_rn(__fdiv_rn(g, 1.41421356237309515f), T);
  } else {
    const float sg = __frcp_rn(__fadd_rn(1.0f, expf(-theta)));
    return __fmul_rn(__fmul_rn(mcoef, __fsub_rn(1.0f, sg)), sg);
  }
}

// parameter i is a weight (its state_dict name contains 'weight'): FeDeepEnsemble's L1 set (fe_deep_ensemble.py:62-64)
__device__ __forceinline__ bool fe_is_weight(const DeNet &net, int i, int off) {
  if (i >= off) return false;
  const auto in = [i](int a, int n) { return i >= a && i < a + n; };
  for (int l = 0; l < net.L; ++l)
    if (in(net.b[l], net.H) || (net.prior && in(net.pb[l], net.H))) return false;
  return !(in(net.mu_b, net.O) || (net.noise && in(net.sg_b, net.O)) || (net.prior && in(net.po_b, net.O)));
}

// ------------------------------------------------------------------------------------------------ Gumbel selection
// GumbelNet's feature_select (gumbel_linear.py:21-40) on the dx numeric columns: x_sel = x_num W^T [B, r] with
// W = RelaxedOneHotCategorical(T, logits).rsample() [r, dx], one W per forward shared by every row.  The member's DeNet is
// BaseNet's layout with num_cont = r (its input row is [x_sel | embedding or one-hot]); the logits [r, dx] follow it.
constexpr uint32_t GB_TAG_FIT = 0x47424654u;      // upper word of the Philox counter of the training draws ('GBFT')
constexpr uint32_t GB_TAG_EVAL = 0x47424556u;     // ... and of the eval draws ('GBEV')

__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// torch.logsumexp of v[0 .. n - 1] over one warp: max, a max of +-inf taken as 0, log(sum exp(v - max)) + max
__device__ __forceinline__ float gb_warp_lse(const float *v, int n) {
  const int lane = threadIdx.x & 31;
  float mx = -INFINITY;
  for (int k = lane; k < n; k += 32) mx = fmaxf(mx, v[k]);
  mx = warp_max(mx);
  if (isinf(mx)) mx = 0.0f;
  float sm = 0.0f;
  for (int k = lane; k < n; k += 32) sm += expf(__fsub_rn(v[k], mx));
  return __fadd_rn(logf(warp_sum(sm)), mx);
}

// W [r, dx] of one member from its logits and uniforms draw(j, k), one warp per row j, in ExpRelaxedCategorical.rsample's
// order: L = logits - lse(logits) (Categorical), g = -log(-log(clamp(u, eps, 1 - eps))), s = (L + g) / T (fp32 division
// by fp32(T), as torch divides an fp32 tensor by a Python float), W = exp(s - lse(s)).
template <class Draw>
__device__ void gb_build_w(const float *theta, int r, int dx, float T, float *W, Draw draw) {
  const int lane = threadIdx.x & 31, nw = blockDim.x >> 5;
  for (int j = threadIdx.x >> 5; j < r; j += nw) {
    const float *th = theta + (size_t)j * dx;
    float *w = W + (size_t)j * dx;
    const float lse = gb_warp_lse(th, dx);
    for (int k = lane; k < dx; k += 32) {
      const float u = fminf(fmaxf(draw(j, k), 1.1920928955078125e-07f), 0.99999988079071044921875f);
      const float g = -logf(-logf(u));
      w[k] = __fdiv_rn(__fadd_rn(__fsub_rn(th[k], lse), g), T);
    }
    __syncwarp();
    const float ls = gb_warp_lse(w, dx);
    __syncwarp();
    for (int k = lane; k < dx; k += 32) w[k] = expf(__fsub_rn(w[k], ls));
  }
}

// In place, row by row (one warp each): d = dW [r, dx] -> d loss / d logits through W = exp(s - lse(s)), s = (L + g) / T
// and L = logits - lse(logits), each logsumexp's backward included (the normalisation terms are not dropped).
__device__ void gb_logits_grad(const float *theta, const float *W, float *d, int r, int dx, float T) {
  const int lane = threadIdx.x & 31, nw = blockDim.x >> 5;
  for (int j = threadIdx.x >> 5; j < r; j += nw) {
    const float *th = theta + (size_t)j * dx, *w = W + (size_t)j * dx;
    float *dr = d + (size_t)j * dx;
    float s1 = 0.0f;
    for (int k = lane; k < dx; k += 32) {
      const float dz = __fmul_rn(dr[k], w[k]);      // exp's backward
      dr[k] = dz;
      s1 += dz;
    }
    s1 = -warp_sum(s1);
    float s2 = 0.0f;
    for (int k = lane; k < dx; k += 32) {
      const float dl = __fdiv_rn(__fadd_rn(dr[k], __fmul_rn(s1, w[k])), T);
      dr[k] = dl;
      s2 += dl;
    }
    s2 = -warp_sum(s2);
    const float lse = gb_warp_lse(th, dx);
    for (int k = lane; k < dx; k += 32) dr[k] = __fadd_rn(dr[k], __fmul_rn(s2, expf(__fsub_rn(th[k], lse))));
  }
}

// ------------------------------------------------------------------------------------------------ fit
struct DeFitArgs {
  const float *Xc, *y;
  const int32_t *Xe, *perm;
  float *params, *m1, *m2, *grad, *losses;
  int n, B, nb, epochs, h;
  uint64_t seed;
  double lr;
  float coef;       // fp32 (1 / (n num_out)) * l1: the L1 term's gradient per unit sign
};

// The whole fit of one member: a's pointers are its ensemble's (params [E, P], m1 / m2 / grad [E, P], losses [E, epochs]).
// Step bi takes rows bi B .. min((bi + 1) B, n) - 1 of the epoch's order, so a.nb decides whether a partial last
// minibatch is trained (a.nb = ceil(n / B)) or dropped.
// GATE: FeDeepEnsemble.fit_one (fe_deep_ensemble.py:46-75) with sel's gate; the unmasked inputs and the gate states of
// the minibatch sit in two more [B, in_ld] buffers after the scratch.  DE_GUMBEL: GumbelDeepEnsemble.fit_one
// (gumbel_linear.py:69-100) with sel's selection layer; the numeric rows sit in one [B, x_ld] buffer after the scratch.
template <int GATE = 0>
__device__ __forceinline__ void de_fit_member(const DeNet &net, const DeFitArgs &a, int member, float *smem,
                                              const DeSel *sel = nullptr) {
  const int B = a.B, O = net.O;
  const DeSmem s = de_carve(net, smem, B);
  float *xraw = s.red + DE_SCRATCH, *gst = xraw + B * net.in_ld;
  constexpr bool GUMBEL = GATE == DE_GUMBEL;
  const int wsz = GUMBEL ? sel->r * sel->dx : 0;
  float *W = GUMBEL ? sel->w + (size_t)member * wsz : nullptr;
  float *prm = a.params + (size_t)member * net.P;
  float *m1 = a.m1 + (size_t)member * net.P, *m2 = a.m2 + (size_t)member * net.P, *g = a.grad + (size_t)member * net.P;
  for (int i = threadIdx.x; i < net.P; i += blockDim.x) {
    m1[i] = 0.0f;
    m2[i] = 0.0f;
    g[i] = 0.0f;
  }
  int step = 0;
  for (int ep = 0; ep < a.epochs; ++ep) {
    float epoch_loss = 0.0f;     // thread 0
    float T = 0.0f;
    if constexpr (GATE == 1 + HB_FE_STG) T = sel->T;
    else if constexpr (GUMBEL) T = (float)(pow(0.8, (double)ep) + 0.1);     // 0.8**epoch + 0.1, a double, used as fp32
    else if constexpr (GATE != 0) T = (float)fmax(sel->t0 * pow(sel->tb, (double)ep), sel->t1);     // torch.tensor(.).clamp(end)
    for (int bi = 0; bi < a.nb; ++bi) {
      ++step;
      const int Bs = min(B, a.n - bi * B);      // rows of this step
      for (int p = threadIdx.x; p < Bs; p += blockDim.x) {
        const int pos = bi * B + p;
        s.rows[p] = a.perm ? a.perm[((size_t)member * a.epochs + ep) * a.n + pos] : de_perm(pos, a.n, a.h, a.seed, ep, member);
      }
      __syncthreads();
      if constexpr (GUMBEL) {
        if (sel->dx > 0) {       // this step's W from fresh uniforms, then x_sel = x_num W^T; x_num stays for the backward
          const int dx = sel->dx, r = sel->r;
          const size_t base = (((size_t)member * a.epochs + ep) * a.nb + bi) * (size_t)wsz;
          const uint64_t q0 = ((uint64_t)ep * a.nb + bi) * (uint64_t)wsz;
          gb_build_w(prm + sel->off, r, dx, T, W, [&](int j, int k) {
            const uint64_t q = q0 + (uint64_t)j * dx + k;
            return sel->draws ? sel->draws[base + (size_t)j * dx + k]
                              : fe_draw<1 + HB_FE_CONCRETE>(a.seed, q >> 1, ((uint64_t)GB_TAG_FIT << 32) | (uint32_t)member,
                                                            (int)(q & 1));
          });
          for (int idx = threadIdx.x; idx < Bs * dx; idx += blockDim.x)
            xraw[(idx / dx) * sel->x_ld + idx % dx] = a.Xc[(int64_t)s.rows[idx / dx] * dx + idx % dx];
          __syncthreads();
          de_dense(xraw, sel->x_ld, Bs, dx, W, nullptr, r, s.xin, net.in_ld, false);
        }
        de_load_inputs(net, prm, a.Xc, a.Xe, nullptr, nullptr, s, Bs, nullptr, net.dc);
      } else {
        de_load_inputs(net, prm, a.Xc, a.Xe, nullptr, nullptr, s, Bs);
      }
      __syncthreads();
      if constexpr (GATE != 0 && !GUMBEL) {       // x * mask with a fresh draw per row and column (the training mask of x.shape)
        const size_t base = (((size_t)member * a.epochs + ep) * a.nb + bi) * (size_t)B * net.din;
        for (int idx = threadIdx.x; idx < B * net.din; idx += blockDim.x) {
          const int p = idx / net.din, k = idx % net.din;
          const uint64_t q = (((uint64_t)ep * a.nb + bi) * B + p) * net.din + k;
          const float r = sel->draws ? sel->draws[base + idx]
                                     : fe_draw<GATE>(a.seed, q >> 1, ((uint64_t)FE_TAG_FIT << 32) | (uint32_t)member, (int)(q & 1));
          const float x = s.xin[p * net.in_ld + k], st = fe_state<GATE>(prm[sel->off + k], r, T);
          xraw[p * net.in_ld + k] = x;
          gst[p * net.in_ld + k] = st;
          s.xin[p * net.in_ld + k] = __fmul_rn(x, fe_mask<GATE>(st));
        }
        __syncthreads();
      }
      de_forward<GATE>(net, prm, s, Bs);
      // the loss over the finite entries of y (loss_likelihood / loss_mse, deep_ensemble.py:140-149)
      if (threadIdx.x < 32) {
        float cnt = 0.0f;
        for (int i = threadIdx.x; i < Bs * O; i += 32) cnt += isfinite(a.y[(int64_t)s.rows[i / O] * O + i % O]) ? 1.0f : 0.0f;
        cnt = warp_sum(cnt);
        if (threadIdx.x == 0) s.red[0] = cnt;
      }
      __syncthreads();
      const float cnt = s.red[0];
      for (int i = threadIdx.x; i < Bs * O; i += blockDim.x) {
        const int p = i / O, o = i % O;
        const float t = a.y[(int64_t)s.rows[p] * O + o];
        float el = 0.0f, gmu = 0.0f, gz = 0.0f;
        if (isfinite(t)) {
          const float mu = s.head[p * 2 * O + o], diff = t - mu;
          if (net.noise) {
            const float z = s.head[p * 2 * O + O + o];
            const float s2 = net.noise_lb + de_softplus(z);
            el = 0.5f * (diff * diff) / s2 + 0.5f * logf(s2);
            gmu = -diff / s2 / cnt;
            gz = (0.5f / s2 - 0.5f * (diff * diff) / (s2 * s2)) / cnt * de_softplus_d(z);
          } else {
            el = diff * diff;
            gmu = -2.0f * diff / cnt;
          }
        }
        s.dhead[p * 2 * O + o] = gmu;
        s.dhead[p * 2 * O + O + o] = gz;
        s.pri[i] = el;      // the prior output is no longer needed: mu already holds it
      }
      __syncthreads();
      if (threadIdx.x < 32) {
        float sum = 0.0f;
        for (int i = threadIdx.x; i < Bs * O; i += 32) sum += s.pri[i];
        sum = warp_sum(sum);
        if (threadIdx.x == 0) epoch_loss += sum / cnt * (float)Bs;      // epoch_loss += data_loss * bxc.shape[0]
      }
      const bool selw = GUMBEL && sel->dx > 0;
      float *dx = GATE && !GUMBEL ? de_backward(net, prm, s, Bs, g, true, 0)
                                  : de_backward(net, prm, s, Bs, g, selw || (net.emb && net.ne > 0), selw ? 0 : net.dc);
      if (selw) {
        // d loss / d W [j, k] = sum over the rows in order of delta_sel[p, j] x_num[p, k], then through the softmax
        const int dx_ = sel->dx;
        for (int idx = threadIdx.x; idx < wsz; idx += blockDim.x) {
          const int j = idx / dx_, k = idx % dx_;
          float acc = 0.0f;
          for (int p = 0; p < Bs; ++p) acc = fmaf(dx[p * net.h_ld + j], xraw[p * sel->x_ld + k], acc);
          g[sel->off + idx] = acc;
        }
        __syncthreads();
        gb_logits_grad(prm + sel->off, W, g + sel->off, sel->r, dx_, T);
        __syncthreads();
      }
      if constexpr (GATE != 0 && !GUMBEL) {
        // column k: d loss / d theta_k = sum over rows in order of (dx x) through the mask, plus the mask penalty's;
        // then dx becomes the delta of the unmasked input (dx mask) for the embedding tables
        for (int k = threadIdx.x; k < net.din; k += blockDim.x) {
          const float theta = prm[sel->off + k];
          float acc = 0.0f;
          for (int p = 0; p < B; ++p) {
            float &d = dx[p * net.h_ld + k];
            const float st = gst[p * net.in_ld + k];
            acc += fe_dtheta<GATE>(st, __fmul_rn(d, xraw[p * net.in_ld + k]), T);
            d = __fmul_rn(d, fe_mask<GATE>(st));
          }
          g[sel->off + k] = sel->mcoef != 0.0f ? __fadd_rn(acc, fe_dnorm<GATE>(theta, sel->mcoef, T)) : acc;
        }
        __syncthreads();
      }
      // embedding tables: the input delta of each row added into the row of its category, rows in batch order
      if (net.emb) {
        for (int c = 0; c < net.ne; ++c) {
          const int wc = net.col_w[c], tab = net.col_u[c] * wc;
          for (int idx = threadIdx.x; idx < tab; idx += blockDim.x) {
            const int u = idx / wc, q = idx % wc;
            float acc = 0.0f;
            for (int p = 0; p < Bs; ++p)
              if (a.Xe[(int64_t)s.rows[p] * net.ne + c] == u) acc += dx[p * net.h_ld + net.dc + net.col_in[c] + q];
            g[net.col_tab[c] + idx] = acc;
          }
        }
        __syncthreads();
      }
      // L1 term + torch.optim.Adam, single-tensor update (torch/optim/adam.py _single_tensor_adam) in IEEE fp32
      const double bc1 = 1.0 - pow(0.9, (double)step);
      const double bc2s = sqrt(1.0 - pow(0.999, (double)step));
      const float neg_step = (float)(-(a.lr / bc1)), bc2f = (float)bc2s;
      for (int i = threadIdx.x; i < net.P; i += blockDim.x) {
        const float p = prm[i];
        const float sg = p > 0.0f ? 1.0f : (p < 0.0f ? -1.0f : 0.0f);
        float gd, gt;
        if constexpr (GATE != 0) {      // L1 over the weights only; the prior net's biases keep gt = 0 and do not move
          const int off = sel->off;
          gd = (i < net.prior0 || i >= off) ? g[i] : 0.0f;
          gt = fe_is_weight(net, i, off) ? __fadd_rn(gd, __fmul_rn(a.coef, sg)) : gd;
        } else {
          gd = i < net.prior0 ? g[i] : 0.0f;
          gt = __fadd_rn(gd, __fmul_rn(a.coef, sg));
        }
        const float mm = __fadd_rn(m1[i], __fmul_rn(0.1f, __fsub_rn(gt, m1[i])));
        const float vv = __fadd_rn(__fmul_rn(m2[i], 0.999f), __fmul_rn(__fmul_rn(0.001f, gt), gt));
        const float denom = __fadd_rn(__fdiv_rn(__fsqrt_rn(vv), bc2f), 1e-8f);
        prm[i] = __fadd_rn(p, __fdiv_rn(__fmul_rn(neg_step, mm), denom));
        m1[i] = mm;
        m2[i] = vv;
        g[i] = gt;
      }
      __syncthreads();
    }
    if (threadIdx.x == 0) a.losses[(size_t)member * a.epochs + ep] = epoch_loss / (float)a.n;
  }
}

template <int GATE>
__global__ void __launch_bounds__(DE_FIT_THREADS) de_fit_kernel(const __grid_constant__ DeNet net, const DeFitArgs a,
                                                                const __grid_constant__ DeSel sel) {
  extern __shared__ float smem[];
  de_fit_member<GATE>(net, a, blockIdx.x, smem, &sel);
}

// Per-ensemble arguments of hb_de_fit_batch: its rows [off, off + n) of the concatenated inputs and what follows from n
struct DeFitSlot {
  int64_t off;
  uint64_t seed;
  float coef;
  int n, B, nb, h;
};

struct DeFitBatchArgs {
  DeFitArgs a;         // concatenated Xc / Xe / y, params [nens, E, P], m1 = the workspace, losses [nens, E, epochs]
  int E;
  DeFitSlot slot[HB_MAX_OUTPUTS];
};

// CTA (b, member) = blockIdx.x = b E + member runs de_fit_kernel<0>'s member on ensemble b's slices
__global__ void __launch_bounds__(DE_FIT_THREADS) de_fit_batch_kernel(const __grid_constant__ DeNet net,
                                                                       const __grid_constant__ DeFitBatchArgs ba) {
  extern __shared__ float smem[];
  const int b = blockIdx.x / ba.E, member = blockIdx.x % ba.E;
  const DeFitSlot &sl = ba.slot[b];
  const size_t EP = (size_t)ba.E * net.P;
  DeFitArgs a = ba.a;
  a.Xc = a.Xc ? a.Xc + sl.off * net.dc : nullptr;
  a.Xe = a.Xe ? a.Xe + sl.off * net.ne : nullptr;
  a.y += sl.off * net.O;
  a.params += b * EP;
  a.m1 += 3 * b * EP;
  a.m2 = a.m1 + EP;
  a.grad = a.m2 + EP;
  a.losses += (size_t)b * ba.E * a.epochs;
  a.n = sl.n;
  a.B = sl.B;
  a.nb = sl.nb;
  a.h = sl.h;
  a.seed = sl.seed;
  a.coef = sl.coef;
  de_fit_member(net, a, member, smem);
}

// ------------------------------------------------------------------------------------------------ predict
struct DePredArgs {
  const float *Xs, *params, *x_mul, *x_add, *y_mean, *y_std;
  const int32_t *Xe;
  float *mu, *var, *dmu, *dvar;
  int m, E, member;
};

// Rows r0 .. r0 + DE_TM - 1 of the candidates (the last one repeated past m) through members e0 .. e1 - 1: the heads mu
// into mus[e - e0][p, o] and, with output_noise, sigma2 into s2s[e - e0][p, o].  GATE: member e's eval mask [din] (one
// draw per column, shared by every row) goes to gmask and multiplies the inputs in the load.  DE_GUMBEL: the tile's
// scaled numeric rows go to gmask [B, x_ld] once, and member e's x_sel takes its W of the call, sel->w [e].
template <int GATE = 0>
__device__ __forceinline__ void de_member_heads(const DeNet &net, const DePredArgs &a, const DeSmem &s, int r0, int e0,
                                                int e1, float *mus, float *s2s, const DeSel *sel = nullptr,
                                                float *gmask = nullptr) {
  const int O = net.O, B = DE_TM;
  for (int p = threadIdx.x; p < B; p += blockDim.x) s.rows[p] = min(r0 + p, a.m - 1);
  __syncthreads();
  if constexpr (GATE == DE_GUMBEL) {
    const int dx = sel->dx;
    for (int idx = threadIdx.x; idx < B * dx; idx += blockDim.x) {
      const int p = idx / dx, k = idx % dx;
      gmask[p * sel->x_ld + k] = __fadd_rn(__fmul_rn(a.x_mul[k], a.Xs[(int64_t)s.rows[p] * dx + k]), a.x_add[k]);
    }
    __syncthreads();
  }
  for (int e = e0; e < e1; ++e) {
    const float *prm = a.params + (size_t)e * net.P;
    if constexpr (GATE == DE_GUMBEL) {
      if (sel->dx > 0) de_dense(gmask, sel->x_ld, B, sel->dx, sel->w + (size_t)e * sel->r * sel->dx, nullptr, sel->r, s.xin, net.in_ld, false);
      de_load_inputs(net, prm, a.Xs, a.Xe, a.x_mul, a.x_add, s, B, nullptr, net.dc);
    } else if constexpr (GATE != 0) {
      for (int k = threadIdx.x; k < net.din; k += blockDim.x) {
        const uint64_t stream = ((uint64_t)FE_TAG_EVAL << 32) | ((uint32_t)e << 16) | (uint32_t)(k >> 1);
        const float r = sel->draws ? sel->draws[(size_t)e * net.din + k] : fe_draw<GATE>(sel->seed, sel->counter, stream, k & 1);
        gmask[k] = fe_mask<GATE>(fe_state<GATE>(prm[sel->off + k], r, sel->T));
      }
      __syncthreads();
      de_load_inputs<true>(net, prm, a.Xs, a.Xe, a.x_mul, a.x_add, s, B, gmask);
    } else {
      de_load_inputs(net, prm, a.Xs, a.Xe, a.x_mul, a.x_add, s, B);
    }
    __syncthreads();
    de_forward<GATE>(net, prm, s, B);
    for (int i = threadIdx.x; i < B * O; i += blockDim.x) {
      const int p = i / O, o = i % O;
      mus[(e - e0) * B * O + i] = s.head[p * 2 * O + o];
      if (net.noise) s2s[(e - e0) * B * O + i] = net.noise_lb + de_softplus(s.head[p * 2 * O + O + o]);
    }
    __syncthreads();
  }
}

// the ensemble combination of tile entry i over ne members in member order (deep_ensemble.py:97-106); single: one
// member's own mu
__device__ __forceinline__ void de_combine(const DeNet &net, const float *mus, const float *s2s, int ne, int i, bool single,
                                           float &mean, float &v) {
  const int BO = DE_TM * net.O;
  mean = 0.0f;
  v = 0.0f;
  if (single) {
    mean = mus[i];
    return;
  }
  for (int e = 0; e < ne; ++e) mean += mus[e * BO + i];
  mean = mean / (float)ne;
  for (int e = 0; e < ne; ++e) {
    const float dlt = mus[e * BO + i] - mean;
    v = fmaf(dlt, dlt, v);
  }
  v = v / (float)ne;
  if (net.noise) {
    float sm = 0.0f;
    for (int e = 0; e < ne; ++e) sm += s2s[e * BO + i];
    v = v + sm / (float)ne;
  } else {
    v = 1e-8f + v;
  }
}

// GATE: sel's gate on every member (no input gradients: FeDeepEnsemble.support_grad = False); the eval mask sits after
// py.  DE_GUMBEL: sel's selection on every member (no input gradients either); the numeric rows sit after py.
template <bool GRAD, int GATE = 0>
__global__ void __launch_bounds__(DE_PRED_THREADS) de_predict_kernel(const __grid_constant__ DeNet net, const DePredArgs a,
                                                                     const __grid_constant__ DeSel sel) {
  static_assert(!(GRAD && GATE), "the gated ensemble has no input gradients");
  extern __shared__ float smem[];
  const int O = net.O, B = DE_TM, r0 = blockIdx.x * DE_TM;
  const DeSmem s = de_carve(net, smem, B);
  const int e0 = a.member >= 0 ? a.member : 0, e1 = a.member >= 0 ? a.member + 1 : a.E, ne = e1 - e0;
  float *mus = s.red + DE_SCRATCH, *s2s = mus + ne * B * O, *py = s2s + ne * B * O;
  de_member_heads<GATE>(net, a, s, r0, e0, e1, mus, s2s, &sel, py + B * O);
  for (int i = threadIdx.x; i < B * O; i += blockDim.x) {
    const int p = i / O, o = i % O, row = r0 + p;
    float mean, v;
    de_combine(net, mus, s2s, ne, i, a.member >= 0, mean, v);
    py[i] = mean;
    if (row < a.m) {
      const float sd = a.y_std[o];
      a.mu[(int64_t)row * O + o] = __fadd_rn(__fmul_rn(mean, sd), a.y_mean[o]);
      if (a.var) a.var[(int64_t)row * O + o] = __fmul_rn(v, __fmul_rn(sd, sd));
    }
  }
  if constexpr (GRAD) {
    const int dc = net.dc;
    for (int i = threadIdx.x; i < B * O * dc; i += blockDim.x) {
      const int row = r0 + i / (O * dc);
      if (row < a.m) {
        a.dmu[(int64_t)r0 * O * dc + i] = 0.0f;
        a.dvar[(int64_t)r0 * O * dc + i] = 0.0f;
      }
    }
    __syncthreads();
    const float invE = 1.0f / (float)ne;
    for (int e = e0; e < e1; ++e) {
      const float *prm = a.params + (size_t)e * net.P;
      de_load_inputs(net, prm, a.Xs, a.Xe, a.x_mul, a.x_add, s, B);
      __syncthreads();
      de_forward(net, prm, s, B);
      for (int o = 0; o < O; ++o) {
        for (int pass = 0; pass < 2; ++pass) {
          // seeds: d py / d (mu_e, z_e) and d ps2 / d (mu_e, z_e) of output o
          for (int i = threadIdx.x; i < B * 2 * O; i += blockDim.x) {
            const int p = i / (2 * O), c = i % (2 * O);
            float sd = 0.0f;
            if (c == o) {
              sd = pass == 0 ? invE : 2.0f * invE * (mus[(e - e0) * B * O + p * O + o] - py[p * O + o]);
            } else if (c == O + o && pass == 1 && net.noise) {
              sd = invE * de_softplus_d(s.head[p * 2 * O + O + o]);
            }
            s.dhead[i] = sd;
          }
          __syncthreads();
          const float *dx = de_backward(net, prm, s, B, nullptr, true, 0);
          float *out = pass == 0 ? a.dmu : a.dvar;
          for (int i = threadIdx.x; i < B * dc; i += blockDim.x) {
            const int p = i / dc, k = i % dc, row = r0 + p;
            if (row < a.m) {
              const float sd = a.y_std[o], sc = pass == 0 ? sd : __fmul_rn(sd, sd);
              float &dst = out[((int64_t)row * O + o) * dc + k];
              dst = __fadd_rn(dst, __fmul_rn(__fmul_rn(dx[p * net.h_ld + k], a.x_mul[k]), sc));
            }
          }
          __syncthreads();
        }
      }
    }
  }
}

// B ensembles of one spec over one candidate batch: CTA (tile, b) = (blockIdx.x, blockIdx.y) runs de_predict_kernel's
// member loop and combination on ensemble b's parameters and scalers, and writes mu / var output-major, [nens O, m]; with
// nsamp > 0 also y_samp[t, row, b O + o] = py + sqrt(ps2) * xi (BaseModel.sample_y, base_model.py:78-84)
struct DePredBatchArgs {
  DePredArgs a;      // params [nens, E, P], x_mul / x_add [nens, dc], y_mean / y_std [nens, O]; mu / var [nens O, m]
  int nens, nsamp;
  const float *xi;   // [nsamp, m, nens O] or NULL: Philox pairs keyed by (seed, counter), element q takes half q % 2 of q / 2
  float *ysamp;      // [nsamp, m, nens O]
  uint64_t seed, counter;
};

__global__ void __launch_bounds__(DE_PRED_THREADS) de_predict_batch_kernel(const __grid_constant__ DeNet net,
                                                                           const __grid_constant__ DePredBatchArgs ba) {
  extern __shared__ float smem[];
  const int O = net.O, B = DE_TM, r0 = blockIdx.x * DE_TM, b = blockIdx.y, ne = ba.a.E;
  const DeSmem s = de_carve(net, smem, B);
  DePredArgs a = ba.a;
  a.params += (size_t)b * ne * net.P;
  if (a.x_mul) {
    a.x_mul += b * net.dc;
    a.x_add += b * net.dc;
  }
  a.y_mean += b * O;
  a.y_std += b * O;
  float *mus = s.red + DE_SCRATCH, *s2s = mus + ne * B * O;
  de_member_heads(net, a, s, r0, 0, ne, mus, s2s);
  const int64_t m = a.m, KO = (int64_t)ba.nens * O;
  for (int i = threadIdx.x; i < B * O; i += blockDim.x) {
    const int p = i / O, o = i % O, row = r0 + p;
    if (row >= a.m) continue;
    float mean, v;
    de_combine(net, mus, s2s, ne, i, false, mean, v);
    const float sd = a.y_std[o];
    const float py = __fadd_rn(__fmul_rn(mean, sd), a.y_mean[o]), ps2 = __fmul_rn(v, __fmul_rn(sd, sd));
    const int64_t col = (int64_t)b * O + o;
    a.mu[col * m + row] = py;
    a.var[col * m + row] = ps2;
    const float ps = __fsqrt_rn(ps2);
    for (int t = 0; t < ba.nsamp; ++t) {
      const int64_t q = ((int64_t)t * m + row) * KO + col;
      float z;
      if (ba.xi) {
        z = ba.xi[q];
      } else {
        float z0, z1;
        philox_normal2(ba.seed, (uint64_t)(q >> 1), ba.counter, z0, z1);
        z = (q & 1) ? z1 : z0;
      }
      ba.ysamp[q] = __fadd_rn(py, __fmul_rn(ps, z));
    }
  }
}

// W of members e0 + blockIdx.x for one Gumbel predict call: uniforms from sel.draws [E, r, dx] or Philox keyed by
// (seed, counter, member), so every candidate tile of the call uses the same W
__global__ void __launch_bounds__(DE_PRED_THREADS) gb_weights_kernel(const float *params, int P, int e0,
                                                                     const __grid_constant__ DeSel sel) {
  const int e = e0 + blockIdx.x, wsz = sel.r * sel.dx;
  gb_build_w(params + (size_t)e * P + sel.off, sel.r, sel.dx, sel.T, sel.w + (size_t)e * wsz, [&](int j, int k) {
    const int q = j * sel.dx + k;
    const uint64_t stream = ((uint64_t)GB_TAG_EVAL << 32) | ((uint32_t)e << 16) | (uint32_t)(q >> 1);
    return sel.draws ? sel.draws[(size_t)e * wsz + q] : fe_draw<1 + HB_FE_CONCRETE>(sel.seed, sel.counter, stream, q & 1);
  });
}

// ------------------------------------------------------------------------------------------------ launchers
// A member's layout and selection constants: BaseNet's; FeNet's, BaseNet's with the gate [din] last; or GumbelNet's,
// BaseNet's over the selected width (num_cont -> r when num_cont > 0) with the logits [r, num_cont] last.  GumbelNet's
// random prior net keeps the original width, so it only runs when r = num_cont or there are no numeric columns; anything
// else is rejected (the reference fails with a shape error in forward).
static bool de_sel_layout(const hb_de_spec_t *spec, const DeVariant &v, DeNet &net, DeSel &sel) {
  sel = DeSel{};
  if (v.kind == DeVariant::GUMBEL) {
    if (!spec || v.r < 1 || v.r > HB_DE_MAX_IN || spec->num_cont < 0 || spec->num_cont > HB_DE_MAX_IN || !(v.T > 0.0f))
      return false;
    const int dx = spec->num_cont;
    if (spec->rand_prior && dx > 0 && v.r != dx) return false;
    hb_de_spec_t narrow = *spec;
    if (dx > 0) narrow.num_cont = (int32_t)v.r;
    if (!de_layout(&narrow, net)) return false;
    sel.gate = DE_GUMBEL;
    sel.off = net.P;
    sel.T = v.T;
    sel.dx = dx;
    sel.r = dx > 0 ? (int)v.r : 0;      // without numeric columns the logits [r, 0] are empty and nothing is drawn
    sel.x_ld = dx > 0 ? (dx | 1) : 0;
    net.P += sel.r * dx;
    return true;
  }
  if (!de_layout(spec, net)) return false;
  sel.off = net.P;
  if (v.kind == DeVariant::GATED) {
    const hb_fe_gate_t *g = v.gate;
    if (!g || g->kind < HB_FE_STG || g->kind > HB_FE_HARD_CONCRETE || !(g->temperature > 0.0f)) return false;
    sel.gate = 1 + g->kind;
    sel.T = g->temperature;
    sel.t0 = g->start_temp;
    sel.t1 = g->end_temp;
    sel.tb = g->anneal_base;
    net.P += net.din;
  }
  return true;
}

// floats of a fit's per-row buffers of B rows: BaseNet's, plus a gate's unmasked inputs and gate states (B in_ld each)
// or a Gumbel selection's numeric rows (B x_ld)
static int64_t de_fit_rows_floats(const DeNet &net, const DeSel &sel, int64_t B) {
  const int64_t extra = sel.gate == DE_GUMBEL ? B * sel.x_ld : sel.gate != 0 ? 2 * B * net.in_ld : 0;
  return de_rows_floats(net, B) + extra;
}

// a predict tile's shared floats after the combination's: a gate's eval mask [din] or a Gumbel tile's numeric rows
static int64_t de_predict_sel_floats(const DeNet &net, const DeSel &sel) {
  return sel.gate == DE_GUMBEL ? (int64_t)DE_TM * sel.x_ld : sel.gate != 0 ? net.din : 0;
}

// a fit's workspace: Adam's exp_avg, exp_avg_sq and the last step's gradient, [E, P] each, then Gumbel's W [E, r, dx]
static int64_t de_fit_ws_bytes(const DeNet &net, const DeSel &sel, int64_t E) {
  return (3 * E * (int64_t)net.P + E * (int64_t)sel.r * sel.dx) * (int64_t)sizeof(float);
}

// The minibatches of a fit over n rows: B rows a step and nb steps an epoch (drop_last: a partial last minibatch is
// dropped, deep_ensemble.py:154; otherwise it is trained, gumbel_linear.py:72), the Feistel half-width h of the epoch's
// order of n, and coef = fp32 (1 / (n num_out)) * l1
struct DeFitShape {
  int B, nb, h;
  float coef;
};

static DeFitShape de_fit_shape(int64_t n, int64_t batch_size, bool drop_last, int O, float l1) {
  DeFitShape f;
  const int64_t B = n > batch_size ? batch_size : n;
  f.B = (int)B;
  f.nb = (int)(!drop_last ? (n + B - 1) / B : n > batch_size ? n / batch_size : 1);
  f.h = 1;
  while ((int64_t(1) << (2 * f.h)) < n) ++f.h;
  f.coef = (1.0f / (float)(n * O)) * l1;
  return f;
}

// every variant's kernel instance, indexed by GATE
static_assert(HB_FE_STG == 0 && HB_FE_CONCRETE == 1 && HB_FE_HARD_CONCRETE == 2, "GATE 0 .. DE_GUMBEL indexes the tables");
static decltype(&de_fit_kernel<0>) const DE_FIT_KERNELS[] = {de_fit_kernel<0>, de_fit_kernel<1 + HB_FE_STG>,
                                                              de_fit_kernel<1 + HB_FE_CONCRETE>,
                                                              de_fit_kernel<1 + HB_FE_HARD_CONCRETE>, de_fit_kernel<DE_GUMBEL>};
static decltype(&de_predict_kernel<false>) const DE_PREDICT_KERNELS[] = {
    de_predict_kernel<false>, de_predict_kernel<false, 1 + HB_FE_STG>, de_predict_kernel<false, 1 + HB_FE_CONCRETE>,
    de_predict_kernel<false, 1 + HB_FE_HARD_CONCRETE>, de_predict_kernel<false, DE_GUMBEL>};

int64_t de_num_params(const hb_de_spec_t *spec, const DeVariant &v) {
  DeNet net;
  DeSel sel;
  return de_sel_layout(spec, v, net, sel) ? net.P : -1;
}

int64_t de_fit_ws_query(const hb_de_spec_t *spec, const DeVariant &v, int64_t E) {
  DeNet net;
  DeSel sel;
  if (!de_sel_layout(spec, v, net, sel) || E < 1 || E > HB_DE_MAX_MEMBERS) return -1;
  return de_fit_ws_bytes(net, sel, E);
}

int launch_de_fit(const float *Xc, const int32_t *Xe, const float *y, int64_t n, const hb_de_spec_t *spec, const DeVariant &v,
                  int64_t E, float *params, double lr, float l1, int64_t batch_size, int64_t num_epochs, const int32_t *perm,
                  const float *draws, uint64_t seed, float *losses, void *ws, int64_t ws_bytes, cudaStream_t st) {
  DeNet net;
  DeSel sel;
  if (!de_sel_layout(spec, v, net, sel) || E < 1 || E > HB_DE_MAX_MEMBERS || n < 1 || n > (1 << 30) || batch_size < 1 ||
      num_epochs < 0)
    return HB_ERR_INVALID;
  if (!y || !params || !ws || (num_epochs > 0 && !losses) || (net.dc > 0 && !Xc) || (net.ne > 0 && !Xe)) return HB_ERR_INVALID;
  if (ws_bytes < de_fit_ws_bytes(net, sel, E)) return HB_ERR_INVALID;
  const DeFitShape f = de_fit_shape(n, batch_size, sel.gate != DE_GUMBEL, net.O, l1);
  if (de_fit_rows_floats(net, sel, f.B) > HB_DE_MAX_BATCH_FLOATS) return HB_ERR_INVALID;
  if (num_epochs == 0) return HB_OK;
  DeFitArgs a;
  a.Xc = Xc;
  a.Xe = Xe;
  a.y = y;
  a.perm = perm;
  a.params = params;
  a.m1 = (float *)ws;
  a.m2 = a.m1 + E * net.P;
  a.grad = a.m2 + E * net.P;
  a.losses = losses;
  a.n = (int)n;
  a.B = f.B;
  a.nb = f.nb;
  a.epochs = (int)num_epochs;
  a.h = f.h;
  a.seed = seed;
  a.lr = lr;
  a.coef = f.coef;
  if (v.kind == DeVariant::GATED)      // mask_loss only when Xc.shape[1] > 0
    sel.mcoef = net.dc > 0 ? (1.0f / (float)(n * net.O)) * v.gate->mask_reg : 0.0f;
  if (sel.gate == DE_GUMBEL) sel.w = a.grad + E * net.P;
  sel.draws = draws;
  const size_t smem = (size_t)(de_fit_rows_floats(net, sel, f.B) + DE_SCRATCH) * sizeof(float);
  const auto kernel = DE_FIT_KERNELS[sel.gate];
  HB_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  kernel<<<(unsigned)E, DE_FIT_THREADS, smem, st>>>(net, a, sel);
  count_launches(1);
  HB_LAUNCH_CHECK("de_fit_kernel");
  return HB_OK;
}

int launch_de_predict(const float *Xs, const int32_t *Xe, int64_t m, const hb_de_spec_t *spec, const DeVariant &v, int64_t E,
                      const float *params, const float *x_mul, const float *x_add, const float *y_mean, const float *y_std,
                      int32_t member, const float *draws, uint64_t seed, uint64_t counter, float *mu, float *var,
                      float *dmu, float *dvar, void *ws, int64_t ws_bytes, cudaStream_t st) {
  DeNet net;
  DeSel sel;
  if (!de_sel_layout(spec, v, net, sel) || E < 1 || E > HB_DE_MAX_MEMBERS || m < 0 || m > (int64_t(1) << 31) - DE_TM)
    return HB_ERR_INVALID;
  if (member < -1 || member >= E) return HB_ERR_INVALID;
  const bool grad = dmu != nullptr;
  if (!params || !y_mean || !y_std || !mu || (member < 0 && !var) || (net.ne > 0 && !Xe)) return HB_ERR_INVALID;
  if (net.dc > 0 && (!Xs || !x_mul || !x_add)) return HB_ERR_INVALID;
  if (sel.dx > 0 && (!ws || ws_bytes < E * (int64_t)sel.r * sel.dx * (int64_t)sizeof(float))) return HB_ERR_INVALID;
  if (grad && (!dvar || net.dc < 1 || member >= 0 || sel.gate != 0)) return HB_ERR_INVALID;
  if (m == 0) return HB_OK;
  DePredArgs a;
  a.Xs = Xs;
  a.Xe = Xe;
  a.params = params;
  a.x_mul = x_mul;
  a.x_add = x_add;
  a.y_mean = y_mean;
  a.y_std = y_std;
  a.mu = mu;
  a.var = var;
  a.dmu = dmu;
  a.dvar = dvar;
  a.m = (int)m;
  a.E = (int)E;
  a.member = member;
  sel.draws = draws;
  sel.seed = seed;
  sel.counter = counter;
  sel.w = (float *)ws;
  const int64_t ne = member >= 0 ? 1 : E;
  if (sel.dx > 0) {
    gb_weights_kernel<<<(unsigned)ne, DE_PRED_THREADS, 0, st>>>(params, net.P, member >= 0 ? member : 0, sel);
    count_launches(1);
    HB_LAUNCH_CHECK("gb_weights_kernel");
  }
  const size_t smem = (size_t)(de_rows_floats(net, DE_TM) + DE_SCRATCH + (2 * ne + 1) * DE_TM * net.O +
                               de_predict_sel_floats(net, sel)) * sizeof(float);
  const auto kernel = grad ? de_predict_kernel<true> : DE_PREDICT_KERNELS[sel.gate];
  HB_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  kernel<<<(unsigned)ceil_div(m, DE_TM), DE_PRED_THREADS, smem, st>>>(net, a, sel);
  count_launches(1);
  HB_LAUNCH_CHECK("de_predict_kernel");
  return HB_OK;
}

int launch_de_fit_batch(const float *Xc, const int32_t *Xe, const float *y, const int64_t *off, int64_t nens,
                        const hb_de_spec_t *spec, int64_t E, float *params, double lr, float l1, int64_t batch_size,
                        int64_t num_epochs, const uint64_t *seeds, float *losses, void *ws, int64_t ws_bytes, cudaStream_t st) {
  DeNet net;
  if (!de_layout(spec, net) || E < 1 || E > HB_DE_MAX_MEMBERS || nens < 1 || nens > HB_MAX_OUTPUTS || batch_size < 1 ||
      num_epochs < 0)
    return HB_ERR_INVALID;
  if (!off || !seeds || !y || !params || !ws || (num_epochs > 0 && !losses) || (net.dc > 0 && !Xc) || (net.ne > 0 && !Xe))
    return HB_ERR_INVALID;
  if (ws_bytes < nens * de_fit_ws_bytes(net, DeSel{}, E)) return HB_ERR_INVALID;
  DeFitBatchArgs ba{};
  int64_t Bmax = 0;
  if (off[0] < 0) return HB_ERR_INVALID;
  for (int64_t b = 0; b < nens; ++b) {
    const int64_t n = off[b + 1] - off[b];
    if (n < 1 || n > (1 << 30)) return HB_ERR_INVALID;
    const DeFitShape f = de_fit_shape(n, batch_size, true, net.O, l1);
    DeFitSlot &sl = ba.slot[b];
    sl.off = off[b];
    sl.seed = seeds[b];
    sl.coef = f.coef;
    sl.n = (int)n;
    sl.B = f.B;
    sl.nb = f.nb;
    sl.h = f.h;
    Bmax = f.B > Bmax ? f.B : Bmax;
  }
  if (de_rows_floats(net, Bmax) > HB_DE_MAX_BATCH_FLOATS) return HB_ERR_INVALID;
  if (num_epochs == 0) return HB_OK;
  DeFitArgs &a = ba.a;
  a.Xc = Xc;
  a.Xe = Xe;
  a.y = y;
  a.perm = nullptr;
  a.params = params;
  a.m1 = (float *)ws;
  a.losses = losses;
  a.epochs = (int)num_epochs;
  a.lr = lr;
  ba.E = (int)E;
  const size_t smem = (size_t)(de_rows_floats(net, Bmax) + DE_SCRATCH) * sizeof(float);
  HB_CUDA(cudaFuncSetAttribute(de_fit_batch_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  de_fit_batch_kernel<<<(unsigned)(nens * E), DE_FIT_THREADS, smem, st>>>(net, ba);
  count_launches(1);
  HB_LAUNCH_CHECK("de_fit_batch_kernel");
  return HB_OK;
}

int launch_de_predict_batch(const float *Xs, const int32_t *Xe, int64_t m, const hb_de_spec_t *spec, int64_t nens, int64_t E,
                            const float *params, const float *x_mul, const float *x_add, const float *y_mean,
                            const float *y_std, float *mu, float *var, int64_t n_samples, const float *xi, uint64_t seed,
                            uint64_t counter, float *y_samp, cudaStream_t st) {
  DeNet net;
  if (!de_layout(spec, net) || E < 1 || E > HB_DE_MAX_MEMBERS || nens < 1 || nens > HB_MAX_OUTPUTS || m < 0 ||
      m > (int64_t(1) << 31) - DE_TM || n_samples < 0 || n_samples > (int64_t(1) << 31))
    return HB_ERR_INVALID;
  if (!params || !y_mean || !y_std || !mu || !var || (net.ne > 0 && !Xe) || (n_samples > 0 && !y_samp)) return HB_ERR_INVALID;
  if (net.dc > 0 && (!Xs || !x_mul || !x_add)) return HB_ERR_INVALID;
  if (m == 0) return HB_OK;
  DePredBatchArgs ba{};
  DePredArgs &a = ba.a;
  a.Xs = Xs;
  a.Xe = Xe;
  a.params = params;
  a.x_mul = x_mul;
  a.x_add = x_add;
  a.y_mean = y_mean;
  a.y_std = y_std;
  a.mu = mu;
  a.var = var;
  a.m = (int)m;
  a.E = (int)E;
  a.member = -1;
  ba.nens = (int)nens;
  ba.nsamp = (int)n_samples;
  ba.xi = xi;
  ba.ysamp = y_samp;
  ba.seed = seed;
  ba.counter = counter;
  const size_t smem = (size_t)(de_rows_floats(net, DE_TM) + DE_SCRATCH + 2 * E * DE_TM * net.O) * sizeof(float);
  HB_CUDA(cudaFuncSetAttribute(de_predict_batch_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  de_predict_batch_kernel<<<dim3((unsigned)ceil_div(m, DE_TM), (unsigned)nens), DE_PRED_THREADS, smem, st>>>(net, ba);
  count_launches(1);
  HB_LAUNCH_CHECK("de_predict_batch_kernel");
  return HB_OK;
}

}  // namespace hb
