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

// y[p, j] = act(bias[j] + sum_k x[p, k] W[j, k]) (+ add[p, j]) for p < B, j < N; W [N, K] row-major (torch's layout).
// Lanes run over rows p, so W[j, k] is one broadcast load per warp.
__device__ void de_dense(const float *x, int ldx, int B, int K, const float *W, const float *bias, int N, float *y, int ldy,
                         bool relu, const float *add = nullptr, int ld_add = 0) {
  for (int idx = threadIdx.x; idx < B * N; idx += blockDim.x) {
    const int p = idx % B, j = idx / B;
    const float *xr = x + p * ldx;
    const float *wr = W + (size_t)j * K;
    float acc = 0.0f;
    for (int k = 0; k < K; ++k) acc = fmaf(xr[k], wr[k], acc);
    float v = acc + bias[j];
    if (relu) v = v < 0.0f ? 0.0f : v;
    if (add) v += add[p * ld_add + j];
    y[p * ldy + j] = v;
  }
}

// The input rows of s.rows: numeric columns (scaled as x * x_mul + x_add when x_mul is given), then the embedding rows
// or one-hot codes of the categorical columns.  A category outside 0 .. u - 1 loads NaN, so its row's outputs are NaN.
__device__ void de_load_inputs(const DeNet &net, const float *prm, const float *X, const int32_t *Xe, const float *x_mul,
                               const float *x_add, const DeSmem &s, int B) {
  for (int idx = threadIdx.x; idx < B * net.din; idx += blockDim.x) {
    const int p = idx / net.din, k = idx % net.din;
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
    s.xin[p * net.in_ld + k] = v;
  }
}

// BaseNet.forward (deep_ensemble.py:229-238) of the B rows in s.xin: prior net into s.pri (through d0 / d1), hidden
// activations into s.act, heads into s.head[p, 0:O] = mu (+ prior) and s.head[p, O:2O] = the sigma2 head's pre-softplus z.
__device__ void de_forward(const DeNet &net, const float *prm, const DeSmem &s, int B) {
  if (net.prior) {
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
  de_dense(src, ld, B, K, prm + net.mu_w, prm + net.mu_b, net.O, s.head, 2 * net.O, false, net.prior ? s.pri : nullptr, net.O);
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

// The whole fit of one member: a's pointers are its ensemble's (params [E, P], m1 / m2 / grad [E, P], losses [E, epochs])
__device__ __forceinline__ void de_fit_member(const DeNet &net, const DeFitArgs &a, int member, float *smem) {
  const int B = a.B, O = net.O;
  const DeSmem s = de_carve(net, smem, B);
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
    for (int bi = 0; bi < a.nb; ++bi) {
      ++step;
      for (int p = threadIdx.x; p < B; p += blockDim.x) {
        const int pos = bi * B + p;
        s.rows[p] = a.perm ? a.perm[((size_t)member * a.epochs + ep) * a.n + pos] : de_perm(pos, a.n, a.h, a.seed, ep, member);
      }
      __syncthreads();
      de_load_inputs(net, prm, a.Xc, a.Xe, nullptr, nullptr, s, B);
      __syncthreads();
      de_forward(net, prm, s, B);
      // the loss over the finite entries of y (loss_likelihood / loss_mse, deep_ensemble.py:140-149)
      if (threadIdx.x < 32) {
        float cnt = 0.0f;
        for (int i = threadIdx.x; i < B * O; i += 32) cnt += isfinite(a.y[(int64_t)s.rows[i / O] * O + i % O]) ? 1.0f : 0.0f;
        cnt = warp_sum(cnt);
        if (threadIdx.x == 0) s.red[0] = cnt;
      }
      __syncthreads();
      const float cnt = s.red[0];
      for (int i = threadIdx.x; i < B * O; i += blockDim.x) {
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
        for (int i = threadIdx.x; i < B * O; i += 32) sum += s.pri[i];
        sum = warp_sum(sum);
        if (threadIdx.x == 0) epoch_loss += sum / cnt * (float)B;      // epoch_loss += data_loss * bxc.shape[0]
      }
      float *dx = de_backward(net, prm, s, B, g, net.emb && net.ne > 0, net.dc);
      // embedding tables: the input delta of each row added into the row of its category, rows in batch order
      if (net.emb) {
        for (int c = 0; c < net.ne; ++c) {
          const int wc = net.col_w[c], tab = net.col_u[c] * wc;
          for (int idx = threadIdx.x; idx < tab; idx += blockDim.x) {
            const int u = idx / wc, q = idx % wc;
            float acc = 0.0f;
            for (int p = 0; p < B; ++p)
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
        const float gd = i < net.prior0 ? g[i] : 0.0f;
        const float gt = __fadd_rn(gd, __fmul_rn(a.coef, sg));
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

__global__ void __launch_bounds__(DE_FIT_THREADS) de_fit_kernel(const __grid_constant__ DeNet net, const DeFitArgs a) {
  extern __shared__ float smem[];
  de_fit_member(net, a, blockIdx.x, smem);
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

// CTA (b, member) = blockIdx.x = b E + member runs de_fit_kernel's member on ensemble b's slices
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
// into mus[e - e0][p, o] and, with output_noise, sigma2 into s2s[e - e0][p, o]
__device__ __forceinline__ void de_member_heads(const DeNet &net, const DePredArgs &a, const DeSmem &s, int r0, int e0,
                                                int e1, float *mus, float *s2s) {
  const int O = net.O, B = DE_TM;
  for (int p = threadIdx.x; p < B; p += blockDim.x) s.rows[p] = min(r0 + p, a.m - 1);
  __syncthreads();
  for (int e = e0; e < e1; ++e) {
    const float *prm = a.params + (size_t)e * net.P;
    de_load_inputs(net, prm, a.Xs, a.Xe, a.x_mul, a.x_add, s, B);
    __syncthreads();
    de_forward(net, prm, s, B);
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

template <bool GRAD>
__global__ void __launch_bounds__(DE_PRED_THREADS) de_predict_kernel(const __grid_constant__ DeNet net, const DePredArgs a) {
  extern __shared__ float smem[];
  const int O = net.O, B = DE_TM, r0 = blockIdx.x * DE_TM;
  const DeSmem s = de_carve(net, smem, B);
  const int e0 = a.member >= 0 ? a.member : 0, e1 = a.member >= 0 ? a.member + 1 : a.E, ne = e1 - e0;
  float *mus = s.red + DE_SCRATCH, *s2s = mus + ne * B * O, *py = s2s + ne * B * O;
  de_member_heads(net, a, s, r0, e0, e1, mus, s2s);
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

// ------------------------------------------------------------------------------------------------ launchers
int64_t de_num_params(const hb_de_spec_t *spec) {
  DeNet net;
  return de_layout(spec, net) ? net.P : -1;
}

int64_t de_fit_ws_query(const hb_de_spec_t *spec, int64_t E) {
  DeNet net;
  if (!de_layout(spec, net) || E < 1 || E > HB_DE_MAX_MEMBERS) return -1;
  return 3 * E * (int64_t)net.P * (int64_t)sizeof(float);
}

int launch_de_fit(const float *Xc, const int32_t *Xe, const float *y, int64_t n, const hb_de_spec_t *spec, int64_t E,
                  float *params, double lr, float l1, int64_t batch_size, int64_t num_epochs, const int32_t *perm,
                  uint64_t seed, float *losses, void *ws, int64_t ws_bytes, cudaStream_t st) {
  DeNet net;
  if (!de_layout(spec, net) || E < 1 || E > HB_DE_MAX_MEMBERS || n < 1 || n > (1 << 30) || batch_size < 1 || num_epochs < 0)
    return HB_ERR_INVALID;
  if (!y || !params || !ws || (num_epochs > 0 && !losses) || (net.dc > 0 && !Xc) || (net.ne > 0 && !Xe)) return HB_ERR_INVALID;
  const int64_t need = de_fit_ws_query(spec, E);
  if (ws_bytes < need) return HB_ERR_INVALID;
  const int64_t B = n > batch_size ? batch_size : n;     // drop_last = n > batch_size (deep_ensemble.py:154)
  if (de_rows_floats(net, B) > HB_DE_MAX_BATCH_FLOATS) return HB_ERR_INVALID;
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
  a.B = (int)B;
  a.nb = (int)(n > batch_size ? n / batch_size : 1);
  a.epochs = (int)num_epochs;
  int h = 1;
  while ((int64_t(1) << (2 * h)) < n) ++h;
  a.h = h;
  a.seed = seed;
  a.lr = lr;
  a.coef = (1.0f / (float)(n * net.O)) * l1;
  const size_t smem = (size_t)(de_rows_floats(net, B) + DE_SCRATCH) * sizeof(float);
  HB_CUDA(cudaFuncSetAttribute(de_fit_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  de_fit_kernel<<<(unsigned)E, DE_FIT_THREADS, smem, st>>>(net, a);
  count_launches(1);
  HB_LAUNCH_CHECK("de_fit_kernel");
  return HB_OK;
}

int launch_de_predict(const float *Xs, const int32_t *Xe, int64_t m, const hb_de_spec_t *spec, int64_t E, const float *params,
                      const float *x_mul, const float *x_add, const float *y_mean, const float *y_std, int32_t member,
                      float *mu, float *var, float *dmu, float *dvar, cudaStream_t st) {
  DeNet net;
  if (!de_layout(spec, net) || E < 1 || E > HB_DE_MAX_MEMBERS || m < 0 || m > (int64_t(1) << 31) - DE_TM) return HB_ERR_INVALID;
  if (member < -1 || member >= E) return HB_ERR_INVALID;
  const bool grad = dmu != nullptr;
  if (!params || !y_mean || !y_std || !mu || (member < 0 && !var) || (net.ne > 0 && !Xe)) return HB_ERR_INVALID;
  if (net.dc > 0 && (!Xs || !x_mul || !x_add)) return HB_ERR_INVALID;
  if (grad && (!dvar || net.dc < 1 || member >= 0)) return HB_ERR_INVALID;
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
  const int64_t ne = member >= 0 ? 1 : E;
  const size_t smem = (size_t)(de_rows_floats(net, DE_TM) + DE_SCRATCH + (2 * ne + 1) * DE_TM * net.O) * sizeof(float);
  const unsigned grid = (unsigned)ceil_div(m, DE_TM);
  if (grad) {
    HB_CUDA(cudaFuncSetAttribute(de_predict_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    de_predict_kernel<true><<<grid, DE_PRED_THREADS, smem, st>>>(net, a);
  } else {
    HB_CUDA(cudaFuncSetAttribute(de_predict_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    de_predict_kernel<false><<<grid, DE_PRED_THREADS, smem, st>>>(net, a);
  }
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
  if (ws_bytes < nens * de_fit_ws_query(spec, E)) return HB_ERR_INVALID;
  DeFitBatchArgs ba{};
  int64_t Bmax = 0;
  if (off[0] < 0) return HB_ERR_INVALID;
  for (int64_t b = 0; b < nens; ++b) {
    const int64_t n = off[b + 1] - off[b];
    if (n < 1 || n > (1 << 30)) return HB_ERR_INVALID;
    const int64_t B = n > batch_size ? batch_size : n;     // as launch_de_fit, per ensemble
    DeFitSlot &sl = ba.slot[b];
    sl.off = off[b];
    sl.seed = seeds[b];
    sl.coef = (1.0f / (float)(n * net.O)) * l1;
    sl.n = (int)n;
    sl.B = (int)B;
    sl.nb = (int)(n > batch_size ? n / batch_size : 1);
    int h = 1;
    while ((int64_t(1) << (2 * h)) < n) ++h;
    sl.h = h;
    Bmax = B > Bmax ? B : Bmax;
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
