// Shared helpers for libhebo_b200 (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <math.h>
#include <type_traits>
#include "../../include/hebo_b200.h"

namespace hb {

constexpr int TILE = 128;      // GEMM / pairwise tile edge; all square work matrices are padded to it
constexpr int NB = 64;         // Cholesky panel width

__host__ __device__ inline int64_t round_up(int64_t x, int64_t m) { return (x + m - 1) / m * m; }
__host__ __device__ inline int64_t ceil_div(int64_t x, int64_t m) { return (x + m - 1) / m; }

// Per-DEVICE lazily built launch state: cudaFuncSetAttribute (dynamic shared memory opt-in) and occupancy queries apply
// to the CURRENT device only, and one process may drive several GPUs (GP(device='cuda:1') after 'cuda:0'), so every
// "first use" flag is kept per device.  slot(): current device index (or -1), *fresh = not initialised here yet.
constexpr int MAX_DEVICES = 64;
struct PerDevice {
  bool done[MAX_DEVICES] = {};
  int sms[MAX_DEVICES] = {};
  int aux[MAX_DEVICES] = {};
  int slot(bool *fresh) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= MAX_DEVICES) return -1;
    *fresh = !done[dev];
    return dev;
  }
};

void set_error(cudaError_t e, const char *where);
int check_launch(const char *where);
void count_launches(int n);            // bookkeeping for bench.py's gpu_launches claim
void prof_begin(cudaStream_t st);      // optional CUDA-event bracket around the dominant kernel
void prof_end(cudaStream_t st);

#define HB_CUDA(call)                                   \
  do {                                                  \
    cudaError_t _e = (call);                            \
    if (_e != cudaSuccess) {                            \
      hb::set_error(_e, #call);                         \
      return HB_ERR_CUDA;                               \
    }                                                   \
  } while (0)

#define HB_LAUNCH_CHECK(name)                           \
  do {                                                  \
    int _s = hb::check_launch(name);                    \
    if (_s != HB_OK) return _s;                         \
  } while (0)

// Kernel-template dispatch: calls f(kk) with kk = std::integral_constant<int, KERN> for the runtime kernel id, so a launch
// site names its instance as decltype(kk)::value.  An unknown id launches nothing and gives HB_ERR_INVALID.
template <class F> int with_kernel(int kern, F &&f) {
  switch (kern) {
    case HB_KERN_MATERN32: f(std::integral_constant<int, HB_KERN_MATERN32>{}); return HB_OK;
    case HB_KERN_MATERN52: f(std::integral_constant<int, HB_KERN_MATERN52>{}); return HB_OK;
    case HB_KERN_RBF:      f(std::integral_constant<int, HB_KERN_RBF>{}); return HB_OK;
    default: return HB_ERR_INVALID;
  }
}
// ... and f(kk, ee) for kernels templated on <KERN, EMB> as well, ee = std::bool_constant<emb>
template <class F> int with_kernel(int kern, bool emb, F &&f) {
  return with_kernel(kern, [&](auto kk) {
    if (emb) f(kk, std::true_type{});
    else f(kk, std::false_type{});
  });
}

// ---------------------------------------------------------------- stationary kernels
// k(r2) with unit outputscale.  KERN: 0 Matern-3/2, 1 Matern-5/2, 2 RBF (gpytorch MaternKernel/RBFKernel).
// The radius and the exponential go through the SFU (MUFU.RSQ / MUFU.EX2: r = r2 * rsqrt(r2), exp(x) = ex2(x log2 e),
// both ~2 ulp): the absolute error of k stays below ~1.5e-7 (it is largest where k ~ 1, i.e. no worse than the fp32
// rounding of k itself), and the per-pair instruction count of the K* / Gram builders drops by about a third compared
// with the IEEE sqrtf / expf sequences.  gram_kernel and kstar_kernel share these functions, so a candidate that
// duplicates a training row reproduces that row of K bit for bit (r2 = 0 gives k = 1 exactly).
__device__ __forceinline__ float fast_radius(float r2) {
  const float c = fmaxf(r2, 1e-30f);   // gpytorch: sqrt(clamp_min(sq_dist, 1e-30))
  float q;
  asm("rsqrt.approx.ftz.f32 %0, %1;" : "=f"(q) : "f"(c));   // c >= 1e-30 is a normal number: ftz changes nothing
  return c * q;
}
// exp(x) for x <= 0 as ex2(x log2 e); results below 2^-126 flush to zero (k ~ 1e-38 is zero for every purpose here)
__device__ __forceinline__ float fast_exp(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x * 1.4426950408889634f));
  return y;
}
template <int KERN>
__device__ __forceinline__ float kern_eval(float r2) {
  if (KERN == HB_KERN_RBF) return fast_exp(-0.5f * r2);
  const float r = fast_radius(r2);
  if (KERN == HB_KERN_MATERN32) {
    const float a = 1.7320508075688772f;
    float ar = a * r;
    return (1.0f + ar) * fast_exp(-ar);
  } else {
    const float a = 2.23606797749979f;
    float ar = a * r;
    return (1.0f + ar + (5.0f / 3.0f) * r2) * fast_exp(-ar);
  }
}

// k and the radial factor h with  dk/dl_k = h * dz_k^2 / l_k  (dz = lengthscale-scaled difference),
// SURVEY Appendix A.
template <int KERN>
__device__ __forceinline__ void kern_eval_grad(float r2, float &k, float &h) {
  if (KERN == HB_KERN_RBF) {
    k = fast_exp(-0.5f * r2);
    h = k;
    return;
  }
  const float r = fast_radius(r2);
  if (KERN == HB_KERN_MATERN32) {
    const float a = 1.7320508075688772f;
    float e = fast_exp(-a * r);
    k = (1.0f + a * r) * e;
    h = 3.0f * e;
  } else {
    const float a = 2.23606797749979f;
    float e = fast_exp(-a * r);
    k = (1.0f + a * r + (5.0f / 3.0f) * r2) * e;
    h = (5.0f / 3.0f) * (1.0f + a * r) * e;
  }
}

// Kumaraswamy-CDF input warp of a MinMax(-1,1)-scaled coordinate (BASELINE config 3; the reference's definitions are the
// torch layer KumarWarp, HEBO/hebo/models/nn/mono_layers/layers.py:85-117, and GPy's InputWarpedGP in gpy_wgp.py:120-128):
//   u = clamp((x + 1) / 2, eps, 1 - eps),  w = 1 - (1 - u^a)^b,  result 2 w - 1;   a, b in (0.01, 10)
// da / db (optional): partial derivatives of the RESULT w.r.t. the exponents.
constexpr float WARP_LO = 0.01f, WARP_HI = 10.0f;
__device__ __forceinline__ float kumar_warp(float x, float a, float b, float *da = nullptr, float *db = nullptr) {
  const float eps = 1e-6f;
  const float u = fminf(fmaxf((x + 1.0f) * 0.5f, eps), 1.0f - eps);
  const float lu = logf(u);
  const float t = expf(a * lu);             // u^a
  const float om = 1.0f - t;                // in (0, 1)
  const float lom = log1pf(-t);
  const float p = expf(b * lom);            // (1 - u^a)^b
  if (da) *da = 2.0f * b * expf((b - 1.0f) * lom) * t * lu;
  if (db) *db = -2.0f * p * lom;
  (void)om;
  return 2.0f * (1.0f - p) - 1.0f;
}

__device__ __forceinline__ float softplus_f(float u) {
  // torch.nn.functional.softplus (beta=1, threshold=20)
  return u > 20.0f ? u : log1pf(expf(u));
}
__device__ __forceinline__ float sigmoid_f(float u) { return 1.0f / (1.0f + expf(-u)); }

// pSGLD update of parameter i: torch.optim.RMSprop step followed by the Langevin term of HEBO/hebo/models/nn/sgld.py:57-70
// (xi == nullptr: no Langevin term)
__device__ __forceinline__ void psgld_update(float *raw, const float *grad, float *sq, int i, float lr, float a, float eps,
                                             float factor, const float *xi) {
  const float g = grad[i];
  const float v = a * sq[i] + (1.0f - a) * g * g;
  sq[i] = v;
  const float avg = sqrtf(v) + eps;
  float x = raw[i] - lr * g / avg;
  if (xi) x += factor * sqrtf(2.0f * lr / avg) * xi[i];
  raw[i] = x;
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// ---- Philox4x32-10 + Box-Muller: two N(0,1) draws per 64-bit counter `row` (the MACE epilogue's production noise and
// the in-kernel draws of hb_sample_y_batch)
__device__ __forceinline__ void philox_round(uint32_t (&c)[4], uint32_t k0, uint32_t k1) {
  const uint32_t M0 = 0xD2511F53u, M1 = 0xCD9E8D57u;
  const uint32_t hi0 = __umulhi(M0, c[0]), lo0 = M0 * c[0];
  const uint32_t hi1 = __umulhi(M1, c[2]), lo1 = M1 * c[2];
  const uint32_t n0 = hi1 ^ c[1] ^ k0, n1 = lo1, n2 = hi0 ^ c[3] ^ k1, n3 = lo0;
  c[0] = n0; c[1] = n1; c[2] = n2; c[3] = n3;
}
// stream: the upper half of the 128-bit Philox counter (0 for the MACE epilogue and hb_sample_y_batch)
__device__ __forceinline__ void philox_normal2(uint64_t seed, uint64_t row, uint64_t stream, float &z0, float &z1) {
  uint32_t c[4] = {(uint32_t)row, (uint32_t)(row >> 32), (uint32_t)stream, (uint32_t)(stream >> 32)};
  uint32_t k0 = (uint32_t)seed, k1 = (uint32_t)(seed >> 32);
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    philox_round(c, k0, k1);
    k0 += 0x9E3779B9u;
    k1 += 0xBB67AE85u;
  }
  const float u0 = ((float)c[0] + 0.5f) * 2.3283064365386963e-10f;   // (0,1)
  const float u1 = ((float)c[1] + 0.5f) * 2.3283064365386963e-10f;
  const float rad = sqrtf(-2.0f * logf(u0));
  float sn, cs;
  sincospif(2.0f * u1, &sn, &cs);
  z0 = rad * cs;
  z1 = rad * sn;
}
__device__ __forceinline__ void philox_normal2(uint64_t seed, uint64_t row, float &z0, float &z1) {
  philox_normal2(seed, row, 0, z0, z1);
}

// the duplicate predicate of the NSGA-II / GA survival (pymoo MixedVariableDuplicateElimination): |o[k] - me[k]| <= 1e-16f
// in every one of the D columns
__device__ __forceinline__ bool same_row(const float *o, const float *me, int D) {
  bool same = true;
  for (int k = 0; k < D && same; ++k) same = fabsf(o[k] - me[k]) <= 1e-16f;
  return same;
}

// lower-triangular tile index decode: t -> (I >= J), t = I*(I+1)/2 + J
__device__ __forceinline__ void tri_decode(int t, int &I, int &J) {
  int i = (int)((sqrtf(8.0f * (float)t + 1.0f) - 1.0f) * 0.5f);
  while (i * (i + 1) / 2 > t) --i;
  while ((i + 1) * (i + 2) / 2 <= t) ++i;
  I = i;
  J = t - i * (i + 1) / 2;
}

}  // namespace hb
