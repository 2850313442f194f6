// Fused elementwise / reduction kernels of the guided step (sm_90a): CFG combine + score-guided DDIM update,
// add_noise, stand-alone top-1, and the motion-guidance loss with its closed-form gradient.
// All are HBM / launch-latency bound: 128-bit coalesced accesses, grid sized in multiples of the SM count.
#include <array>
#include <mutex>
#include <utility>

#include "mc_common.cuh"

namespace mc {

constexpr int kSMs = 132;  // H100 SXM

union Pack8 {
  uint4 u;
  __half h[8];
};

__device__ __forceinline__ uint4 ldg_nc_128(const void* p) {
  uint4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
               : "l"(p));
  return r;
}

// One element of utils/motionclone_functions.py:239 + :339-404 with every intermediate rounded to fp16, in the order
// the eager ATen kernels round (each binary op: fp32 opmath, fp16 result; h = round to fp16). The 0-dim fp32 CPU
// operands stay fp32, and `tensor / cpu_scalar` multiplies by the fp32 reciprocal. Per branch of the reference:
//   CFG combine (:239, only with eps_uncond):  e = h(ec + h(cfg * h(ec - eu)))
//   epsilon      (:340-341)  x0 = h(h(x - h(sb*e)) * inv_sa);            pe = e
//   sample       (:343-344)  x0 = e;                                     pe = h(h(x - h(sa*x0)) * inv_sb)
//   v_prediction (:346-347)  x0 = h(h(sa*x) - h(sb*e));                  pe = h(h(sa*e) + h(sb*x))
//   clip_sample  (:358-360)  x0 = h(min(max(x0, -r), r)) in fp32, NaN kept (clamp_scalar_kernel_impl)
//   use_clipped_model_output (:369)                                      pe = h(h(x - h(sa*x0)) * inv_sb)
//   score        (:382)      pe = h(pe - h(sc*g))
//   direction and sum (:386, :389)  xp = h(h(sap*x0) + h(c*pe)),  c = sqrt(1 - a_prev - std^2)
//   eta > 0      (:402-404)  xp = h(xp + h(std*noise))
// sb=sqrt(1-a_t), sa=sqrt(a_t), inv_* their fp32 reciprocals, sap=sqrt(a_prev), sc=guidance_scale*sqrt(1-a_t).
struct DdimCoef {
  float cfg, sb, inv_sa, sap, c, sc;
  float sa, inv_sb, clip, std;  // read by the sample / v_prediction / clip / re-derive / noise variants only
};

enum { kPredEpsilon = MC_DDIM_PRED_EPSILON, kPredSample = MC_DDIM_PRED_SAMPLE, kPredV = MC_DDIM_PRED_V };

template <int PRED, bool CLIP, bool REDERIVE, bool NOISE>
__device__ __forceinline__ __half ddim_one(__half ec, __half eu, bool has_u, __half x, __half g, bool has_g, __half nz,
                                           const DdimCoef& k, __half& x0_out) {
  const float fec = __half2float(ec);
  float e = fec;  // eps already combined by the caller (customized_step API) when there is no uncond operand
  if (has_u) {
    const float d = round_half(fec - __half2float(eu));         // cond - uncond
    const float m = round_half(k.cfg * d);                      // cfg * (...)
    e = round_half(fec + m);                                    // eps
  }
  float x0, e2;
  if constexpr (PRED == kPredEpsilon) {
    const float t1 = round_half(k.sb * e);                      // sqrt(1-a_t) * eps
    const float t2 = round_half(__half2float(x) - t1);          // x - ...
    x0 = round_half(t2 * k.inv_sa);                             // / sqrt(a_t)  (CUDA: * fp32 reciprocal)
    e2 = e;
  } else if constexpr (PRED == kPredSample) {
    x0 = e;
    const float t1 = round_half(k.sa * x0);                     // sqrt(a_t) * x0
    const float t2 = round_half(__half2float(x) - t1);
    e2 = round_half(t2 * k.inv_sb);                             // / sqrt(1-a_t)
  } else {
    const float xf = __half2float(x);
    x0 = round_half(round_half(k.sa * xf) - round_half(k.sb * e));
    e2 = round_half(round_half(k.sa * e) + round_half(k.sb * xf));
  }
  if constexpr (CLIP) {
    if (x0 == x0) x0 = round_half(fminf(fmaxf(x0, -k.clip), k.clip));
  }
  if constexpr (REDERIVE) {
    const float t1 = round_half(k.sa * x0);
    const float t2 = round_half(__half2float(x) - t1);
    e2 = round_half(t2 * k.inv_sb);
  }
  if (has_g) {
    const float g2 = round_half(k.sc * __half2float(g));        // guidance_scale*sqrt(1-a_t) * score
    e2 = round_half(e2 - g2);
  }
  const float dir = round_half(k.c * e2);                       // sqrt(1-a_prev-std^2) * eps'
  const float t3 = round_half(k.sap * x0);                      // sqrt(a_prev) * x0
  x0_out = __float2half_rn(x0);
  if constexpr (NOISE) {
    const float xp = round_half(t3 + dir);
    return __float2half_rn(xp + round_half(k.std * __half2float(nz)));  // + std * variance_noise
  }
  return __float2half_rn(t3 + dir);
}

// <epsilon, no clip, no re-derive, no noise, no x0 store> is the guided sampling loop's step; the other instantiations
// add only what their branch needs (noise: a fifth 128-bit load; WRITE_X0: a second 128-bit store of pred_original_sample).
template <int PRED, bool CLIP, bool REDERIVE, bool NOISE, bool WRITE_X0>
__global__ void __launch_bounds__(256) cfg_ddim_step_kernel(const __half* __restrict__ ec, const __half* __restrict__ eu,
                                                            const __half* __restrict__ x,
                                                            const __half* __restrict__ score, __half* __restrict__ out,
                                                            int64_t n, DdimCoef k, const __half* __restrict__ noise,
                                                            __half* __restrict__ x0_out) {
  const int64_t nvec = n / 8;
  const bool has_g = score != nullptr;
  const bool has_u = eu != nullptr;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < nvec; i += (int64_t)gridDim.x * blockDim.x) {
    Pack8 a, b, c, d, z, o, p;
    a.u = ldg_nc_128(ec + i * 8);
    if (has_u) b.u = ldg_nc_128(eu + i * 8);
    c.u = ldg_nc_128(x + i * 8);
    if (has_g) d.u = ldg_nc_128(score + i * 8);
    if constexpr (NOISE) z.u = ldg_nc_128(noise + i * 8);
#pragma unroll
    for (int j = 0; j < 8; ++j)
      o.h[j] = ddim_one<PRED, CLIP, REDERIVE, NOISE>(a.h[j], has_u ? b.h[j] : __half(), has_u, c.h[j],
                                                     has_g ? d.h[j] : __half(), has_g, NOISE ? z.h[j] : __half(), k,
                                                     p.h[j]);
    *reinterpret_cast<uint4*>(out + i * 8) = o.u;
    if constexpr (WRITE_X0) *reinterpret_cast<uint4*>(x0_out + i * 8) = p.u;
  }
  // tail (n % 8), one thread each
  const int64_t tail0 = nvec * 8;
  const int64_t ti = tail0 + blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (ti < n) {
    __half p;
    out[ti] = ddim_one<PRED, CLIP, REDERIVE, NOISE>(ec[ti], has_u ? eu[ti] : __half(), has_u, x[ti],
                                                    has_g ? score[ti] : __half(), has_g, NOISE ? noise[ti] : __half(), k,
                                                    p);
    if constexpr (WRITE_X0) x0_out[ti] = p;
  }
}

__global__ void __launch_bounds__(256) add_noise_kernel(const __half* __restrict__ x0, const __half* __restrict__ nz,
                                                        __half* __restrict__ out, int64_t n, float sa, float sb) {
  const int64_t nvec = n / 8;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < nvec; i += (int64_t)gridDim.x * blockDim.x) {
    Pack8 a, b, o;
    a.u = ldg_nc_128(x0 + i * 8);
    b.u = ldg_nc_128(nz + i * 8);
#pragma unroll
    for (int j = 0; j < 8; ++j)
      o.h[j] = __float2half_rn(round_half(sa * __half2float(a.h[j])) + round_half(sb * __half2float(b.h[j])));
    *reinterpret_cast<uint4*>(out + i * 8) = o.u;
  }
  const int64_t ti = nvec * 8 + blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (ti < n) out[ti] = __float2half_rn(round_half(sa * __half2float(x0[ti])) + round_half(sb * __half2float(nz[ti])));
}

// top-1 of fp16 rows of length L (8, 16 or 32): L/8 lanes per row, 128-bit loads, lowest index wins ties
template <int L>
__global__ void __launch_bounds__(256) top1_rows_kernel(const __half* __restrict__ probs, int64_t rows,
                                                        __half* __restrict__ val, uint8_t* __restrict__ idx) {
  constexpr int LPR = L / 8;  // lanes per row
  const int64_t gtid = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  const int64_t row = gtid / LPR;
  const int sub = (int)(gtid % LPR);
  float bv = -1.f;
  int bi = 0;
  if (row < rows) {
    Pack8 a;
    a.u = ldg_nc_128(probs + row * L + sub * 8);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float v = __half2float(a.h[j]);
      if (v > bv) {
        bv = v;
        bi = sub * 8 + j;
      }
    }
  }
#pragma unroll
  for (int off = 1; off < LPR; off <<= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, bv, off);
    const int oi = __shfl_xor_sync(0xffffffffu, bi, off);
    if (ov > bv || (ov == bv && oi < bi)) {
      bv = ov;
      bi = oi;
    }
  }
  if (row < rows && sub == 0) {
    val[row] = __float2half_rn(bv);
    idx[row] = (uint8_t)bi;
  }
}

// top-1 of fp16 rows of any other length L <= 32: one thread per row and 2-byte loads, since a row starts at row*L
// halves (any alignment); lowest index wins ties
__global__ void __launch_bounds__(256) top1_rows_any_kernel(const __half* __restrict__ probs, int64_t rows, int L,
                                                            __half* __restrict__ val, uint8_t* __restrict__ idx) {
  const int64_t row = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (row >= rows) return;
  const __half* p = probs + row * L;
  float bv = -1.f;
  int bi = 0;
  for (int j = 0; j < L; ++j) {
    const float v = __half2float(__ldg(p + j));
    if (v > bv) {
      bv = v;
      bi = j;
    }
  }
  val[row] = __float2half_rn(bv);
  idx[row] = (uint8_t)bi;
}

// out = a + b + bias[c] on channel-innermost (NHWC / token-major) fp16 tensors: the resnet's `input + conv2(...)`
// (models/resnet.py:209-211) with conv2's (and the shortcut conv's) bias folded in, one pass instead of three.
// Rounding: the eager graph rounds conv+bias to fp16, then the sum; here h(h(a + bias) + b).
__global__ void __launch_bounds__(256) bias_residual_add_kernel(const __half* __restrict__ a, const __half* __restrict__ b,
                                                                const __half* __restrict__ bias, __half* __restrict__ out,
                                                                int64_t nvec, int VC) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < nvec; i += (int64_t)gridDim.x * blockDim.x) {
    Pack8 x, y, z, o;
    x.u = ldg_nc_128(a + i * 8);
    y.u = ldg_nc_128(b + i * 8);
    z.u = *reinterpret_cast<const uint4*>(bias + (i % VC) * 8);
#pragma unroll
    for (int j = 0; j < 8; ++j)
      o.h[j] = __float2half_rn(round_half(__half2float(x.h[j]) + __half2float(z.h[j])) + __half2float(y.h[j]));
    *reinterpret_cast<uint4*>(out + i * 8) = o.u;
  }
}

// Up to kMaxLossModules guided modules, passed by value: 64 x 32 B + 4 B = 2 052 B of the 4 KB kernel parameter space,
// so no device-side pointer table and no host-to-device copy. 64 covers every temporal attention of the SD1.5 UNet (40)
// plus a mid-block motion module (2).
constexpr int kMaxLossModules = 64;
struct LossArgs {
  const __half* cur[kMaxLossModules];
  const __half* ref[kMaxLossModules];
  __half* dcur[kMaxLossModules];
  int64_t n[kMaxLossModules];
  int M;
};

__device__ __forceinline__ float block_sum(float v, float* red) {
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0) red[warp] = v;
  __syncthreads();
  float t = 0.f;
  if (warp == 0) {
    t = (lane < (int)(blockDim.x >> 5)) ? red[lane] : 0.f;
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) t += __shfl_xor_sync(0xffffffffu, t, off);
  }
  return t;  // valid in warp 0
}

// one CTA per module (deterministic tree); the last CTA to finish adds the per-module fp16 losses in module order
__global__ void __launch_bounds__(1024) motion_loss_fwd_kernel(LossArgs a, __half* __restrict__ per_module,
                                                               __half* __restrict__ total,
                                                               unsigned int* __restrict__ done_counter) {
  __shared__ float red[32];
  __shared__ bool last;
  const int m = blockIdx.x;
  const __half* cur = a.cur[m];
  const __half* ref = a.ref[m];
  const int64_t n = a.n[m];
  float s = 0.f;
  for (int64_t i = threadIdx.x; i < n; i += blockDim.x) {
    const float d = round_half(__half2float(cur[i]) - __half2float(ref[i]));  // F.mse_loss on half: (a-b) -> fp16
    s += round_half(d * d);                                                    // (...)^2 -> fp16, summed in fp32
  }
  const float tot = block_sum(s, red);
  if (threadIdx.x == 0) {
    per_module[m] = __float2half_rn(tot / (float)n);
    __threadfence();
    const unsigned int prev = atomicAdd(done_counter, 1u);
    last = (prev == (unsigned int)(gridDim.x - 1));
  }
  __syncthreads();
  if (last && threadIdx.x == 0) {
    __threadfence();
    float t = 0.f;
    for (int j = 0; j < a.M; ++j) t += __half2float(*((volatile __half*)per_module + j));
    *total = __float2half_rn(t);
    *done_counter = 0u;
  }
}

__global__ void __launch_bounds__(256) motion_loss_bwd_kernel(LossArgs a, const __half* __restrict__ gout) {
  const int m = blockIdx.y;
  const int64_t n = a.n[m];
  const float g = __half2float(*gout) * 2.f / (float)n;
  const __half* cur = a.cur[m];
  const __half* ref = a.ref[m];
  __half* dc = a.dcur[m];
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    dc[i] = __float2half_rn(g * (__half2float(cur[i]) - __half2float(ref[i])));
}

// Ticket word of the last-CTA reduction, ONE PER DEVICE (zero-initialised once, re-zeroed by the kernel). The loss kernels
// of one device must not run concurrently on two streams (the guided step issues them on one stream).
static unsigned int* loss_counter() {
  static unsigned int* ptrs[64] = {};
  static std::mutex mu;
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return nullptr;
  std::lock_guard<std::mutex> lock(mu);
  if (ptrs[dev] == nullptr) {
    if (cudaMalloc(&ptrs[dev], sizeof(unsigned int)) != cudaSuccess) return nullptr;
    cudaMemset(ptrs[dev], 0, sizeof(unsigned int));
  }
  return ptrs[dev];
}

static unsigned grid_for(int64_t nvec, int threads) {
  int64_t blocks = (nvec + threads - 1) / threads;
  const int64_t cap = (int64_t)kSMs * 8;
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  return (unsigned)blocks;
}

}  // namespace mc

using DdimStepKernel = void (*)(const __half*, const __half*, const __half*, const __half*, __half*, int64_t,
                                mc::DdimCoef, const __half*, __half*);

// row PRED of the variant table; column bits: 1 clip, 2 re-derive, 4 noise, 8 x0 store
template <int PRED, size_t... V>
static constexpr std::array<DdimStepKernel, sizeof...(V)> ddim_step_row(std::index_sequence<V...>) {
  return {mc::cfg_ddim_step_kernel<PRED, (V & 1) != 0, (V & 2) != 0, (V & 4) != 0, (V & 8) != 0>...};
}

static int launch_ddim_step(const char* what, int pred, unsigned variant, const void* eps_cond, const void* eps_uncond,
                            const void* x, const void* score, const void* noise, void* x_prev, void* pred_x0, int64_t n,
                            const mc::DdimCoef& k, void* stream) {
  using namespace mc;
  static constexpr std::array<DdimStepKernel, 16> table[3] = {
      ddim_step_row<kPredEpsilon>(std::make_index_sequence<16>()),
      ddim_step_row<kPredSample>(std::make_index_sequence<16>()),
      ddim_step_row<kPredV>(std::make_index_sequence<16>())};
  if (!eps_cond || !x || !x_prev || n <= 0) {
    set_error("%s: null pointer or n <= 0", what);
    return MC_E_INVALID;
  }
  const uintptr_t al = (uintptr_t)eps_cond | (uintptr_t)eps_uncond | (uintptr_t)x | (uintptr_t)x_prev |
                       (uintptr_t)score | (uintptr_t)noise | (uintptr_t)pred_x0;
  if (al & 15) {
    set_error("%s: pointers must be 16-byte aligned", what);
    return MC_E_INVALID;
  }
  table[pred][variant]<<<grid_for(n / 8 + 8, 256), 256, 0, (cudaStream_t)stream>>>(
      (const __half*)eps_cond, (const __half*)eps_uncond, (const __half*)x, (const __half*)score, (__half*)x_prev, n, k,
      (const __half*)noise, (__half*)pred_x0);
  count_launch();
  return check_launch(what);
}

extern "C" int mc_cfg_ddim_step(const void* eps_cond, const void* eps_uncond, const void* x, const void* score,
                                void* x_prev, int64_t n, float cfg_scale, float sqrt_beta_t, float inv_sqrt_alpha_t,
                                float sqrt_alpha_prev, float dir_coef, float score_coef, void* stream) {
  mc::DdimCoef k{cfg_scale, sqrt_beta_t, inv_sqrt_alpha_t, sqrt_alpha_prev, dir_coef, score_coef, 0.f, 0.f, 0.f, 0.f};
  return launch_ddim_step("cfg_ddim_step", MC_DDIM_PRED_EPSILON, 0u, eps_cond, eps_uncond, x, score, nullptr, x_prev,
                          nullptr, n, k, stream);
}

extern "C" int mc_ddim_step_ex(const void* eps_cond, const void* eps_uncond, const void* x, const void* score,
                               const void* noise, void* x_prev, void* pred_x0, int64_t n, int prediction_type, int flags,
                               float cfg_scale, float sqrt_beta_t, float inv_sqrt_alpha_t, float sqrt_alpha_prev,
                               float dir_coef, float score_coef, float sqrt_alpha_t, float inv_sqrt_beta_t,
                               float clip_range, float std_dev, void* stream) {
  using namespace mc;
  if (prediction_type < MC_DDIM_PRED_EPSILON || prediction_type > MC_DDIM_PRED_V) {
    set_error("ddim_step_ex: prediction_type=%d is not epsilon (0), sample (1) or v_prediction (2)", prediction_type);
    return MC_E_UNSUPPORTED;
  }
  if (flags & ~(MC_DDIM_CLIP_SAMPLE | MC_DDIM_REDERIVE_EPS)) {
    set_error("ddim_step_ex: unknown flag bits 0x%x", (unsigned)flags);
    return MC_E_UNSUPPORTED;
  }
  if ((flags & MC_DDIM_CLIP_SAMPLE) && !(clip_range >= 0.f)) {
    set_error("ddim_step_ex: clip_range must be >= 0 with MC_DDIM_CLIP_SAMPLE");
    return MC_E_INVALID;
  }
  if (!noise && std_dev != 0.f) {
    set_error("ddim_step_ex: std_dev=%g needs a noise tensor (NULL noise is not eta = 0)", (double)std_dev);
    return MC_E_INVALID;
  }
  const unsigned variant = ((flags & MC_DDIM_CLIP_SAMPLE) ? 1u : 0u) | ((flags & MC_DDIM_REDERIVE_EPS) ? 2u : 0u) |
                           (noise ? 4u : 0u) | (pred_x0 ? 8u : 0u);
  DdimCoef k{cfg_scale, sqrt_beta_t, inv_sqrt_alpha_t, sqrt_alpha_prev, dir_coef, score_coef,
             sqrt_alpha_t, inv_sqrt_beta_t, clip_range, std_dev};
  return launch_ddim_step("ddim_step_ex", prediction_type, variant, eps_cond, eps_uncond, x, score, noise, x_prev, pred_x0,
                          n, k, stream);
}

extern "C" int mc_add_noise(const void* x0, const void* noise, void* out, int64_t n, float sqrt_alpha,
                            float sqrt_one_minus_alpha, void* stream) {
  using namespace mc;
  if (!x0 || !noise || !out || n <= 0) {
    set_error("add_noise: null pointer or n <= 0");
    return MC_E_INVALID;
  }
  if (((uintptr_t)x0 | (uintptr_t)noise | (uintptr_t)out) & 15) {
    set_error("add_noise: pointers must be 16-byte aligned");
    return MC_E_INVALID;
  }
  add_noise_kernel<<<grid_for(n / 8 + 8, 256), 256, 0, (cudaStream_t)stream>>>((const __half*)x0, (const __half*)noise,
                                                                             (__half*)out, n, sqrt_alpha,
                                                                             sqrt_one_minus_alpha);
  count_launch();
  return check_launch("add_noise");
}

extern "C" int mc_top1_rows(const void* probs, int64_t rows, int L, void* top_val, uint8_t* top_idx, void* stream) {
  using namespace mc;
  if (!probs || !top_val || !top_idx || rows <= 0) {
    set_error("top1_rows: null pointer or rows <= 0");
    return MC_E_INVALID;
  }
  if (L < 1 || L > 32) {
    set_error("top1_rows: L=%d outside the supported range 1..32", L);
    return MC_E_UNSUPPORTED;
  }
  const int lpr = (L == 8 || L == 16 || L == 32) ? L / 8 : 1;  // lanes per row
  const int64_t threads = rows * lpr;
  const unsigned grid = (unsigned)((threads + 255) / 256);
  cudaStream_t st = (cudaStream_t)stream;
  if (L == 8)
    top1_rows_kernel<8><<<grid, 256, 0, st>>>((const __half*)probs, rows, (__half*)top_val, top_idx);
  else if (L == 16)
    top1_rows_kernel<16><<<grid, 256, 0, st>>>((const __half*)probs, rows, (__half*)top_val, top_idx);
  else if (L == 32)
    top1_rows_kernel<32><<<grid, 256, 0, st>>>((const __half*)probs, rows, (__half*)top_val, top_idx);
  else
    top1_rows_any_kernel<<<grid, 256, 0, st>>>((const __half*)probs, rows, L, (__half*)top_val, top_idx);
  count_launch();
  return check_launch("top1_rows");
}

static int fill_loss_args(mc::LossArgs& a, int M, const void* const* cur, const void* const* ref, const int64_t* n,
                          void* const* d_cur) {
  if (M <= 0 || M > mc::kMaxLossModules || !cur || !ref || !n) return MC_E_INVALID;
  a.M = M;
  for (int m = 0; m < M; ++m) {
    if (!cur[m] || !ref[m] || n[m] <= 0) return MC_E_INVALID;
    a.cur[m] = (const __half*)cur[m];
    a.ref[m] = (const __half*)ref[m];
    a.dcur[m] = d_cur ? (__half*)d_cur[m] : nullptr;
    a.n[m] = n[m];
  }
  return MC_OK;
}

extern "C" int mc_motion_loss_fwd(int M, const void* const* cur, const void* const* ref, const int64_t* n,
                                  void* loss_per_module, void* loss_total, void* stream) {
  using namespace mc;
  LossArgs a{};
  if (fill_loss_args(a, M, cur, ref, n, nullptr) != MC_OK || !loss_per_module || !loss_total) {
    set_error("motion_loss_fwd: bad arguments (1 <= M <= 64, non-null pointers, n > 0)");
    return MC_E_INVALID;
  }
  unsigned int* ctr = loss_counter();
  if (!ctr) {
    set_error("motion_loss_fwd: cudaMalloc of the completion counter failed");
    return MC_E_CUDA;
  }
  motion_loss_fwd_kernel<<<M, 1024, 0, (cudaStream_t)stream>>>(a, (__half*)loss_per_module, (__half*)loss_total, ctr);
  count_launch();
  return check_launch("motion_loss_fwd");
}

extern "C" int mc_motion_loss_bwd(int M, const void* const* cur, const void* const* ref, const int64_t* n,
                                  const void* d_loss_total, void* const* d_cur, void* stream) {
  using namespace mc;
  LossArgs a{};
  if (!d_cur || !d_loss_total || fill_loss_args(a, M, cur, ref, n, d_cur) != MC_OK) {
    set_error("motion_loss_bwd: bad arguments (1 <= M <= 64, non-null pointers, n > 0)");
    return MC_E_INVALID;
  }
  int64_t nmax = 0;
  for (int m = 0; m < M; ++m) nmax = n[m] > nmax ? n[m] : nmax;
  dim3 grid((unsigned)((nmax + 255) / 256 > 64 ? 64 : (nmax + 255) / 256), (unsigned)M);
  motion_loss_bwd_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(a, (const __half*)d_loss_total);
  count_launch();
  return check_launch("motion_loss_bwd");
}

extern "C" int mc_bias_residual_add(const void* a, const void* b, const void* bias, void* out, int64_t n, int C,
                                    void* stream) {
  using namespace mc;
  if (!a || !b || !bias || !out || n <= 0 || C <= 0) {
    set_error("bias_residual_add: null pointer or non-positive size");
    return MC_E_INVALID;
  }
  if (C % 8 != 0 || n % C != 0) {
    set_error("bias_residual_add: C must be a multiple of 8 and divide n (C=%d)", C);
    return MC_E_UNSUPPORTED;
  }
  bias_residual_add_kernel<<<grid_for(n / 8, 256), 256, 0, (cudaStream_t)stream>>>(
      (const __half*)a, (const __half*)b, (const __half*)bias, (__half*)out, n / 8, C / 8);
  count_launch();
  return check_launch("bias_residual_add");
}
