// Memory-bound glue of the UNet3D forward and of the guided pass's backward on token-major fp16 activations (sm_90a):
//   * LayerNorm over C (+ the temporal positional-encoding add)    (models/attention.py:189-212, motion_module.py:204-215,
//     :281-282), forward and input gradient
//   * GEGLU  h * gelu_erf(gate), forward and backward               (diffusers-0.16 FeedForward used at attention.py:211,
//     motion_module.py:209)
// GroupNorm lives in groupnorm.cu. Weights are frozen on this path (t2v_video_sample.py:67-68): input gradients only.
#include <math.h>
#include <stdlib.h>

#include "mc_common.cuh"

namespace mc {

union Vec8 {
  uint4 u;
  __half2 h2[4];
  __half h[8];
};

// ---------------------------------------------------------------------------------------------------------------
// LayerNorm over the last dim C (multiple of 8, <= 2048). Rows are contiguous, so a tile of TR consecutive rows is ONE
// 1-D bulk copy (TMA engine) into shared memory and one bulk store back: the bytes in flight per SM are set by the tile
// size and the number of resident CTAs (2 stages x ~20 KB x up to 5 CTAs), not by how many registers a warp can keep
// loaded - the register-only version of this kernel held 24 warps x 1.3 KB = 30 KB per SM in flight at C = 320 (80
// registers per thread) and measured 0.36-0.43 of the HBM peak. One warp per row, two-pass statistics in fp32 in the same
// summation order as before (per-lane sums, then the xor butterfly); the result overwrites the row in its stage.
// ---------------------------------------------------------------------------------------------------------------
template <int VPL>  // vectors (of 8 halfs) per lane
__global__ void __launch_bounds__(256) layernorm_kernel(const __half* __restrict__ x, __half* __restrict__ y,
                                                        const __half* __restrict__ gamma, const __half* __restrict__ beta,
                                                        const __half* __restrict__ post_add,
                                                        const __half* __restrict__ pre_bias, int rows_per_frame, int frames,
                                                        int64_t rows, int C, float eps, int TR, int64_t n_tiles) {
  extern __shared__ __align__(128) uint8_t ln_smem[];
  const uint32_t stage_bytes = (uint32_t)TR * C * 2;
  uint64_t* bars = reinterpret_cast<uint64_t*>(ln_smem + 2 * stage_bytes);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int V = C / 8;
  if (tid == 0) {
    mbar_init(bars, 1), mbar_init(bars + 1, 1);
    fence_mbar_init();
  }
  __syncthreads();
  auto tile_bytes = [&](int64_t t) {
    const int64_t r = rows - t * TR;
    return (uint32_t)((r < TR ? r : TR) * C * 2);
  };
  auto load_tile = [&](int64_t t, int st) {
    mbar_arrive_expect_tx(bars + st, tile_bytes(t));
    bulk_g2s(ln_smem + st * stage_bytes, x + t * TR * C, tile_bytes(t), bars + st);
  };
  // gamma, beta and the folded residual bias: staged once per CTA behind the two stages (3 x C halfs)
  __half* s_par = reinterpret_cast<__half*>(ln_smem + 2 * stage_bytes + 16);
  for (int v = tid; v < V; v += 256) {
    reinterpret_cast<uint4*>(s_par)[v] = *reinterpret_cast<const uint4*>(gamma + v * 8);
    reinterpret_cast<uint4*>(s_par + C)[v] = *reinterpret_cast<const uint4*>(beta + v * 8);
    reinterpret_cast<uint4*>(s_par + 2 * C)[v] =
        pre_bias ? *reinterpret_cast<const uint4*>(pre_bias + v * 8) : make_uint4(0u, 0u, 0u, 0u);
  }
  __syncthreads();
  int64_t tile = blockIdx.x;
  if (tid == 0 && tile < n_tiles) load_tile(tile, 0);
  for (int k = 0; tile < n_tiles; tile += gridDim.x, ++k) {
    const int st = k & 1;
    if (tid == 0 && tile + gridDim.x < n_tiles) {
      bulk_wait_read_all();  // the store that left the other stage one trip ago has read its bytes
      load_tile(tile + gridDim.x, st ^ 1);
    }
    mbar_wait(bars + st, (k >> 1) & 1);
    uint8_t* stage = ln_smem + st * stage_bytes;
    const int64_t row_base = tile * TR;
    const int live = (int)((rows - row_base) < TR ? (rows - row_base) : TR);
    for (int r = warp; r < live; r += 8) {
      __half* xr = reinterpret_cast<__half*>(stage) + (int64_t)r * C;
      Vec8 a[VPL];
      float s = 0.f;
#pragma unroll
      for (int i = 0; i < VPL; ++i) {
        const int v = lane + i * 32;
        a[i].u = make_uint4(0u, 0u, 0u, 0u);
        if (v < V) {
          a[i].u = *reinterpret_cast<const uint4*>(xr + v * 8);
          if (pre_bias) {  // x + pre_bias[c] (fp16, as a separate elementwise add would round it) is what gets normalised
            Vec8 pb;
            pb.u = reinterpret_cast<const uint4*>(s_par + 2 * C)[v];
#pragma unroll
            for (int j = 0; j < 4; ++j) a[i].h2[j] = __hadd2(a[i].h2[j], pb.h2[j]);
          }
        }
      }
#pragma unroll
      for (int i = 0; i < VPL; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) s += __half2float(a[i].h[j]);  // padding vectors are zeros
#pragma unroll
      for (int off = 16; off > 0; off >>= 1) s += __shfl_xor_sync(0xffffffffu, s, off);
      const float mean = s / (float)C;
      float q = 0.f;
#pragma unroll
      for (int i = 0; i < VPL; ++i) {
        if (lane + i * 32 < V) {
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            const float d = __half2float(a[i].h[j]) - mean;
            q += d * d;
          }
        }
      }
#pragma unroll
      for (int off = 16; off > 0; off >>= 1) q += __shfl_xor_sync(0xffffffffu, q, off);
      const float rstd = rsqrtf(q / (float)C + eps);
      const int64_t row = row_base + r;
      const __half* pa = post_add ? post_add + (int64_t)((row / rows_per_frame) % frames) * C : nullptr;
#pragma unroll
      for (int i = 0; i < VPL; ++i) {
        const int v = lane + i * 32;
        if (v < V) {
          Vec8 o, pe, w, bt;
          w.u = reinterpret_cast<const uint4*>(s_par)[v];
          bt.u = reinterpret_cast<const uint4*>(s_par + C)[v];
          if (pa) pe.u = *reinterpret_cast<const uint4*>(pa + v * 8);
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            float f = (__half2float(a[i].h[j]) - mean) * rstd * __half2float(w.h[j]) + __half2float(bt.h[j]);
            if (pa) f = round_half(f) + __half2float(pe.h[j]);  // eager: LayerNorm output (fp16) + pe (fp16)
            o.h[j] = __float2half_rn(f);
          }
          *reinterpret_cast<uint4*>(xr + v * 8) = o.u;
        }
      }
    }
    fence_proxy_async();  // the rows written above -> visible to the bulk-store engine
    __syncthreads();
    if (tid == 0) {
      bulk_s2g(y + row_base * C, stage, tile_bytes(tile));
      bulk_commit();
    }
  }
  if (tid == 0) bulk_wait_read_all();
}

// ---------------------------------------------------------------------------------------------------------------
// GEGLU: out[t, j] = fp16( h[t, j] * fp16(gelu_erf(gate[t, j])) ),  in = [T, 2I] = [h | gate]
// ---------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ float gelu_erf(float x) {
  return 0.5f * x * (1.f + erff(x * 0.70710678118654752440f));
}

__global__ void __launch_bounds__(256) geglu_kernel(const __half* __restrict__ in, __half* __restrict__ out, int64_t T,
                                                    int I) {
  const int VI = I / 8;
  const int64_t nvec = T * VI;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < nvec; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t t = i / VI;
    const int v = (int)(i % VI);
    const __half* row = in + t * 2 * I;
    Vec8 hh, gg, o;
    hh.u = *reinterpret_cast<const uint4*>(row + v * 8);
    gg.u = *reinterpret_cast<const uint4*>(row + I + v * 8);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float ge = round_half(gelu_erf(__half2float(gg.h[j])));  // F.gelu output is fp16 in the eager graph
      o.h[j] = __float2half_rn(__half2float(hh.h[j]) * ge);
    }
    *reinterpret_cast<uint4*>(out + i * 8) = o.u;
  }
}

// GEGLU through a lookup table. The erf-based kernel above is ISSUE-bound (~50 instructions per element: 127 us for the
// 503 MB of the C = 320 layers, where HBM needs 77 us). fp16 has only 65 536 values, so fp16(gelu_erf(gate)) is a table
// of 128 KB: built once per device with the SAME device code as geglu_kernel (bit-identical results), copied into shared
// memory by one persistent 1024-thread CTA per SM, and `h * gelu` becomes one HMUL2 per pair (the product of two fp16
// numbers is exact in fp32, so HMUL2's single rounding equals the eager fp32-multiply-then-round).
__device__ __half g_gelu_lut[65536];

__global__ void gelu_lut_init_kernel() {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const __half x = __ushort_as_half((unsigned short)i);
  g_gelu_lut[i] = __float2half_rn(gelu_erf(__half2float(x)));
}

__global__ void __launch_bounds__(1024) geglu_lut_kernel(const __half* __restrict__ in, __half* __restrict__ out, int64_t T,
                                                         int I) {
  extern __shared__ __align__(16) unsigned short s_lut[];  // 65536 entries
  {
    const uint4* src = reinterpret_cast<const uint4*>(g_gelu_lut);
    uint4* dst = reinterpret_cast<uint4*>(s_lut);
    for (int i = threadIdx.x; i < 65536 / 8; i += blockDim.x) dst[i] = src[i];
  }
  __syncthreads();
  const int VI = I / 8;
  const int64_t nvec = T * VI;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  auto gate_mul = [&](const Vec8& hh, const Vec8& gg) {
    uint32_t r[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const unsigned lo = s_lut[__half_as_ushort(gg.h[2 * k])], hi = s_lut[__half_as_ushort(gg.h[2 * k + 1])];
      const unsigned packed = lo | (hi << 16);
      const __half2 prod = __hmul2(hh.h2[k], *reinterpret_cast<const __half2*>(&packed));
      r[k] = *reinterpret_cast<const uint32_t*>(&prod);
    }
    return make_uint4(r[0], r[1], r[2], r[3]);
  };
  int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  for (; i + stride < nvec; i += 2 * stride) {  // two vectors per trip: 4 x 16 B in flight per thread
    const int64_t i1 = i + stride;
    const int64_t t0 = i / VI, t1 = i1 / VI;
    const int v0 = (int)(i - t0 * VI), v1 = (int)(i1 - t1 * VI);
    Vec8 h0, g0, h1, g1;
    h0.u = *reinterpret_cast<const uint4*>(in + t0 * 2 * I + v0 * 8);
    g0.u = *reinterpret_cast<const uint4*>(in + t0 * 2 * I + I + v0 * 8);
    h1.u = *reinterpret_cast<const uint4*>(in + t1 * 2 * I + v1 * 8);
    g1.u = *reinterpret_cast<const uint4*>(in + t1 * 2 * I + I + v1 * 8);
    *reinterpret_cast<uint4*>(out + i * 8) = gate_mul(h0, g0);
    *reinterpret_cast<uint4*>(out + i1 * 8) = gate_mul(h1, g1);
  }
  if (i < nvec) {
    const int64_t t0 = i / VI;
    const int v0 = (int)(i - t0 * VI);
    Vec8 h0, g0;
    h0.u = *reinterpret_cast<const uint4*>(in + t0 * 2 * I + v0 * 8);
    g0.u = *reinterpret_cast<const uint4*>(in + t0 * 2 * I + I + v0 * 8);
    *reinterpret_cast<uint4*>(out + i * 8) = gate_mul(h0, g0);
  }
}

static bool g_gelu_lut_ready[64] = {};

}  // namespace mc

extern "C" int mc_layernorm(const void* x, void* y, const void* gamma, const void* beta, const void* post_add,
                            const void* pre_bias, int rows_per_frame, int frames, int64_t rows, int C, float eps,
                            void* stream) {
  using namespace mc;
  if (!x || !y || !gamma || !beta || rows <= 0) {
    set_error("layernorm: null pointer or rows <= 0");
    return MC_E_INVALID;
  }
  if (C % 8 != 0 || C > 2048) {
    set_error("layernorm: need C %% 8 == 0 and C <= 2048 (got %d)", C);
    return MC_E_UNSUPPORTED;
  }
  if (post_add != nullptr && (rows_per_frame <= 0 || frames <= 0)) {
    set_error("layernorm: post_add needs rows_per_frame > 0 and frames > 0");
    return MC_E_INVALID;
  }
  if (((uintptr_t)x | (uintptr_t)y | (uintptr_t)gamma | (uintptr_t)beta | (uintptr_t)post_add | (uintptr_t)pre_bias) % 16) {
    set_error("layernorm: pointers must be 16-byte aligned");
    return MC_E_INVALID;
  }
  // rows per tile: ~20 KB stages (C = 320 -> 32 rows, 640 -> 16, 1280 -> 8), at most 4 rows per warp
  int rw = 20480 / (C * 2 * 8);
  rw = rw < 1 ? 1 : (rw > 4 ? 4 : rw);
  const int TR = 8 * rw;
  const int64_t n_tiles = (rows + TR - 1) / TR;
  const size_t smem = 2 * (size_t)TR * C * 2 + 16 + 3 * (size_t)C * 2;
  int per_sm = (int)((227 * 1024) / (smem + 1024));
  per_sm = per_sm > 8 ? 8 : per_sm;
  int64_t blocks = n_tiles < (int64_t)132 * per_sm ? n_tiles : (int64_t)132 * per_sm;
  cudaStream_t st = (cudaStream_t)stream;
  const int vpl = (C / 8 + 31) / 32;
#define MC_LN(V)                                                                                                   \
  do {                                                                                                             \
    cudaFuncSetAttribute(layernorm_kernel<V>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);             \
    layernorm_kernel<V><<<(unsigned)blocks, 256, smem, st>>>((const __half*)x, (__half*)y, (const __half*)gamma,   \
                                                             (const __half*)beta, (const __half*)post_add,        \
                                                             (const __half*)pre_bias, rows_per_frame, frames, rows, C, \
                                                             eps, TR, n_tiles);                                    \
  } while (0)
  switch (vpl) {
    case 1: MC_LN(1); break;
    case 2: MC_LN(2); break;
    case 3: MC_LN(3); break;
    case 4: MC_LN(4); break;
    case 5: MC_LN(5); break;
    case 6: MC_LN(6); break;
    case 7: MC_LN(7); break;
    default: MC_LN(8); break;
  }
#undef MC_LN
  count_launch();
  return check_launch("layernorm");
}

extern "C" int mc_geglu(const void* in, void* out, int64_t T, int I, void* stream) {
  using namespace mc;
  if (!in || !out || T <= 0 || I <= 0) {
    set_error("geglu: null pointer or non-positive dims");
    return MC_E_INVALID;
  }
  if (I % 8 != 0) {
    set_error("geglu: inner dim must be a multiple of 8 (got %d)", I);
    return MC_E_UNSUPPORTED;
  }
  const int64_t nvec = T * (I / 8);
  cudaStream_t st = (cudaStream_t)stream;
  int dev = 0, sms = 132;
  if (nvec >= (int64_t)1 << 20 && cudaGetDevice(&dev) == cudaSuccess && dev >= 0 && dev < 64) {
    // >= 16 MB of output: the persistent table kernel (one 1024-thread CTA per SM, 128 KB of shared memory)
    if (!g_gelu_lut_ready[dev]) {  // once per device, ordered before the first use on this stream
      gelu_lut_init_kernel<<<65536 / 256, 256, 0, st>>>();
      count_launch();
      int rc0 = check_launch("gelu_lut_init");
      if (rc0 != MC_OK) return rc0;
      cudaFuncSetAttribute(geglu_lut_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 65536 * 2);
      g_gelu_lut_ready[dev] = true;
    }
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    geglu_lut_kernel<<<sms, 1024, 65536 * 2, st>>>((const __half*)in, (__half*)out, T, I);
    count_launch();
    return check_launch("geglu_lut");
  }
  int64_t blocks = (nvec + 255) / 256;
  if (blocks > 132 * 16) blocks = 132 * 16;
  geglu_kernel<<<(unsigned)blocks, 256, 0, st>>>((const __half*)in, (__half*)out, T, I);
  count_launch();
  return check_launch("geglu");
}

// ================================================================================================================
// Backward kernels for the autograd-carrying (guided, conditional) pass. Weights are frozen on this path
// (t2v_video_sample.py:67-68), so only input gradients are produced.
// ================================================================================================================
namespace mc {

// LayerNorm backward (input gradient only): one warp per row, statistics recomputed from x
template <int VPL>
__global__ void __launch_bounds__(256) layernorm_bwd_kernel(const __half* __restrict__ x, const __half* __restrict__ dy,
                                                            __half* __restrict__ dx, const __half* __restrict__ gamma,
                                                            const __half* __restrict__ pre_bias, int64_t rows, int C,
                                                            float eps) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int V = C / 8;
  for (int64_t row = (int64_t)blockIdx.x * 8 + warp; row < rows; row += (int64_t)gridDim.x * 8) {
    const __half* xr = x + row * C;
    const __half* dr = dy + row * C;
    Vec8 a[VPL], d[VPL];
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < VPL; ++i) {
      const int v = lane + i * 32;
      if (v < V) {
        a[i].u = *reinterpret_cast<const uint4*>(xr + v * 8);
        d[i].u = *reinterpret_cast<const uint4*>(dr + v * 8);
        if (pre_bias) {
          Vec8 pb;
          pb.u = *reinterpret_cast<const uint4*>(pre_bias + v * 8);
#pragma unroll
          for (int j = 0; j < 4; ++j) a[i].h2[j] = __hadd2(a[i].h2[j], pb.h2[j]);
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) s += __half2float(a[i].h[j]);
      }
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) s += __shfl_xor_sync(0xffffffffu, s, off);
    const float mean = s / (float)C;
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < VPL; ++i) {
      const int v = lane + i * 32;
      if (v < V) {
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const float t = __half2float(a[i].h[j]) - mean;
          q += t * t;
        }
      }
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) q += __shfl_xor_sync(0xffffffffu, q, off);
    const float rstd = rsqrtf(q / (float)C + eps);
    float sa = 0.f, sb = 0.f;
#pragma unroll
    for (int i = 0; i < VPL; ++i) {
      const int v = lane + i * 32;
      if (v < V) {
        Vec8 w;
        w.u = *reinterpret_cast<const uint4*>(gamma + v * 8);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const float dxh = __half2float(d[i].h[j]) * __half2float(w.h[j]);
          sa += dxh;
          sb += dxh * (__half2float(a[i].h[j]) - mean) * rstd;
        }
      }
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
      sa += __shfl_xor_sync(0xffffffffu, sa, off);
      sb += __shfl_xor_sync(0xffffffffu, sb, off);
    }
    sa /= (float)C;
    sb /= (float)C;
    __half* outr = dx + row * C;
#pragma unroll
    for (int i = 0; i < VPL; ++i) {
      const int v = lane + i * 32;
      if (v < V) {
        Vec8 w, o;
        w.u = *reinterpret_cast<const uint4*>(gamma + v * 8);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const float xh = (__half2float(a[i].h[j]) - mean) * rstd;
          const float dxh = __half2float(d[i].h[j]) * __half2float(w.h[j]);
          o.h[j] = __float2half_rn(rstd * (dxh - sa - xh * sb));
        }
        *reinterpret_cast<uint4*>(outr + v * 8) = o.u;
      }
    }
  }
}

// GEGLU backward: din[t, j] = dout * gelu(gate), din[t, I + j] = dout * h * gelu'(gate)
__global__ void __launch_bounds__(256) geglu_bwd_kernel(const __half* __restrict__ in, const __half* __restrict__ dout,
                                                        __half* __restrict__ din, int64_t T, int I) {
  const int VI = I / 8;
  const int64_t nvec = T * VI;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < nvec; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t t = i / VI;
    const int v = (int)(i % VI);
    const __half* row = in + t * 2 * I;
    Vec8 hh, gg, dd, o1, o2;
    hh.u = *reinterpret_cast<const uint4*>(row + v * 8);
    gg.u = *reinterpret_cast<const uint4*>(row + I + v * 8);
    dd.u = *reinterpret_cast<const uint4*>(dout + i * 8);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float g = __half2float(gg.h[j]), d = __half2float(dd.h[j]), h = __half2float(hh.h[j]);
      const float cdf = 0.5f * (1.f + erff(g * 0.70710678118654752440f));
      const float pdf = 0.39894228040143267794f * __expf(-0.5f * g * g);
      o1.h[j] = __float2half_rn(d * round_half(g * cdf));
      o2.h[j] = __float2half_rn(round_half(d * h) * (cdf + g * pdf));
    }
    __half* orow = din + t * 2 * I;
    *reinterpret_cast<uint4*>(orow + v * 8) = o1.u;
    *reinterpret_cast<uint4*>(orow + I + v * 8) = o2.u;
  }
}

}  // namespace mc

extern "C" int mc_layernorm_bwd(const void* x, const void* dy, void* dx, const void* gamma, const void* pre_bias,
                                int64_t rows, int C, float eps, void* stream) {
  using namespace mc;
  if (!x || !dy || !dx || !gamma || rows <= 0) {
    set_error("layernorm_bwd: null pointer or rows <= 0");
    return MC_E_INVALID;
  }
  if (C % 8 != 0 || C > 1280) {
    set_error("layernorm_bwd: need C %% 8 == 0 and C <= 1280 (got %d)", C);
    return MC_E_UNSUPPORTED;
  }
  int64_t blocks = (rows + 7) / 8;
  if (blocks > 132 * 16) blocks = 132 * 16;
  cudaStream_t st = (cudaStream_t)stream;
  const int vpl = (C / 8 + 31) / 32;
#define MC_LNB(V)                                                                                                     \
  layernorm_bwd_kernel<V><<<(unsigned)blocks, 256, 0, st>>>((const __half*)x, (const __half*)dy, (__half*)dx,         \
                                                            (const __half*)gamma, (const __half*)pre_bias, rows, C, eps)
  switch (vpl) {
    case 1: MC_LNB(1); break;
    case 2: MC_LNB(2); break;
    case 3: MC_LNB(3); break;
    case 4: MC_LNB(4); break;
    default: MC_LNB(5); break;
  }
#undef MC_LNB
  count_launch();
  return check_launch("layernorm_bwd");
}

extern "C" int mc_geglu_bwd(const void* in, const void* dout, void* din, int64_t T, int I, void* stream) {
  using namespace mc;
  if (!in || !dout || !din || T <= 0 || I <= 0) {
    set_error("geglu_bwd: null pointer or non-positive dims");
    return MC_E_INVALID;
  }
  if (I % 8 != 0) {
    set_error("geglu_bwd: inner dim must be a multiple of 8 (got %d)", I);
    return MC_E_UNSUPPORTED;
  }
  const int64_t nvec = T * (I / 8);
  int64_t blocks = (nvec + 255) / 256;
  if (blocks > 132 * 16) blocks = 132 * 16;
  geglu_bwd_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>((const __half*)in, (const __half*)dout, (__half*)din,
                                                                        T, I);
  count_launch();
  return check_launch("geglu_bwd");
}
