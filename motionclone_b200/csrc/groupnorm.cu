// GroupNorm(32) [+ time-embedding add] [+ SiLU] on channels_last `[(b f), h, w, C]` fp16 activations, forward and input
// gradient (sm_90a). Reference: InflatedGroupNorm + nonlinearity, models/resnet.py:21-29, :186-204; the transformer
// input norms models/attention.py:61,105 and models/motion_module.py:112,145 — all through ATen's NCHW GroupNorm, which
// on a channels_last activation costs a layout copy in, a layout copy before the next cuDNN conv and two passes of
// its own. These kernels read NHWC directly.
//
// HBM-bound: forward = 2 reads + 1 write of the tensor (statistics pass, then apply; the second read is an L2 hit for
// tensors under ~60 MB), backward = 2 x (x, dz) reads + 1 write. What bounds a streaming kernel is bytes in flight per
// SM, and register-staged loads cap that at 40-60 KB.
// So the tensor moves like the temporal-attention tiles do:
//   * a CTA owns a CONTIGUOUS run of pixels of one frame and walks it in tiles of <= 32 KB, each brought in by ONE bulk
//     copy (cp.async.bulk, TMA engine, SASS UBLKCP) signalled on an mbarrier, two stages deep: tile t+1 is in flight
//     while tile t is consumed, so 3 resident CTAs keep ~190 KB per SM in flight with no registers held;
//   * threads read the tile from shared memory with conflict-free 128-bit loads, thread -> (8-channel vector column,
//     pixel lane), so per-channel coefficients live in registers (no per-element integer division);
//   * the apply / backward-apply passes transform the tile IN PLACE and send it home with one bulk store;
//   * statistics: inside a CTA (<= a few hundred samples per group) plain fp32 sums / sums of squares, reduced with adds
//     only (shared memory, one warp per group, shuffles); ACROSS the splits of a frame the (count, mean, M2) partials are
//     merged with Chan's formula (robust to |mean| >> std) by the LAST CTA of the frame (atomic ticket), which writes
//     (mean, rstd): the apply pass reads 2 floats per group instead of re-folding the partials in every CTA.
// Frame-pooled statistics (nn.GroupNorm on a 5-D `[b, C, f, h, w]` tensor: one mean / variance per group over F
// consecutive frames) add a second level to that merge, in separate `_pooled` kernel instantiations: the last CTA of a
// frame leaves the frame's (count, mean, M2) in its split-0 partial slot; the last frame of the pool (second ticket)
// folds the F frame triples in frame order and writes the pool's (mean, rstd) into the row of each of its F frames, so
// the apply and backward-apply kernels are the per-frame ones. The merge order depends on (F, S, PX) only, and at F = 1
// every value is bitwise the per-frame one (one triple merged into an empty state, and a sum of one term, are exact).
// Workspace layout (device memory, caller-owned): [8192 B tickets: 1024 per frame, 1024 per pool | N*G*2 floats
// finalised | N*S*G*3 floats partial]. The ticket region must be zero on first use; every call leaves it zero again.
#include <math.h>

#include "mc_common.cuh"

namespace mc {

union GVec8 {
  uint4 u;
  __half h[8];
};

constexpr int kGnMaxFrames = 1024;
constexpr int kGnTicketBytes = 2 * kGnMaxFrames * 4;  // one uint32 per frame, then one per pool: N <= 1024
constexpr int kGnMaxSplits = 128;
constexpr int kGnTileBytes = 32 * 1024;  // shared-memory tile per CTA (forward: one tensor; backward: x and dz halves)
constexpr int kGnHeader = 128;           // mbarrier

// Chan et al. merge of (n, mean, M2) partials
__device__ __forceinline__ void chan_merge(float& n, float& mean, float& m2, float nb, float meanb, float m2b) {
  if (nb == 0.f) return;
  const float nn = n + nb;
  const float delta = meanb - mean;
  const float w = nb / nn;
  mean += delta * w;
  m2 += m2b + delta * delta * n * w;
  n = nn;
}

__device__ __forceinline__ float silu_fwd(float f) { return __fdividef(f, 1.f + __expf(-f)); }
__device__ __forceinline__ float silu_grad(float y) {
  const float s = __fdividef(1.f, 1.f + __expf(-y));
  return s * (1.f + y * (1.f - s));
}

// sum over the (lanes x cg) per-(thread, channel) slots of group g held in shared memory; result valid in every lane
__device__ __forceinline__ void gn_group_sum2(const float* __restrict__ s_a, const float* __restrict__ s_b, int g, int cg,
                                              int lanes, int V, int lane, float& ta, float& tb) {
  ta = tb = 0.f;
  for (int k = lane; k < lanes * cg; k += 32) {
    const int l = k / cg, c = g * cg + (k - l * cg);
    const int slot = (l * V + (c >> 3)) * 8 + (c & 7);
    ta += s_a[slot];
    tb += s_b[slot];
  }
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) {
    ta += __shfl_xor_sync(0xffffffffu, ta, off);
    tb += __shfl_xor_sync(0xffffffffu, tb, off);
  }
}

// One bulk copy of pixels [p0, p0 + npx) of frame n into `buf`, completion on `bar` (issued by one thread).
__device__ __forceinline__ void gn_fetch(uint8_t* buf, const __half* __restrict__ t, int n, int HW, int C, int p0, int npx,
                                         uint64_t* bar) {
  bulk_g2s(buf, t + ((int64_t)n * HW + p0) * C, (uint32_t)npx * C * 2, bar);
}

// ---------------------------------------------------------------------------------------------------------------
// forward, pass 1: statistics. grid (N, S); CTA = pixels [HW*s/S, HW*(s+1)/S) of frame n in trips of PX pixels.
// thread -> (vector column v = tid % V, pixel lane pl = tid / V).
// ---------------------------------------------------------------------------------------------------------------
// POOLED: statistics over the F = frames_per_stat consecutive frames of a pool (second merge level, see the top).
template <bool POOLED>
__device__ __forceinline__ void gn_stats_body(const __half* __restrict__ x, const __half* __restrict__ chan_bias,
                                              int frames_per_row, float* __restrict__ partial, float* __restrict__ stats,
                                              unsigned* __restrict__ tickets, int HW, int C, int G, int S, int lanes,
                                              int PX, float eps, int frames_per_stat) {
  extern __shared__ __align__(128) uint8_t smem[];
  __shared__ unsigned s_ticket;
  uint64_t* bar = reinterpret_cast<uint64_t*>(smem);  // bar[0], bar[1]: one per stage
  uint8_t* buf = smem + kGnHeader;
  float* s_sum = reinterpret_cast<float*>(smem + kGnHeader);  // [NT * 8], overlays the tiles once they have been consumed
  const int NT = blockDim.x, tid = threadIdx.x;
  float* s_sq = s_sum + NT * 8;
  const int V = C / 8;
  const int n = blockIdx.x, s = blockIdx.y;
  const int v = tid % V, pl = tid / V;
  const bool active = pl < lanes;
  const int p_begin = (int)(((int64_t)HW * s) / S), p_end = (int)(((int64_t)HW * (s + 1)) / S);
  const int ntrips = (p_end - p_begin + PX - 1) / PX;
  const int stage_bytes = (PX * C * 2 + 127) / 128 * 128;

  if (tid == 0) {
    mbar_init(bar, 1);
    mbar_init(bar + 1, 1);
    fence_mbar_init();
  }
  __syncthreads();
  auto fetch = [&](int t) {  // one thread
    const int p0 = p_begin + t * PX, npx = min(PX, p_end - p0);
    mbar_arrive_expect_tx(bar + (t & 1), (uint32_t)npx * C * 2);
    gn_fetch(buf + (t & 1) * stage_bytes, x, n, HW, C, p0, npx, bar + (t & 1));
  };
  if (tid == 0 && ntrips > 0) fetch(0);
  uint64_t sum2[4], sq2[4];  // channel pairs (2j, 2j + 1): eight fp32 accumulators
#pragma unroll
  for (int j = 0; j < 4; ++j) sum2[j] = sq2[j] = f2_pack(0.f, 0.f);
  const bool has_cb = chan_bias != nullptr;
  GVec8 cb;
  cb.u = make_uint4(0u, 0u, 0u, 0u);
  if (has_cb && active) cb.u = *reinterpret_cast<const uint4*>(chan_bias + (int64_t)(n / frames_per_row) * C + v * 8);
  for (int t = 0; t < ntrips; ++t) {
    if (tid == 0 && t + 1 < ntrips) fetch(t + 1);  // its stage was released by the barrier that ended trip t - 1
    const int npx = min(PX, p_end - (p_begin + t * PX));
    const uint8_t* tile = buf + (t & 1) * stage_bytes;
    mbar_wait(bar + (t & 1), (t >> 1) & 1);
    if (active) {
#pragma unroll 2
      for (int pp = pl; pp < npx; pp += lanes) {
        GVec8 a;
        a.u = *reinterpret_cast<const uint4*>(tile + ((int64_t)pp * C + v * 8) * 2);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          float f0 = __half2float(a.h[2 * j]), f1 = __half2float(a.h[2 * j + 1]);
          if (has_cb) {  // the eager `h + temb` is an fp16 tensor
            f0 = round_half(f0 + __half2float(cb.h[2 * j]));
            f1 = round_half(f1 + __half2float(cb.h[2 * j + 1]));
          }
          const uint64_t f = f2_pack(f0, f1);
          sum2[j] = f2_add(sum2[j], f);
          sq2[j] = f2_fma(f, f, sq2[j]);
        }
      }
    }
    if (t + 1 < ntrips) __syncthreads();  // every thread is done with this stage
  }
  float sum[8], sq[8];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    f2_unpack(sum2[j], sum[2 * j], sum[2 * j + 1]);
    f2_unpack(sq2[j], sq[2 * j], sq[2 * j + 1]);
  }
  __syncthreads();  // the tile is dead: its shared memory becomes the reduction slots
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    s_sum[tid * 8 + j] = active ? sum[j] : 0.f;
    s_sq[tid * 8 + j] = active ? sq[j] : 0.f;
  }
  __syncthreads();
  const int cg = C / G, warp = tid >> 5, lane = tid & 31, nwarps = NT >> 5;
  const float cnt = (float)cg * (float)(p_end - p_begin);  // samples per group in this split
  for (int g = warp; g < G; g += nwarps) {  // one warp per group: adds only
    float ts, tq;
    gn_group_sum2(s_sum, s_sq, g, cg, lanes, V, lane, ts, tq);
    if (lane == 0) {
      const float mean = cnt > 0.f ? ts / cnt : 0.f;
      float* out = partial + (((int64_t)n * S + s) * G + g) * 3;
      out[0] = cnt, out[1] = mean, out[2] = cnt > 0.f ? fmaxf(tq - ts * mean, 0.f) : 0.f;
    }
  }
  // ---- the last CTA of frame n folds the S partials into (mean, rstd) with Chan's formula ----
  __threadfence();
  __syncthreads();
  if (tid == 0) s_ticket = atomicAdd(&tickets[n], 1u);
  __syncthreads();
  if (s_ticket != (unsigned)(S - 1)) return;
  __threadfence();
  float* f_n = s_sum;  // re-use of the slots: three arrays of NT floats (slices * G <= NT)
  float* f_mean = s_sum + NT;
  float* f_m2 = s_sum + 2 * NT;
  const int slices = (NT / G) > 0 ? (NT / G) : 1;
  for (int idx = tid; idx < G * slices; idx += NT) {
    const int g = idx % G, k = idx / G;
    float an = 0.f, amean = 0.f, am2 = 0.f;
    for (int s2 = k; s2 < S; s2 += slices) {
      const float* p = partial + (((int64_t)n * S + s2) * G + g) * 3;
      chan_merge(an, amean, am2, __ldcg(p), __ldcg(p + 1), __ldcg(p + 2));
    }
    f_n[idx] = an, f_mean[idx] = amean, f_m2[idx] = am2;  // idx < G * slices <= NT (G <= 128 <= NT)
  }
  __syncthreads();
  for (int g = tid; g < G; g += NT) {
    float an = 0.f, amean = 0.f, am2 = 0.f;
    for (int k = 0; k < slices; ++k) chan_merge(an, amean, am2, f_n[k * G + g], f_mean[k * G + g], f_m2[k * G + g]);
    if (POOLED) {  // the frame's triple goes to its split-0 partial slot (already folded above)
      float* out = partial + ((int64_t)n * S * G + g) * 3;
      out[0] = an, out[1] = amean, out[2] = am2;
    } else {
      stats[((int64_t)n * G + g) * 2] = amean;
      stats[((int64_t)n * G + g) * 2 + 1] = rsqrtf(am2 / an + eps);
    }
  }
  if (tid == 0) tickets[n] = 0u;
  if (!POOLED) return;
  // ---- the last frame of the pool folds its F frame triples, in frame order, into (mean, rstd) ----
  const int F = frames_per_stat, f0 = n - n % F;
  __threadfence();
  __syncthreads();
  if (tid == 0) s_ticket = atomicAdd(&tickets[kGnMaxFrames + n / F], 1u);
  __syncthreads();
  if (s_ticket != (unsigned)(F - 1)) return;
  __threadfence();
  for (int g = tid; g < G; g += NT) {
    float an = 0.f, amean = 0.f, am2 = 0.f;
    for (int f = f0; f < f0 + F; ++f) {
      const float* p = partial + ((int64_t)f * S * G + g) * 3;
      chan_merge(an, amean, am2, __ldcg(p), __ldcg(p + 1), __ldcg(p + 2));
    }
    const float rstd = rsqrtf(am2 / an + eps);
    for (int f = f0; f < f0 + F; ++f) {
      stats[((int64_t)f * G + g) * 2] = amean;
      stats[((int64_t)f * G + g) * 2 + 1] = rstd;
    }
  }
  if (tid == 0) tickets[kGnMaxFrames + n / F] = 0u;
}

__global__ void __launch_bounds__(512, 2) groupnorm_stats_kernel(const __half* __restrict__ x,
                                                              const __half* __restrict__ chan_bias, int frames_per_row,
                                                              float* __restrict__ partial, float* __restrict__ stats,
                                                              unsigned* __restrict__ tickets, int HW, int C, int G, int S,
                                                              int lanes, int PX, float eps) {
  gn_stats_body<false>(x, chan_bias, frames_per_row, partial, stats, tickets, HW, C, G, S, lanes, PX, eps, 1);
}

__global__ void __launch_bounds__(512, 2) groupnorm_stats_pooled_kernel(
    const __half* __restrict__ x, const __half* __restrict__ chan_bias, int frames_per_row, float* __restrict__ partial,
    float* __restrict__ stats, unsigned* __restrict__ tickets, int HW, int C, int G, int S, int lanes, int PX, float eps,
    int frames_per_stat) {
  gn_stats_body<true>(x, chan_bias, frames_per_row, partial, stats, tickets, HW, C, G, S, lanes, PX, eps,
                      frames_per_stat);
}

// forward, pass 2: y = a[c] * x + b[c] with a = rstd * gamma, b = beta - mean * a (ATen's fused-parameter form) [-> SiLU]
// The tile is transformed in place in shared memory and leaves with one bulk store.
template <bool SILU>
__global__ void __launch_bounds__(512, 2) groupnorm_apply_kernel(const __half* __restrict__ x, __half* __restrict__ y,
                                                              const __half* __restrict__ chan_bias, int frames_per_row,
                                                              const float* __restrict__ stats,
                                                              const __half* __restrict__ gamma,
                                                              const __half* __restrict__ beta, int HW, int C, int G, int S,
                                                              int lanes, int PX) {
  extern __shared__ __align__(128) uint8_t smem[];
  uint64_t* bar = reinterpret_cast<uint64_t*>(smem);  // bar[0], bar[1]
  uint8_t* buf = smem + kGnHeader;
  const int tid = threadIdx.x, V = C / 8;
  const int n = blockIdx.x, s = blockIdx.y;
  const int v = tid % V, pl = tid / V;
  const bool active = pl < lanes;
  const int c0 = v * 8, cg = C / G;
  const int p_begin = (int)(((int64_t)HW * s) / S), p_end = (int)(((int64_t)HW * (s + 1)) / S);
  const int ntrips = (p_end - p_begin + PX - 1) / PX;
  const int stage_bytes = (PX * C * 2 + 127) / 128 * 128;
  if (tid == 0) {
    mbar_init(bar, 1);
    mbar_init(bar + 1, 1);
    fence_mbar_init();
  }
  __syncthreads();
  auto fetch = [&](int t) {  // one thread
    const int p0 = p_begin + t * PX, npx = min(PX, p_end - p0);
    mbar_arrive_expect_tx(bar + (t & 1), (uint32_t)npx * C * 2);
    gn_fetch(buf + (t & 1) * stage_bytes, x, n, HW, C, p0, npx, bar + (t & 1));
  };
  if (tid == 0 && ntrips > 0) fetch(0);
  // coefficients (L2-resident) while the first tile is in flight
  float a[8], b[8];
  GVec8 cb;
  cb.u = make_uint4(0u, 0u, 0u, 0u);
  const bool has_cb = chan_bias != nullptr;
  if (active) {
    GVec8 w, bt;
    w.u = *reinterpret_cast<const uint4*>(gamma + c0);
    bt.u = *reinterpret_cast<const uint4*>(beta + c0);
    if (has_cb) cb.u = *reinterpret_cast<const uint4*>(chan_bias + (int64_t)(n / frames_per_row) * C + c0);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int g = (c0 + j) / cg;
      const float mean = stats[((int64_t)n * G + g) * 2], rstd = stats[((int64_t)n * G + g) * 2 + 1];
      a[j] = rstd * __half2float(w.h[j]);
      b[j] = fmaf(-mean, a[j], __half2float(bt.h[j]));
    }
  }
  for (int t = 0; t < ntrips; ++t) {
    if (tid == 0 && t + 1 < ntrips) {
      if (t >= 1) bulk_wait_read_all();  // the store of trip t - 1 has finished reading the stage tile t + 1 lands in
      fetch(t + 1);
    }
    const int p0 = p_begin + t * PX, npx = min(PX, p_end - p0);
    uint8_t* tile = buf + (t & 1) * stage_bytes;
    mbar_wait(bar + (t & 1), (t >> 1) & 1);
    if (active) {
#pragma unroll 2
      for (int pp = pl; pp < npx; pp += lanes) {
        uint4* slot = reinterpret_cast<uint4*>(tile + ((int64_t)pp * C + c0) * 2);
        GVec8 in, o;
        in.u = *slot;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          float xv = __half2float(in.h[j]);
          if (has_cb) xv = round_half(xv + __half2float(cb.h[j]));
          float f = fmaf(xv, a[j], b[j]);
          if (SILU) f = silu_fwd(round_half(f));  // ATen rounds the GroupNorm output to fp16 before the separate SiLU kernel
          o.h[j] = __float2half_rn(f);
        }
        *slot = o.u;
      }
    }
    fence_proxy_async();  // generic-proxy writes of the tile -> visible to the bulk-store engine
    __syncthreads();
    if (tid == 0) {
      bulk_s2g(y + ((int64_t)n * HW + p0) * C, tile, (uint32_t)npx * C * 2);
      bulk_commit();
    }
  }
  if (tid == 0) bulk_wait_read_all();  // shared memory must outlive the last store's reads
}

// ---------------------------------------------------------------------------------------------------------------
// backward (input gradient; weights are frozen on this path, t2v_video_sample.py:67-68)
//   dxhat = dy * gamma, dy = dz * silu'(y) when SiLU was fused;  A = mean_group(dxhat), B = mean_group(dxhat * xhat)
//   dx = rstd * (dxhat - A - xhat * B)
// pass 1: per (frame, split) partial sums of dxhat and dxhat * xhat per group; last CTA of the frame -> (A, B)
// ---------------------------------------------------------------------------------------------------------------
struct GnBwdCoef {
  float mean[8], rstd[8], w[8], b[8];
};

__device__ __forceinline__ void gn_bwd_coef(GnBwdCoef& k, const float* __restrict__ stats, const __half* __restrict__ gamma,
                                            const __half* __restrict__ beta, int n, int c0, int cg, int G) {
  GVec8 w, b;
  w.u = *reinterpret_cast<const uint4*>(gamma + c0);
  b.u = *reinterpret_cast<const uint4*>(beta + c0);
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int g = (c0 + j) / cg;
    k.mean[j] = stats[((int64_t)n * G + g) * 2];
    k.rstd[j] = stats[((int64_t)n * G + g) * 2 + 1];
    k.w[j] = __half2float(w.h[j]);
    k.b[j] = __half2float(b.h[j]);
  }
}

// POOLED: the last CTA of a frame keeps the frame's raw sums; the last frame of the pool adds the F of them in frame
// order and scales by 1 / (F * HW * cg). `stats` holds the pool's (mean, rstd) in the row of every frame.
template <bool SILU, bool POOLED>
__device__ __forceinline__ void gn_bwd_reduce_body(
    const __half* __restrict__ x, const __half* __restrict__ chan_bias, int frames_per_row, const __half* __restrict__ dz,
    const float* __restrict__ stats, const __half* __restrict__ gamma, const __half* __restrict__ beta,
    float* __restrict__ partial, float* __restrict__ ab, unsigned* __restrict__ tickets, int HW, int C, int G, int S,
    int lanes, int PX, int frames_per_stat) {
  extern __shared__ __align__(128) uint8_t smem[];
  __shared__ unsigned s_ticket;
  uint64_t* bar = reinterpret_cast<uint64_t*>(smem);  // bar[0], bar[1]
  uint8_t* buf = smem + kGnHeader;                    // stage = [x tile | dz tile]
  float* s_a = reinterpret_cast<float*>(smem + kGnHeader);  // [NT * 8], overlays the tiles once consumed
  const int NT = blockDim.x, tid = threadIdx.x, V = C / 8;
  float* s_b = s_a + NT * 8;
  const int n = blockIdx.x, s = blockIdx.y;
  const int v = tid % V, pl = tid / V, cg = C / G, c0 = v * 8;
  const bool active = pl < lanes;
  const int p_begin = (int)(((int64_t)HW * s) / S), p_end = (int)(((int64_t)HW * (s + 1)) / S);
  const int ntrips = (p_end - p_begin + PX - 1) / PX;
  const int tile_bytes = (PX * C * 2 + 127) / 128 * 128, stage_bytes = 2 * tile_bytes;
  if (tid == 0) {
    mbar_init(bar, 1);
    mbar_init(bar + 1, 1);
    fence_mbar_init();
  }
  __syncthreads();
  auto fetch = [&](int t) {  // one thread
    const int p0 = p_begin + t * PX, npx = min(PX, p_end - p0);
    mbar_arrive_expect_tx(bar + (t & 1), 2u * (uint32_t)npx * C * 2);
    gn_fetch(buf + (t & 1) * stage_bytes, x, n, HW, C, p0, npx, bar + (t & 1));
    gn_fetch(buf + (t & 1) * stage_bytes + tile_bytes, dz, n, HW, C, p0, npx, bar + (t & 1));
  };
  if (tid == 0 && ntrips > 0) fetch(0);
  float sa[8], sb[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) sa[j] = sb[j] = 0.f;
  GnBwdCoef k;
  GVec8 cb;
  cb.u = make_uint4(0u, 0u, 0u, 0u);
  const bool has_cb = chan_bias != nullptr;
  if (active) {
    gn_bwd_coef(k, stats, gamma, beta, n, c0, cg, G);
    if (has_cb) cb.u = *reinterpret_cast<const uint4*>(chan_bias + (int64_t)(n / frames_per_row) * C + c0);
  }
  for (int t = 0; t < ntrips; ++t) {
    if (tid == 0 && t + 1 < ntrips) fetch(t + 1);
    const int npx = min(PX, p_end - (p_begin + t * PX));
    const uint8_t* tx = buf + (t & 1) * stage_bytes;
    const uint8_t* td = tx + tile_bytes;
    mbar_wait(bar + (t & 1), (t >> 1) & 1);
    if (active) {
#pragma unroll 2
      for (int pp = pl; pp < npx; pp += lanes) {
        GVec8 a, d;
        a.u = *reinterpret_cast<const uint4*>(tx + ((int64_t)pp * C + c0) * 2);
        d.u = *reinterpret_cast<const uint4*>(td + ((int64_t)pp * C + c0) * 2);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          float xv = __half2float(a.h[j]);
          if (has_cb) xv = round_half(xv + __half2float(cb.h[j]));
          const float xh = (xv - k.mean[j]) * k.rstd[j];
          float dy = __half2float(d.h[j]);
          if (SILU) dy *= silu_grad(round_half(fmaf(xh, k.w[j], k.b[j])));
          const float dxh = dy * k.w[j];
          sa[j] += dxh;
          sb[j] = fmaf(dxh, xh, sb[j]);
        }
      }
    }
    if (t + 1 < ntrips) __syncthreads();
  }
  __syncthreads();
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    s_a[tid * 8 + j] = active ? sa[j] : 0.f;
    s_b[tid * 8 + j] = active ? sb[j] : 0.f;
  }
  __syncthreads();
  const int warp = tid >> 5, lane = tid & 31, nwarps = NT >> 5;
  for (int g = warp; g < G; g += nwarps) {
    float ta, tb;
    gn_group_sum2(s_a, s_b, g, cg, lanes, V, lane, ta, tb);
    if (lane == 0) {
      float* out = partial + (((int64_t)n * S + s) * G + g) * 2;
      out[0] = ta, out[1] = tb;
    }
  }
  __threadfence();
  __syncthreads();
  if (tid == 0) s_ticket = atomicAdd(&tickets[n], 1u);
  __syncthreads();
  if (s_ticket != (unsigned)(S - 1)) return;
  __threadfence();
  const float inv_m = 1.f / ((float)HW * (float)cg);
  float* f_a = s_a;  // re-use of the slots: [slices * G] x 2 (slices * G <= NT); fixed partition -> deterministic sums
  float* f_b = s_a + NT;
  const int slices = (NT / G) > 0 ? (NT / G) : 1;
  for (int idx = tid; idx < G * slices; idx += NT) {
    const int g = idx % G, kk = idx / G;
    float ta = 0.f, tb = 0.f;
    for (int s2 = kk; s2 < S; s2 += slices) {
      const float* p = partial + (((int64_t)n * S + s2) * G + g) * 2;
      ta += __ldcg(p), tb += __ldcg(p + 1);
    }
    f_a[idx] = ta, f_b[idx] = tb;
  }
  __syncthreads();
  for (int g = tid; g < G; g += NT) {
    float ta = 0.f, tb = 0.f;
    for (int kk = 0; kk < slices; ++kk) ta += f_a[kk * G + g], tb += f_b[kk * G + g];
    if (POOLED) {  // raw frame sums -> the frame's split-0 partial slot (already folded above)
      float* out = partial + ((int64_t)n * S * G + g) * 2;
      out[0] = ta, out[1] = tb;
    } else {
      ab[((int64_t)n * G + g) * 2] = ta * inv_m;
      ab[((int64_t)n * G + g) * 2 + 1] = tb * inv_m;
    }
  }
  if (tid == 0) tickets[n] = 0u;
  if (!POOLED) return;
  const int F = frames_per_stat, f0 = n - n % F;
  __threadfence();
  __syncthreads();
  if (tid == 0) s_ticket = atomicAdd(&tickets[kGnMaxFrames + n / F], 1u);
  __syncthreads();
  if (s_ticket != (unsigned)(F - 1)) return;
  __threadfence();
  const float inv_pool = 1.f / ((float)F * (float)HW * (float)cg);  // F = 1: the float inv_m is
  for (int g = tid; g < G; g += NT) {
    const float* p = partial + ((int64_t)f0 * S * G + g) * 2;
    float ta = __ldcg(p), tb = __ldcg(p + 1);
    for (int f = f0 + 1; f < f0 + F; ++f) {
      p = partial + ((int64_t)f * S * G + g) * 2;
      ta += __ldcg(p), tb += __ldcg(p + 1);
    }
    for (int f = f0; f < f0 + F; ++f) {
      ab[((int64_t)f * G + g) * 2] = ta * inv_pool;
      ab[((int64_t)f * G + g) * 2 + 1] = tb * inv_pool;
    }
  }
  if (tid == 0) tickets[kGnMaxFrames + n / F] = 0u;
}

template <bool SILU>
__global__ void __launch_bounds__(512) groupnorm_bwd_reduce_kernel(
    const __half* __restrict__ x, const __half* __restrict__ chan_bias, int frames_per_row, const __half* __restrict__ dz,
    const float* __restrict__ stats, const __half* __restrict__ gamma, const __half* __restrict__ beta,
    float* __restrict__ partial, float* __restrict__ ab, unsigned* __restrict__ tickets, int HW, int C, int G, int S,
    int lanes, int PX) {
  gn_bwd_reduce_body<SILU, false>(x, chan_bias, frames_per_row, dz, stats, gamma, beta, partial, ab, tickets, HW, C, G, S,
                                  lanes, PX, 1);
}

template <bool SILU>
__global__ void __launch_bounds__(512) groupnorm_bwd_reduce_pooled_kernel(
    const __half* __restrict__ x, const __half* __restrict__ chan_bias, int frames_per_row, const __half* __restrict__ dz,
    const float* __restrict__ stats, const __half* __restrict__ gamma, const __half* __restrict__ beta,
    float* __restrict__ partial, float* __restrict__ ab, unsigned* __restrict__ tickets, int HW, int C, int G, int S,
    int lanes, int PX, int frames_per_stat) {
  gn_bwd_reduce_body<SILU, true>(x, chan_bias, frames_per_row, dz, stats, gamma, beta, partial, ab, tickets, HW, C, G, S,
                                 lanes, PX, frames_per_stat);
}

// pass 2: dx over the dz tile, in place, then one bulk store
template <bool SILU>
__global__ void __launch_bounds__(512) groupnorm_bwd_apply_kernel(
    const __half* __restrict__ x, const __half* __restrict__ chan_bias, int frames_per_row, const __half* __restrict__ dz,
    __half* __restrict__ dx, const float* __restrict__ stats, const float* __restrict__ ab, const __half* __restrict__ gamma,
    const __half* __restrict__ beta, int HW, int C, int G, int S, int lanes, int PX) {
  extern __shared__ __align__(128) uint8_t smem[];
  uint64_t* bar = reinterpret_cast<uint64_t*>(smem);  // bar[0], bar[1]
  uint8_t* buf = smem + kGnHeader;                    // stage = [x tile | dz tile]
  const int tid = threadIdx.x, V = C / 8;
  const int n = blockIdx.x, s = blockIdx.y;
  const int v = tid % V, pl = tid / V;
  const bool active = pl < lanes;
  const int c0 = v * 8, cg = C / G;
  const int p_begin = (int)(((int64_t)HW * s) / S), p_end = (int)(((int64_t)HW * (s + 1)) / S);
  const int ntrips = (p_end - p_begin + PX - 1) / PX;
  const int tile_bytes = (PX * C * 2 + 127) / 128 * 128, stage_bytes = 2 * tile_bytes;
  if (tid == 0) {
    mbar_init(bar, 1);
    mbar_init(bar + 1, 1);
    fence_mbar_init();
  }
  __syncthreads();
  auto fetch = [&](int t) {  // one thread
    const int p0 = p_begin + t * PX, npx = min(PX, p_end - p0);
    mbar_arrive_expect_tx(bar + (t & 1), 2u * (uint32_t)npx * C * 2);
    gn_fetch(buf + (t & 1) * stage_bytes, x, n, HW, C, p0, npx, bar + (t & 1));
    gn_fetch(buf + (t & 1) * stage_bytes + tile_bytes, dz, n, HW, C, p0, npx, bar + (t & 1));
  };
  if (tid == 0 && ntrips > 0) fetch(0);
  GnBwdCoef k;
  float ga[8], gb[8];
  GVec8 cb;
  cb.u = make_uint4(0u, 0u, 0u, 0u);
  const bool has_cb = chan_bias != nullptr;
  if (active) {
    gn_bwd_coef(k, stats, gamma, beta, n, c0, cg, G);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int g = (c0 + j) / cg;
      ga[j] = ab[((int64_t)n * G + g) * 2];
      gb[j] = ab[((int64_t)n * G + g) * 2 + 1];
    }
    if (has_cb) cb.u = *reinterpret_cast<const uint4*>(chan_bias + (int64_t)(n / frames_per_row) * C + c0);
  }
  for (int t = 0; t < ntrips; ++t) {
    if (tid == 0 && t + 1 < ntrips) {
      if (t >= 1) bulk_wait_read_all();  // the store of trip t - 1 has finished reading the stage tile t + 1 lands in
      fetch(t + 1);
    }
    const int p0 = p_begin + t * PX, npx = min(PX, p_end - p0);
    const uint8_t* tx = buf + (t & 1) * stage_bytes;
    uint8_t* td = buf + (t & 1) * stage_bytes + tile_bytes;
    mbar_wait(bar + (t & 1), (t >> 1) & 1);
    if (active) {
#pragma unroll 2
      for (int pp = pl; pp < npx; pp += lanes) {
        uint4* dslot = reinterpret_cast<uint4*>(td + ((int64_t)pp * C + c0) * 2);
        GVec8 a, d, o;
        a.u = *reinterpret_cast<const uint4*>(tx + ((int64_t)pp * C + c0) * 2);
        d.u = *dslot;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          float xv = __half2float(a.h[j]);
          if (has_cb) xv = round_half(xv + __half2float(cb.h[j]));
          const float xh = (xv - k.mean[j]) * k.rstd[j];
          float dy = __half2float(d.h[j]);
          if (SILU) dy *= silu_grad(round_half(fmaf(xh, k.w[j], k.b[j])));
          const float dxh = dy * k.w[j];
          o.h[j] = __float2half_rn(k.rstd[j] * (dxh - ga[j] - xh * gb[j]));
        }
        *dslot = o.u;
      }
    }
    fence_proxy_async();
    __syncthreads();
    if (tid == 0) {
      bulk_s2g(dx + ((int64_t)n * HW + p0) * C, td, (uint32_t)npx * C * 2);
      bulk_commit();
    }
  }
  if (tid == 0) bulk_wait_read_all();
}

// ---------------------------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------------------------
struct GnLaunch {
  int V, lanes, NT;
};

static GnLaunch gn_launch(int C) {
  GnLaunch g;
  g.V = C / 8;
  g.lanes = 256 / g.V;
  if (g.lanes < 1) g.lanes = 1;
  if (g.V * g.lanes < 192 && g.V * (g.lanes + 1) <= 512) ++g.lanes;  // e.g. C = 1280: 2 pixel lanes, 320 threads
  g.NT = (g.V * g.lanes + 31) / 32 * 32;
  return g;
}

// Tiling of a frame: PX pixels (one bulk copy of <= `tile_bytes` per tensor) per trip, S splits (CTAs) per frame; a CTA
// makes more than one trip only when the frame would need more than kGnMaxSplits splits.
struct GnTiling {
  int PX, S, smem;
};

// `tensors` tiles of <= tile_bytes each per stage, two stages (64 KB per CTA -> 3 CTAs per SM; the backward kernels hold
// more registers: 2). ONE wave per sample: at most 132 x ctas_per_sm CTAs for the `frames_per_sample` frames of one
// sample, each walking ceil(tiles / S) tiles through its two-stage pipeline (a grid of 1.5 waves costs two: measured on
// the 16 x 64 x 64 x 320 layers).
// S and PX depend on the frames of ONE sample, never on how many samples share the launch: a frame's fp32 statistics
// are summed in an order fixed by (S, PX), so a batched call gives every sample the bits of its own single-sample call.
static GnTiling gn_tiling(int frames_per_sample, int HW, int C, int NT, int tensors, int tile_bytes, int ctas_per_sm) {
  GnTiling t;
  t.PX = tile_bytes / (C * 2);
  if (t.PX < 1) t.PX = 1;
  if (t.PX > HW) t.PX = HW;
  const int tiles = (HW + t.PX - 1) / t.PX;
  t.S = (132 * ctas_per_sm) / frames_per_sample;
  if (t.S < 1) t.S = 1;
  if (t.S > tiles) t.S = tiles;
  if (t.S > kGnMaxSplits) t.S = kGnMaxSplits;
  const int tile = (t.PX * C * 2 + 127) / 128 * 128;
  const int stages = 2 * tensors * tile;
  const int slots = 2 * NT * 8 * (int)sizeof(float);  // reduction slots overlay the tiles
  t.smem = kGnHeader + (stages > slots ? stages : slots);
  return t;
}

template <typename K>
static void gn_allow_smem(K kern, int smem) {
  if (smem > 48 * 1024) cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
}

static int gn_check(const char* what, int N, int HW, int C, int G, int samples) {
  if (N <= 0 || HW <= 0) {
    set_error("%s: non-positive dims", what);
    return MC_E_INVALID;
  }
  if (samples <= 0 || N % samples != 0) {
    set_error("%s: samples must be positive and divide N (got N=%d samples=%d)", what, N, samples);
    return MC_E_INVALID;
  }
  if (C % 8 != 0 || C % G != 0 || C > 4096 || G > 128 || N > kGnMaxFrames) {
    set_error("%s: need C %% 8 == 0, C %% G == 0, C <= 4096, G <= 128, N <= 1024 (got N=%d C=%d G=%d)", what, N, C, G);
    return MC_E_UNSUPPORTED;
  }
  return MC_OK;
}

// a pool of F frames never straddles a tiling sample, so each sample's statistics stay its own
static int gn_check_pool(const char* what, int N, int samples, int frames_per_stat) {
  if (frames_per_stat < 1 || N % frames_per_stat != 0 || (N / samples) % frames_per_stat != 0) {
    set_error("%s: frames_per_stat must be >= 1 and divide N / samples (got N=%d samples=%d frames_per_stat=%d)", what,
              N, samples, frames_per_stat);
    return MC_E_INVALID;
  }
  return MC_OK;
}

struct GnWorkspace {
  unsigned* tickets;
  float* finalised;  // fwd: (mean, rstd); bwd: (A/m, B/m)   [N, G, 2]
  float* partial;
};

static GnWorkspace gn_workspace(void* ws, int N, int G) {
  GnWorkspace w;
  w.tickets = reinterpret_cast<unsigned*>(ws);
  w.finalised = reinterpret_cast<float*>(reinterpret_cast<char*>(ws) + kGnTicketBytes);
  w.partial = w.finalised + (int64_t)N * G * 2;
  return w;
}

}  // namespace mc

extern "C" int64_t mc_groupnorm_workspace_bytes(int N, int G) {
  return mc::kGnTicketBytes + (int64_t)N * G * 2 * sizeof(float) + (int64_t)N * mc::kGnMaxSplits * G * 3 * sizeof(float);
}

namespace mc {

// pool = 0: per-frame statistics (the original kernels); pool = F >= 1: statistics pooled over F frames
static int gn_forward(const char* what, const void* x, const void* chan_bias, int frames_per_bias_row, void* y,
                      const void* gamma, const void* beta, void* workspace, int64_t workspace_bytes, int N, int HW, int C,
                      int G, int samples, int pool, float eps, int fuse_silu, void* stream) {
  if (!x || !y || !gamma || !beta || !workspace) {
    set_error("%s: null pointer", what);
    return MC_E_INVALID;
  }
  int rc = gn_check(what, N, HW, C, G, samples);
  if (rc != MC_OK) return rc;
  if (pool != 0 && (rc = gn_check_pool(what, N, samples, pool)) != MC_OK) return rc;
  if (chan_bias != nullptr && frames_per_bias_row <= 0) {
    set_error("%s: frames_per_bias_row must be positive when chan_bias is given", what);
    return MC_E_INVALID;
  }
  if (workspace_bytes < mc_groupnorm_workspace_bytes(N, G)) {
    set_error("%s: workspace too small (%lld < %lld bytes)", what, (long long)workspace_bytes,
              (long long)mc_groupnorm_workspace_bytes(N, G));
    return MC_E_INVALID;
  }
  const GnLaunch L = gn_launch(C);
  const GnWorkspace w = gn_workspace(workspace, N, G);
  cudaStream_t st = (cudaStream_t)stream;
  const GnTiling T = gn_tiling(N / samples, HW, C, L.NT, 1, kGnTileBytes, 3);
  if (pool != 0) {
    gn_allow_smem(groupnorm_stats_pooled_kernel, T.smem);
    groupnorm_stats_pooled_kernel<<<dim3(N, T.S), L.NT, T.smem, st>>>(
        (const __half*)x, (const __half*)chan_bias, frames_per_bias_row, w.partial, w.finalised, w.tickets, HW, C, G, T.S,
        L.lanes, T.PX, eps, pool);
  } else {
    gn_allow_smem(groupnorm_stats_kernel, T.smem);
    groupnorm_stats_kernel<<<dim3(N, T.S), L.NT, T.smem, st>>>((const __half*)x, (const __half*)chan_bias,
                                                               frames_per_bias_row, w.partial, w.finalised, w.tickets, HW,
                                                               C, G, T.S, L.lanes, T.PX, eps);
  }
  count_launch();
  rc = check_launch("groupnorm_stats");
  if (rc != MC_OK) return rc;
  if (fuse_silu) {
    gn_allow_smem(groupnorm_apply_kernel<true>, T.smem);
    groupnorm_apply_kernel<true><<<dim3(N, T.S), L.NT, T.smem, st>>>(
        (const __half*)x, (__half*)y, (const __half*)chan_bias, frames_per_bias_row, w.finalised, (const __half*)gamma,
        (const __half*)beta, HW, C, G, T.S, L.lanes, T.PX);
  } else {
    gn_allow_smem(groupnorm_apply_kernel<false>, T.smem);
    groupnorm_apply_kernel<false><<<dim3(N, T.S), L.NT, T.smem, st>>>(
        (const __half*)x, (__half*)y, (const __half*)chan_bias, frames_per_bias_row, w.finalised, (const __half*)gamma,
        (const __half*)beta, HW, C, G, T.S, L.lanes, T.PX);
  }
  count_launch();
  return check_launch("groupnorm_apply");
}

}  // namespace mc

extern "C" int mc_groupnorm_nhwc_batched(const void* x, const void* chan_bias, int frames_per_bias_row, void* y,
                                         const void* gamma, const void* beta, void* workspace, int64_t workspace_bytes,
                                         int N, int HW, int C, int G, int samples, float eps, int fuse_silu, void* stream) {
  return mc::gn_forward("groupnorm_nhwc", x, chan_bias, frames_per_bias_row, y, gamma, beta, workspace, workspace_bytes,
                        N, HW, C, G, samples, 0, eps, fuse_silu, stream);
}

extern "C" int mc_groupnorm_nhwc_pooled(const void* x, const void* chan_bias, int frames_per_bias_row, void* y,
                                        const void* gamma, const void* beta, void* workspace, int64_t workspace_bytes,
                                        int N, int HW, int C, int G, int samples, int frames_per_stat, float eps,
                                        int fuse_silu, void* stream) {
  if (frames_per_stat < 1) {  // 0 would select the per-frame kernels in gn_forward
    mc::set_error("groupnorm_nhwc_pooled: frames_per_stat must be >= 1 (got %d)", frames_per_stat);
    return MC_E_INVALID;
  }
  return mc::gn_forward("groupnorm_nhwc_pooled", x, chan_bias, frames_per_bias_row, y, gamma, beta, workspace,
                        workspace_bytes, N, HW, C, G, samples, frames_per_stat, eps, fuse_silu, stream);
}

extern "C" int mc_groupnorm_nhwc(const void* x, const void* chan_bias, int frames_per_bias_row, void* y,
                                 const void* gamma, const void* beta, void* workspace, int64_t workspace_bytes, int N,
                                 int HW, int C, int G, float eps, int fuse_silu, void* stream) {
  return mc_groupnorm_nhwc_batched(x, chan_bias, frames_per_bias_row, y, gamma, beta, workspace, workspace_bytes, N, HW,
                                   C, G, 1, eps, fuse_silu, stream);
}

extern "C" int mc_groupnorm_nhwc_stats(const void* workspace, void* stats, int N, int HW, int G, float eps, void* stream) {
  using namespace mc;
  (void)HW, (void)eps;  // kept in the signature: the statistics are final once mc_groupnorm_nhwc has run
  if (!workspace || !stats || N <= 0 || G <= 0) {
    set_error("groupnorm_nhwc_stats: null pointer or non-positive dims");
    return MC_E_INVALID;
  }
  const GnWorkspace w = gn_workspace(const_cast<void*>(workspace), N, G);
  const cudaError_t e = cudaMemcpyAsync(stats, w.finalised, (size_t)N * G * 2 * sizeof(float), cudaMemcpyDeviceToDevice,
                                        (cudaStream_t)stream);
  if (e != cudaSuccess) {
    set_error("groupnorm_nhwc_stats: %s", cudaGetErrorString(e));
    return MC_E_CUDA;
  }
  return MC_OK;
}

namespace mc {

template <bool SILU>
static void gn_launch_bwd_reduce(int pool, dim3 grid, int NT, int smem, cudaStream_t st, const __half* x,
                                 const __half* cb, int fpr, const __half* dz, const float* stats, const __half* gamma,
                                 const __half* beta, const GnWorkspace& w, int HW, int C, int G, const GnTiling& T,
                                 int lanes) {
  if (pool != 0) {
    gn_allow_smem(groupnorm_bwd_reduce_pooled_kernel<SILU>, smem);
    groupnorm_bwd_reduce_pooled_kernel<SILU><<<grid, NT, smem, st>>>(x, cb, fpr, dz, stats, gamma, beta, w.partial,
                                                                     w.finalised, w.tickets, HW, C, G, T.S, lanes, T.PX,
                                                                     pool);
  } else {
    gn_allow_smem(groupnorm_bwd_reduce_kernel<SILU>, smem);
    groupnorm_bwd_reduce_kernel<SILU><<<grid, NT, smem, st>>>(x, cb, fpr, dz, stats, gamma, beta, w.partial, w.finalised,
                                                              w.tickets, HW, C, G, T.S, lanes, T.PX);
  }
}

// pool = 0: per-frame statistics; pool = F >= 1: `stats` and the gradient sums pooled over F frames
static int gn_backward(const char* what, const void* x, const void* chan_bias, int frames_per_bias_row, const void* dz,
                       void* dx, const void* stats, const void* gamma, const void* beta, void* workspace,
                       int64_t workspace_bytes, int N, int HW, int C, int G, int samples, int pool, int fuse_silu,
                       void* stream) {
  if (!x || !dz || !dx || !stats || !gamma || !beta || !workspace) {
    set_error("%s: null pointer", what);
    return MC_E_INVALID;
  }
  int rc = gn_check(what, N, HW, C, G, samples);
  if (rc != MC_OK) return rc;
  if (pool != 0 && (rc = gn_check_pool(what, N, samples, pool)) != MC_OK) return rc;
  if (chan_bias != nullptr && frames_per_bias_row <= 0) {
    set_error("%s: frames_per_bias_row must be positive when chan_bias is given", what);
    return MC_E_INVALID;
  }
  if (workspace_bytes < mc_groupnorm_workspace_bytes(N, G)) {
    set_error("%s: workspace too small", what);
    return MC_E_INVALID;
  }
  const GnLaunch L = gn_launch(C);
  const GnWorkspace w = gn_workspace(workspace, N, G);
  cudaStream_t st = (cudaStream_t)stream;
  const GnTiling T = gn_tiling(N / samples, HW, C, L.NT, 2, kGnTileBytes / 2, 2);
  const __half *xp = (const __half*)x, *cbp = (const __half*)chan_bias, *dzp = (const __half*)dz;
  const __half *gp = (const __half*)gamma, *bp = (const __half*)beta;
  const float* sp = (const float*)stats;
  if (fuse_silu)
    gn_launch_bwd_reduce<true>(pool, dim3(N, T.S), L.NT, T.smem, st, xp, cbp, frames_per_bias_row, dzp, sp, gp, bp, w, HW,
                               C, G, T, L.lanes);
  else
    gn_launch_bwd_reduce<false>(pool, dim3(N, T.S), L.NT, T.smem, st, xp, cbp, frames_per_bias_row, dzp, sp, gp, bp, w,
                                HW, C, G, T, L.lanes);
  count_launch();
  rc = check_launch("groupnorm_bwd_reduce");
  if (rc != MC_OK) return rc;
  if (fuse_silu) {
    gn_allow_smem(groupnorm_bwd_apply_kernel<true>, T.smem);
    groupnorm_bwd_apply_kernel<true><<<dim3(N, T.S), L.NT, T.smem, st>>>(xp, cbp, frames_per_bias_row, dzp, (__half*)dx,
                                                                         sp, w.finalised, gp, bp, HW, C, G, T.S, L.lanes,
                                                                         T.PX);
  } else {
    gn_allow_smem(groupnorm_bwd_apply_kernel<false>, T.smem);
    groupnorm_bwd_apply_kernel<false><<<dim3(N, T.S), L.NT, T.smem, st>>>(xp, cbp, frames_per_bias_row, dzp, (__half*)dx,
                                                                          sp, w.finalised, gp, bp, HW, C, G, T.S, L.lanes,
                                                                          T.PX);
  }
  count_launch();
  return check_launch("groupnorm_bwd_apply");
}

}  // namespace mc

extern "C" int mc_groupnorm_nhwc_bwd_batched(const void* x, const void* chan_bias, int frames_per_bias_row,
                                             const void* dz, void* dx, const void* stats, const void* gamma,
                                             const void* beta, void* workspace, int64_t workspace_bytes, int N, int HW,
                                             int C, int G, int samples, int fuse_silu, void* stream) {
  return mc::gn_backward("groupnorm_nhwc_bwd", x, chan_bias, frames_per_bias_row, dz, dx, stats, gamma, beta, workspace,
                         workspace_bytes, N, HW, C, G, samples, 0, fuse_silu, stream);
}

extern "C" int mc_groupnorm_nhwc_bwd_pooled(const void* x, const void* chan_bias, int frames_per_bias_row,
                                            const void* dz, void* dx, const void* stats, const void* gamma,
                                            const void* beta, void* workspace, int64_t workspace_bytes, int N, int HW,
                                            int C, int G, int samples, int frames_per_stat, int fuse_silu, void* stream) {
  if (frames_per_stat < 1) {
    mc::set_error("groupnorm_nhwc_bwd_pooled: frames_per_stat must be >= 1 (got %d)", frames_per_stat);
    return MC_E_INVALID;
  }
  return mc::gn_backward("groupnorm_nhwc_bwd_pooled", x, chan_bias, frames_per_bias_row, dz, dx, stats, gamma, beta,
                         workspace, workspace_bytes, N, HW, C, G, samples, frames_per_stat, fuse_silu, stream);
}

extern "C" int mc_groupnorm_nhwc_bwd(const void* x, const void* chan_bias, int frames_per_bias_row, const void* dz,
                                     void* dx, const void* stats, const void* gamma, const void* beta, void* workspace,
                                     int64_t workspace_bytes, int N, int HW, int C, int G, int fuse_silu, void* stream) {
  return mc_groupnorm_nhwc_bwd_batched(x, chan_bias, frames_per_bias_row, dz, dx, stats, gamma, beta, workspace,
                                       workspace_bytes, N, HW, C, G, 1, fuse_silu, stream);
}
