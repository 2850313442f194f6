// TMA tensor maps (cp.async.bulk.tensor) + swizzled wgmma shared-memory descriptors, sm_90a.
//
// An attention operand tile is [ROWS][DH] fp16 (rows = tokens of one frame / head, DH contiguous in global memory).
// In shared memory it is a sequence of PARTS along DH, each landed by ONE tensor-map load:
//   SW128 part: [ROWS][64 elements = 128 B], CU_TENSOR_MAP_SWIZZLE_128B   (1024-byte aligned)
//   SW32  part: [ROWS][16 elements =  32 B], CU_TENSOR_MAP_SWIZZLE_32B
// DH < 64 -> one SW128 part whose columns DH..63 are zero-filled by the TMA unit (the map's innermost extent is DH, the
// box is 64 wide: out-of-bounds elements read as 0); DH = 80 -> SW128 + SW32; DH = 160 -> 2 x SW128 + 2 x SW32.
// The same bytes serve as
//   K-major operand  (rows = M or N, DH = K):  canonical  Swizzle<3,4,3> o ((8,n),2):((8,SBO),1)   [units of 16 B]
//   MN-major operand (DH = N, rows = K):       canonical  Swizzle<3,4,3> o ((8,n),(8,k)):((1,LBO),(8,SBO))
// so V needs no transpose for P V, and K / Q / dO tiles are shared between the GEMMs of the backward pass.
#pragma once
#include <cuda.h>

#include "tc_common.cuh"

namespace mc {

// ---- host: tensor-map encode through the runtime's driver entry point (no link-time dependency on libcuda) ----
typedef CUresult (*mc_encode_tiled_fn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                       const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                       CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

inline mc_encode_tiled_fn tensor_map_encoder() {
  static mc_encode_tiled_fn fn = [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess ||
        q != cudaDriverEntryPointSuccess)
      p = nullptr;
    return (mc_encode_tiled_fn)p;
  }();
  return fn;
}

// fp16 tensor [frames][rows][heads][DH]: element (b, r, h, e) at base + b*stride_b + r*stride_r + h*DH + e (elements).
// Box = (box_e, 1 head, 128 rows, 1 frame); coordinates (e0, h, r0, b). Returns 0 on success.
inline int make_attn_tensor_map(CUtensorMap* map, const void* base, int DH, int H, int64_t rows, int64_t frames,
                                int64_t stride_r, int64_t stride_b, int box_e, int box_rows, bool swizzle128) {
  mc_encode_tiled_fn enc = tensor_map_encoder();
  // The encoder is a DRIVER entry point: it needs the primary context current on the calling thread. A thread that has
  // not yet made a runtime call (autograd's backward worker on its first node) has none -> CUDA_ERROR_INVALID_CONTEXT.
  static thread_local bool ctx_bound = false;
  if (!ctx_bound) {
    cudaFree(nullptr);  // binds the runtime's primary context to this thread (no-op otherwise)
    ctx_bound = true;
  }
  if (!enc) {
    set_error("cuTensorMapEncodeTiled: driver entry point unavailable (cudaGetDriverEntryPoint failed)");
    return -1;
  }
  cuuint64_t gdim[4] = {(cuuint64_t)DH, (cuuint64_t)H, (cuuint64_t)rows, (cuuint64_t)frames};
  cuuint64_t gstr[3] = {(cuuint64_t)DH * 2, (cuuint64_t)stride_r * 2, (cuuint64_t)stride_b * 2};
  if (frames == 1) gstr[2] = gstr[1] * (cuuint64_t)rows;  // unused dimension: any legal stride
  cuuint32_t box[4] = {(cuuint32_t)box_e, 1u, (cuuint32_t)box_rows, 1u};
  cuuint32_t estr[4] = {1u, 1u, 1u, 1u};
  CUresult r = enc(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, const_cast<void*>(base), gdim, gstr, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle128 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_32B,
                   CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS)
    set_error("cuTensorMapEncodeTiled -> CUresult %d: base %p dims (%d, %d, %lld, %lld) strides (%lld, %lld) elements, box "
              "(%d, 1, %d, 1), swizzle %s", (int)r, base, DH, H, (long long)rows, (long long)frames, (long long)stride_r,
              (long long)stride_b, box_e, box_rows, swizzle128 ? "128B" : "32B");
  return r == CUDA_SUCCESS ? 0 : (int)r;
}

// Text cross-attention takes the whole key axis (77 tokens) as one tile in the backward: at most this many keys.
constexpr int kMaxTextKeys = 80;

struct AttnMaps {
  CUtensorMap m128, m32;
};
// maps for one operand tensor (box height `rows`); the SW32 map is only encoded when the head dim has 16-wide parts
template <int DH>
int make_attn_maps(AttnMaps& m, const void* base, int H, int N, int B, int64_t sr, int64_t sb, int rows) {
  int rc = make_attn_tensor_map(&m.m128, base, DH, H, N, B, sr, sb, 64, rows, true);
  if (rc) return rc;
  if (DH >= 64 && DH % 64 != 0) rc = make_attn_tensor_map(&m.m32, base, DH, H, N, B, sr, sb, 16, rows, false);
  else m.m32 = m.m128;
  return rc;
}

// ---- device: tensor-map load into shared memory, completion on an mbarrier ----
__device__ __forceinline__ void tma_load_4d(void* sdst, const CUtensorMap* map, uint64_t* bar, int c0, int c1, int c2,
                                            int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
      ::"r"(smem_u32(sdst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* map) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(map) : "memory");
}

// ---- operand-tile geometry (the row count of a tile is a multiple of 8: whole swizzle atoms) ----
template <int DH, int ROWS = 128>
struct TileParts {
  static_assert(DH % 8 == 0, "head dim must be a multiple of 8 (16-byte rows)");
  static_assert(ROWS % 8 == 0 && ROWS <= 256, "tile rows");
  static constexpr int N64 = DH >= 64 ? DH / 64 : 1;   // SW128 parts
  static constexpr int REM = DH >= 64 ? DH % 64 : 0;
  static_assert(REM % 16 == 0, "head dims above 64 must be 64*a + 16*b");
  static constexpr int N16 = REM / 16;                 // SW32 parts
  static constexpr int DHP = DH >= 64 ? DH : (DH + 15) / 16 * 16;  // extent seen by the MMA (zero-padded below 64)
  static constexpr int KS64 = DH >= 64 ? 4 : DHP / 16;             // k16 steps per SW128 part when DH is the K dim
  static constexpr int W64 = DH >= 64 ? 64 : DHP;                  // N extent per SW128 part when DH is the N dim
  static constexpr int P64 = ROWS * 128, P16 = ROWS * 32;          // bytes per part
  static constexpr int BYTES = N64 * P64 + N16 * P16;
  static constexpr int KSTEPS = N64 * KS64 + N16;
  __host__ __device__ static constexpr int part64_off(int p) { return p * P64; }
  __host__ __device__ static constexpr int part16_off(int p) { return N64 * P64 + p * P16; }
};

// one thread: issue the loads of one [ROWS][DH] tile (rows r0.. of head h, frame b); bytes = TileParts<DH, ROWS>::BYTES.
// The maps' box height must be ROWS.
template <int DH, int ROWS = 128>
__device__ __forceinline__ void tma_load_tile(uint8_t* sdst, const CUtensorMap* map128, const CUtensorMap* map32,
                                              uint64_t* bar, int r0, int h, int b) {
  using T = TileParts<DH, ROWS>;
#pragma unroll
  for (int p = 0; p < T::N64; ++p) tma_load_4d(sdst + T::part64_off(p), map128, bar, p * 64, h, r0, b);
#pragma unroll
  for (int p = 0; p < T::N16; ++p) tma_load_4d(sdst + T::part16_off(p), map32, bar, T::N64 * 64 + p * 16, h, r0, b);
}

// ---- swizzled wgmma descriptors ----
// K-major SW128 part, k16 step ks (0..3): rows 128 B apart, 8-row groups 1024 B apart, 32 B per k step
__device__ __forceinline__ uint64_t desc_k128(uint32_t part_addr, int ks) { return gmma_desc(part_addr + ks * 32, 16, 1024, 1); }
// K-major SW32 part (one k16 step): rows 32 B apart, 8-row groups 256 B apart
__device__ __forceinline__ uint64_t desc_k32(uint32_t part_addr) { return gmma_desc(part_addr, 16, 256, 3); }
// MN-major SW128 part (64 elements wide), k16 step ks over the ROWS (16 rows = 2048 B): 8-row groups 1024 B apart
__device__ __forceinline__ uint64_t desc_mn128(uint32_t part_addr, int ks) { return gmma_desc(part_addr + ks * 2048, 16384, 1024, 1); }
// MN-major SW32 part (16 elements wide), k16 step ks over the rows (16 rows = 512 B): 8-row groups 256 B apart
__device__ __forceinline__ uint64_t desc_mn32(uint32_t part_addr, int ks) { return gmma_desc(part_addr + ks * 512, 4096, 256, 3); }

__host__ __device__ constexpr int align1k(int bytes) { return (bytes + 1023) / 1024 * 1024; }

// D[64 x BN] (+)= A B^T with A = rows arow0 .. arow0 + 63 of an [AROWS][DH] tile and B = a [BN][DH] tile, both K-major
// (the head dim is contracted). Issues the wgmma chain; the caller fences, commits and waits.
template <int DH, int AROWS, int BN>
__device__ __forceinline__ void gemm_kk(float* d, uint32_t sA, int arow0, uint32_t sB) {
  using TA = TileParts<DH, AROWS>;
  using TB = TileParts<DH, BN>;
  int acc = 0;
#pragma unroll
  for (int p = 0; p < TA::N64; ++p)
#pragma unroll
    for (int ks = 0; ks < TA::KS64; ++ks) {
      wgmma_ss<BN>(d, desc_k128(sA + TA::part64_off(p) + arow0 * 128, ks), desc_k128(sB + TB::part64_off(p), ks), acc);
      acc = 1;
    }
#pragma unroll
  for (int p = 0; p < TA::N16; ++p) {
    wgmma_ss<BN>(d, desc_k32(sA + TA::part16_off(p) + arow0 * 32), desc_k32(sB + TB::part16_off(p)), acc);
    acc = 1;
  }
}

// D[64 x ACC_W] (+)= A B with A = fp16 fragments in registers (KR / 16 k16 steps of 4 registers) and B = a [KR][DH] tile
// read MN-major (its rows are contracted). ACC_W = 64 per SW128 part (columns past DH come out as 0) + 16 per SW32 part;
// the accumulator's 8-column block i is output columns 8i .. 8i + 7 across the parts.
template <int DH>
struct AccW {
  using T = TileParts<DH, 64>;
  static constexpr int W = T::N64 * 64 + T::N16 * 16;
  static constexpr int REGS = W / 2;
};
template <int DH, int KR>
__device__ __forceinline__ void gemm_rmn(float* d, const uint32_t* a, uint32_t sB) {
  using TB = TileParts<DH, KR>;
#pragma unroll
  for (int ks = 0; ks < KR / 16; ++ks) {
#pragma unroll
    for (int p = 0; p < TB::N64; ++p) wgmma_rs<64>(d + p * 32, a + 4 * ks, desc_mn128(sB + TB::part64_off(p), ks), 1);
#pragma unroll
    for (int p = 0; p < TB::N16; ++p)
      wgmma_rs<16>(d + TB::N64 * 32 + p * 8, a + 4 * ks, desc_mn32(sB + TB::part16_off(p), ks), 1);
  }
}

__device__ __forceinline__ float ex2_approx(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// exp2 on the FMA pipe instead of the MUFU unit, for a fixed fraction of the softmax exponentials (the two units then
// share the work). x = n + f with n = round(x) by the 1.5 * 2^23 trick (the integer lands in the low mantissa bits),
// 2^f on [-0.5, 0.5] by the degree-4 minimax polynomial (max relative error 2.7e-6; the probabilities are rounded to fp16,
// half-ulp 4.9e-4, right after), 2^n by adding n << 23 to the exponent field. Inputs are clamped at -126 (result 2^-126:
// 0 in fp16).
__device__ __forceinline__ float ex2_poly(float s, float c, float negm) {
  constexpr float k4 = 0.009570101276040077f;
  constexpr float k3 = 0.05591786280274391f;
  constexpr float k2 = 0.240247443318367f;
  constexpr float k1 = 0.6931217908859253f;
  constexpr float k0 = 0.9999992847442627f;
  const float x = fmaxf(fmaf(s, c, negm), -126.f);
  const float t = __fadd_rn(x, 12582912.f);
  const float f = __fsub_rn(x, __fadd_rn(t, -12582912.f));  // f = x - round(x)
  float p = fmaf(k4, f, k3);
  p = fmaf(p, f, k2);
  p = fmaf(p, f, k1);
  p = fmaf(p, f, k0);
  return __uint_as_float(__float_as_uint(p) + (__float_as_uint(t) << 23));
}
// Every MC_EX2_POLY_PERIOD-th pair of an unrolled softmax loop takes the polynomial (0: none).
#ifndef MC_EX2_POLY_PERIOD
#define MC_EX2_POLY_PERIOD 4
#endif
__device__ __forceinline__ void ex2_pair(int pair_index, float s0, float s1, float c, float negm, float& p0, float& p1) {
  if (MC_EX2_POLY_PERIOD > 0 && pair_index % (MC_EX2_POLY_PERIOD > 0 ? MC_EX2_POLY_PERIOD : 1) == (MC_EX2_POLY_PERIOD - 1)) {
    p0 = ex2_poly(s0, c, negm);
    p1 = ex2_poly(s1, c, negm);
  } else {
    p0 = ex2_approx(fmaf(s0, c, negm));
    p1 = ex2_approx(fmaf(s1, c, negm));
  }
}

}  // namespace mc
