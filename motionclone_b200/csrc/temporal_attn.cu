// Fused temporal self-attention over the frame axis (forward + backward) for sm_90a.
//
// Replaces VersatileAttention's core (reference models/motion_module.py:309-332 -> models/attention.py:461-490), the
// second softmax pass of get_temp_attn_prob (utils/motionclone_functions.py:260-283 -> models/attention.py:564-611),
// torch.topk(k=1) (utils/motionclone_functions.py:79) and torch.gather (…:92) — one pass over Q, K, V.
//
// Shape of the problem: per (batch, position, head) a 16x16 (L x L, L in 1..32) attention with DH in [8,160]:
// arithmetic intensity L/2 flop/byte => HBM-bound (DESIGN.md §4, T1/T2). One CTA stages a tile of
// (all L frames) x (P positions) x (HG heads) of Q, K, V in shared memory with 1-D bulk copies (TMA engine, UBLKCP)
// signalled on mbarriers; each warp owns (position, head) items: QK^T, the fp16-rounded softmax and PV run on
// m16n8k16 tensor-core fragments straight out of ldmatrix, O is written back over Q's tile and leaves with bulk
// stores. A wgmma tile (M >= 64) would have to pad 16-row problems 4-8x for an op that has
// 8 flop/byte to spend; see DESIGN.md §4 (T1/T2) for the arithmetic behind this choice.
//
// The frame pitch in shared memory is padded to 16 (mod 128) bytes so the 8 row addresses of every ldmatrix phase
// fall in 8 different 16 B bank groups (rows of one (position, head) item are `pitch` apart).
//
// Clip lengths other than 8, 16 and 32 frames run "ragged" in the next larger tile (LP = 8 for L <= 8, 16 for L <= 16,
// 32 otherwise), in separate instantiations (RAGGED = true) so the tile lengths themselves keep their machine code:
// only frames 0..L-1 are copied in and out, frames L..LP-1 of every staged tile are zero-filled, key columns >= L are
// left out of the softmax (probability exactly 0) and no per-row output or input is touched for a frame >= L.
#include <math.h>
#include <stdlib.h>

#include <type_traits>

#include "mc_common.cuh"

// The file can be compiled as four translation units (build time): -DMC_TA_PART=1 keeps the forward entry point and its
// tile-length instantiations, =2 the backward ones, =3 / =4 the ragged forward / backward instantiations; undefined / 0
// keeps everything.
#ifndef MC_TA_PART
#define MC_TA_PART 0
#endif

namespace mc {

constexpr int kHeaderBytes = 128;

// L is the tile length (8, 16 or 32). RAGGED: the clip has fewer frames than the tile (TAParams::L at run time).
template <int DH_, int L_, bool RAGGED_ = false>
struct TACfg {
  static constexpr int DH = DH_;
  static constexpr int L = L_;
  static constexpr bool RAGGED = RAGGED_;
  static constexpr int MT = (L + 15) / 16;           // 16-row query tiles per item
  static constexpr int NKT = (L == 8) ? 2 : L / 8;   // 8-wide key tiles in the score fragment
  static constexpr int KK = (L == 8) ? 1 : L / 16;   // k16 steps over keys (P V, dS K, ...)
  static constexpr int PP = (L == 8) ? 2 : 1;        // positions packed into one 16-row item
  static constexpr int NDT = DH / 8;                 // 8-wide tiles over the head dim
  static constexpr int KS = DH / 16;                 // k16 steps over the head dim
  static constexpr bool KTAIL = (DH % 16) == 8;      // one extra k8 step
  static_assert(DH % 8 == 0 && DH >= 8, "head dim must be a multiple of 8");
  static_assert(L == 8 || L == 16 || L == 32, "L in {8,16,32}");
};

struct TileGeom {
  int P, HG, W;        // positions / heads per tile, W = HG*DH halfs per (frame, position) row of ONE tensor
  int PS;              // halfs between positions inside a staged row: W, or 3W when Q|K|V are staged as one run
  int fused;           // 1: q, k, v are column slices of one [.., 3C] buffer and the tile holds all heads ->
                       //    ONE bulk copy per frame brings P positions x (Q|K|V) (P*3C*2 bytes)
  int pitch;           // bytes between frames in the Q/K/V tile(s)
  int pitch_x;         // bytes between frames in the extra tile of the backward (dO): rows of P*W halfs
  int tensor_bytes;    // bytes of one staged Q/K/V tensor (separate mode) or of the fused tile
  int x_bytes;         // bytes of the extra tile
};

// Compile-time twin of TileGeom for the tile shapes the SD1.5 UNet actually produces (P = 1; all 8 heads as one fused
// Q|K|V run, or a 2/4-head group staged per tensor): every shared-memory address in the item loop becomes an immediate,
// and the item -> (position, head) split needs no integer division. Any other shape runs on the runtime TileGeom.
constexpr int pad16c(int row_bytes) { return row_bytes + ((16 - (row_bytes % 128)) + 128) % 128; }

template <int DH, int L, int P_, int HG_, bool FUSED>
struct CGeom {
  static constexpr int P = P_, HG = HG_, W = HG_ * DH, PS = FUSED ? 3 * HG_ * DH : HG_ * DH, fused = FUSED ? 1 : 0;
  static constexpr int pitch = pad16c(P_ * PS * 2), pitch_x = pad16c(P_ * W * 2);
  static constexpr int tensor_bytes = (L * pitch + 127) / 128 * 128, x_bytes = (L * pitch_x + 127) / 128 * 128;
};

struct TAParams {
  const __half *q, *k, *v;
  const __half* d_o;          // bwd only
  __half *o, *dq, *dk, *dv;   // fwd: o; bwd: dq, dk, dv
  mc_temporal_layout in, out, dol;
  __half* probs;              // fwd out [B*D,H,L,L]
  const __half* d_probs;      // bwd in
  __half* top_val;
  uint8_t* top_idx;
  const uint8_t* gather_idx;
  __half* gathered;           // fwd out [B*D,H,L]
  const __half* d_gathered;   // bwd in
  int B, D, H;
  TileGeom g;
  float scale;
  int L;                      // frames of the clip (<= the tile length; read by the ragged instantiations only)
};

// Byte offset (inside one staged tensor) of "virtual row" idx of an item whose first position is pl0.
// L >= 16: idx is the frame.  L == 8: two positions are packed, idx = 8*(position in pair) + frame; when the tile
// holds an odd number of positions the last one is paired with itself (duplicate rows compute and store identical
// values).
template <int L, typename G>
__device__ __forceinline__ uint32_t vrow_off(int idx, int pl0, const G& g) {
  if (L == 8) return (idx & 7) * g.pitch + (min(pl0 + (idx >> 3), g.P - 1) * g.PS) * 2;  // odd tail: pair with itself
  return idx * g.pitch + (pl0 * g.PS) * 2;
}
// same for the extra (dO / dQ) tile of the backward, whose rows are always P*W halfs
template <int L, typename G>
__device__ __forceinline__ uint32_t xrow_off(int idx, int pl0, const G& g) {
  if (L == 8) return (idx & 7) * g.pitch_x + (min(pl0 + (idx >> 3), g.P - 1) * g.W) * 2;
  return idx * g.pitch_x + (pl0 * g.W) * 2;
}

// Stage `ntensors` tensors (same layout) of this CTA's tile: rows of W halfs per (frame, position).
// rows of `w` halfs per (frame, position); smem: frame pitch `spitch` bytes, position stride `sps` halfs.
// When positions are contiguous on both sides (global stride_p == w == sps) one copy per frame moves all P of them.
// `nf`: frames 0..nf-1 are copied (the clip length; a compile-time constant outside the ragged instantiations).
__device__ __forceinline__ void stage_rows(int nf, uint8_t* sdst, int spitch, int sps, int w, int P, const __half* gsrc,
                                           const mc_temporal_layout& lay, int64_t gbase, uint64_t* bar, int lane) {
  const bool merged = (lay.stride_p == w) && (sps == w);
  const int ncopies = merged ? nf : nf * P;
  const uint32_t bytes = (merged ? P : 1) * w * 2;
  for (int i = lane; i < ncopies; i += 32) {
    const int f = merged ? i : i / P;
    const int pl = merged ? 0 : i % P;
    bulk_g2s(sdst + f * spitch + pl * sps * 2, gsrc + gbase + f * lay.stride_f + pl * lay.stride_p, bytes, bar);
  }
}

__device__ __forceinline__ void store_rows(int nf, __half* gdst, const uint8_t* ssrc, int spitch, int sps, int w, int P,
                                           const mc_temporal_layout& lay, int64_t gbase, int lane) {
  const bool merged = (lay.stride_p == w) && (sps == w);
  const int ncopies = merged ? nf : nf * P;
  const uint32_t bytes = (merged ? P : 1) * w * 2;
  for (int i = lane; i < ncopies; i += 32) {
    const int f = merged ? i : i / P;
    const int pl = merged ? 0 : i % P;
    bulk_s2g(gdst + gbase + f * lay.stride_f + pl * lay.stride_p, ssrc + f * spitch + pl * sps * 2, bytes);
  }
}

// Ragged tiles: zero frames nf..L-1 of `ntiles` staged tiles (`stride` bytes apart, frames `pitch` bytes apart) with
// ordinary stores, so that the padded rows and key columns hold zeros rather than whatever shared memory held before
// (a NaN pattern there would survive 0 * NaN in P V). Every thread of the CTA takes part.
__device__ __forceinline__ void zero_frames(uint8_t* base, int ntiles, int stride, int pitch, int nf, int L) {
  const int chunks = (L - nf) * pitch / 16;  // pitch is a multiple of 16 bytes
  for (int i = threadIdx.x; i < ntiles * chunks; i += blockDim.x) {
    const int tile = i / chunks, c = i % chunks;
    *reinterpret_cast<uint4*>(base + tile * stride + nf * pitch + c * 16) = make_uint4(0u, 0u, 0u, 0u);
  }
}

// S[mt] = Q K^T for one 16-row query tile: s[nt][0..3] in the m16n8 accumulator layout.
template <int L, bool X, typename G>
__device__ __forceinline__ uint32_t row_off(int idx, int pl0, const G& g) {
  return X ? xrow_off<L>(idx, pl0, g) : vrow_off<L>(idx, pl0, g);
}

// AX / BX: operand lives in the extra (dO) tile rather than in the Q/K/V tile(s)
template <typename C, bool AX = false, bool BX = false, typename G>
__device__ __forceinline__ void qk_scores(float (&s)[C::NKT][4], uint32_t sQ, uint32_t sK, int mt, int pl0,
                                          int colbase, const G& g, int lane) {
#pragma unroll
  for (int nt = 0; nt < C::NKT; ++nt)
#pragma unroll
    for (int e = 0; e < 4; ++e) s[nt][e] = 0.f;
  const int m = lane >> 3, r8 = lane & 7;
  const uint32_t a_row = sQ + row_off<C::L, AX>(mt * 16 + r8 + (m & 1) * 8, pl0, g) + (colbase + (m >> 1) * 8) * 2;
#pragma unroll
  for (int ks = 0; ks < C::KS; ++ks) {
    uint32_t a0, a1, a2, a3;
    ldsm_x4(a0, a1, a2, a3, a_row + ks * 32);
#pragma unroll
    for (int nt = 0; nt < C::NKT; nt += 2) {
      uint32_t b0, b1, b2, b3;
      const uint32_t b_row =
          sK + row_off<C::L, BX>((nt + (m >> 1)) * 8 + r8, pl0, g) + (colbase + ks * 16 + (m & 1) * 8) * 2;
      ldsm_x4(b0, b1, b2, b3, b_row);
      mma_16816(s[nt], a0, a1, a2, a3, b0, b1);
      mma_16816(s[nt + 1], a0, a1, a2, a3, b2, b3);
    }
  }
  if (C::KTAIL) {
    const int m2 = (lane >> 3) & 1;
    uint32_t a0, a1;
    ldsm_x2(a0, a1, sQ + row_off<C::L, AX>(mt * 16 + r8 + m2 * 8, pl0, g) + (colbase + C::DH - 8) * 2);
#pragma unroll
    for (int nt = 0; nt < C::NKT; nt += 2) {
      uint32_t b0, b1;
      ldsm_x2(b0, b1, sK + row_off<C::L, BX>((nt + m2) * 8 + r8, pl0, g) + (colbase + C::DH - 8) * 2);
      mma_1688(s[nt], a0, a1, b0);
      mma_1688(s[nt + 1], a0, a1, b1);
    }
  }
}

// In place: s <- fp16-rounded probabilities (as fp32 values). Rounding points follow models/attention.py:466-483:
// scores -> fp16 (baddbmm output), softmax in fp32 with the butterfly summation order of ATen's warp softmax,
// probabilities -> fp16.
// Ragged tiles (nf < L keys): key columns >= nf are left out of the row max and contribute an exact +0 to the sum, so
// the summation tree over L columns gives the same partial sums as ATen's warp softmax over nf columns, which pads a
// row to next_pow2(nf) lanes with -inf (exp -> 0) and reduces with xor offsets from the largest down.
template <typename C>
__device__ __forceinline__ bool key_valid(int nt, int hf, int e, int t, int nf) {
  const bool in_tile = (C::L != 8) || (nt == hf);
  return in_tile && (!C::RAGGED || (C::L == 8 ? 0 : nt * 8) + 2 * t + e < nf);
}

template <typename C>
__device__ __forceinline__ void softmax_rows(float (&s)[C::NKT][4], float scale, int nf, int lane) {
  const int t = lane & 3;
#pragma unroll
  for (int hf = 0; hf < 2; ++hf) {
    float x[C::NKT][2];
    float mx = -INFINITY;
#pragma unroll
    for (int nt = 0; nt < C::NKT; ++nt) {
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        x[nt][e] = round_half(s[nt][2 * hf + e] * scale);
        if (C::RAGGED && !key_valid<C>(nt, hf, e, t, nf)) x[nt][e] = -INFINITY;  // exp -> exactly +0
        if (key_valid<C>(nt, hf, e, t, nf)) mx = fmaxf(mx, x[nt][e]);
      }
    }
    mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
    mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
#pragma unroll
    for (int nt = 0; nt < C::NKT; ++nt)
#pragma unroll
      for (int e = 0; e < 2; ++e) x[nt][e] = expf(x[nt][e] - mx);
    float z[2];
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      if (C::L == 32)
        z[e] = (x[0][e] + x[2][e]) + (x[1][e] + x[3][e]);
      else if (C::L == 16)
        z[e] = x[0][e] + x[1][e];
      else
        z[e] = x[hf][e];
      z[e] += __shfl_xor_sync(0xffffffffu, z[e], 2);
      z[e] += __shfl_xor_sync(0xffffffffu, z[e], 1);
    }
    const float sum = z[0] + z[1];
    // x / sum, correctly rounded, with ONE reciprocal per row: y = RN(1/sum), q = RN(x y), r = x - q sum (exact, fma),
    // q' = RN(q + r y) is RN(x / sum) (Markstein) for the operands that occur here (1 <= sum <= L, 0 <= x <= 1; an x so
    // small that r underflows gives an fp16 zero either way). Bit-identical to ATen's `exp(x - max) / sum` and ~2x
    // fewer instructions than L independent IEEE divisions.
    const float y = __frcp_rn(sum);
#pragma unroll
    for (int nt = 0; nt < C::NKT; ++nt) {
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const float q0 = x[nt][e] * y;
        const float q1 = fmaf(fmaf(-q0, sum, x[nt][e]), y, q0);
        s[nt][2 * hf + e] = key_valid<C>(nt, hf, e, t, nf) ? round_half(q1) : 0.f;
      }
    }
  }
}

// acc[nd][.] += A(16 x keys, register fragments pa[kk][0..3]) * T(keys x DH) with T row-major in smem (V, K, Q, dO)
template <typename C, bool TX = false, typename G>
__device__ __forceinline__ void mma_a_rowmajor_b(float (&acc)[C::NDT][4], const uint32_t (&pa)[C::KK][4],
                                                 uint32_t sT, int pl0, int colbase, const G& g, int lane) {
  const int m = lane >> 3, r8 = lane & 7;
#pragma unroll
  for (int kk = 0; kk < C::KK; ++kk) {
#pragma unroll
    for (int n0 = 0; n0 + 1 < C::NDT; n0 += 2) {
      uint32_t b0, b1, b2, b3;
      ldsm_x4_t(b0, b1, b2, b3,
                sT + row_off<C::L, TX>(kk * 16 + (m & 1) * 8 + r8, pl0, g) + (colbase + (n0 + (m >> 1)) * 8) * 2);
      mma_16816(acc[n0], pa[kk][0], pa[kk][1], pa[kk][2], pa[kk][3], b0, b1);
      mma_16816(acc[n0 + 1], pa[kk][0], pa[kk][1], pa[kk][2], pa[kk][3], b2, b3);
    }
    if (C::NDT & 1) {
      uint32_t b0, b1;
      ldsm_x2_t(b0, b1,
                sT + row_off<C::L, TX>(kk * 16 + ((lane >> 3) & 1) * 8 + r8, pl0, g) + (colbase + (C::NDT - 1) * 8) * 2);
      mma_16816(acc[C::NDT - 1], pa[kk][0], pa[kk][1], pa[kk][2], pa[kk][3], b0, b1);
    }
  }
}

// write a 16 x DH fp32 accumulator tile (query/key tile mt) as fp16 into a staged tensor, scaled by `mul`
template <typename C, bool TX = false, typename G>
__device__ __forceinline__ void store_acc(const float (&acc)[C::NDT][4], float mul, uint8_t* sT_generic, int mt,
                                          int pl0, int colbase, const G& g, int lane) {
  const int gq = lane >> 2, t = lane & 3;
#pragma unroll
  for (int hf = 0; hf < 2; ++hf) {
    uint8_t* row = sT_generic + row_off<C::L, TX>(mt * 16 + gq + 8 * hf, pl0, g) + (colbase + 2 * t) * 2;
#pragma unroll
    for (int nd = 0; nd < C::NDT; ++nd)
      *reinterpret_cast<__half2*>(row + nd * 16) = __floats2half2_rn(acc[nd][2 * hf] * mul, acc[nd][2 * hf + 1] * mul);
  }
}

// fragments of P (or dS) as the A operand: pa[kk] = rows x keys[kk*16 .. +16)
template <typename C>
__device__ __forceinline__ void probs_to_afrag(uint32_t (&pa)[C::KK][4], const float (&p)[C::NKT][4]) {
#pragma unroll
  for (int kk = 0; kk < C::KK; ++kk) {
    pa[kk][0] = pack_half2(p[2 * kk][0], p[2 * kk][1]);
    pa[kk][1] = pack_half2(p[2 * kk][2], p[2 * kk][3]);
    pa[kk][2] = pack_half2(p[2 * kk + 1][0], p[2 * kk + 1][1]);
    pa[kk][3] = pack_half2(p[2 * kk + 1][2], p[2 * kk + 1][3]);
  }
}

// row bookkeeping of an item: global row index R = ((b*D + pos)*H + h)*nf + frame for accumulator half hf of tile mt
// (nf: frames of the clip, the row stride of every per-row tensor)
template <typename C>
__device__ __forceinline__ int64_t out_row(int b, int p_first, int p_last, int h, int mt, int gq, int hf, int D,
                                           int H, int nf) {
  if (C::L == 8) return ((int64_t)(b * D + min(p_first + hf, p_last)) * H + h) * nf + gq;
  return ((int64_t)(b * D + p_first) * H + h) * nf + mt * 16 + gq + 8 * hf;
}
// frame of that row; a ragged tile's rows at frames >= nf are padding and neither load nor store per-row data
template <typename C>
__device__ __forceinline__ int row_frame(int mt, int gq, int hf) {
  return C::L == 8 ? gq : mt * 16 + gq + 8 * hf;
}

// ================================================================================================================
// forward
// ================================================================================================================
// One (position[-pair], head) item of the forward: scores, softmax, per-row by-products, O = P V over the item's Q rows.
// `bar_v` (nullable): barrier of a separately staged V, waited on first use.
template <typename C, typename G>
__device__ __forceinline__ void fwd_item(const TAParams& prm, const G& g, uint8_t* sQ, uint32_t sQa, uint32_t sKa,
                                         uint32_t sVa, int b, int p0, int h0, int item, int lane, bool has_o,
                                         uint64_t* bar_v, bool& v_ready, int nf) {
  constexpr int DH = C::DH;
  constexpr int L = C::L;
  const int gq = lane >> 2, t = lane & 3;
  const int pl0 = (item / g.HG) * C::PP;
  const int hl = item % g.HG;
  const int colbase = hl * DH;
  const int h = h0 + hl;
#pragma unroll
  for (int mt = 0; mt < C::MT; ++mt) {
    float s[C::NKT][4];
    qk_scores<C>(s, sQa, sKa, mt, pl0, colbase, g, lane);
    softmax_rows<C>(s, prm.scale, nf, lane);

    // ---- per-row outputs: probabilities, top-1 (lowest index on ties), gathered probability ----
#pragma unroll
    for (int hf = 0; hf < 2; ++hf) {
      const int64_t R = out_row<C>(b, p0 + pl0, p0 + g.P - 1, h, mt, gq, hf, prm.D, prm.H, nf);
      const bool row_ok = !C::RAGGED || row_frame<C>(mt, gq, hf) < nf;
      if (prm.probs != nullptr && row_ok) {
        __half* prow = prm.probs + R * nf;
#pragma unroll
        for (int nt = 0; nt < C::NKT; ++nt) {
          if (L == 8 && nt != hf) continue;
          const int col = (L == 8 ? 0 : nt * 8) + 2 * t;
          if (C::RAGGED) {  // row R starts at R*nf halves: any parity, so 2-byte stores only
            if (col < nf) prow[col] = __float2half_rn(s[nt][2 * hf]);
            if (col + 1 < nf) prow[col + 1] = __float2half_rn(s[nt][2 * hf + 1]);
          } else {
            *reinterpret_cast<__half2*>(prow + col) = __floats2half2_rn(s[nt][2 * hf], s[nt][2 * hf + 1]);
          }
        }
      }
      if (prm.top_val != nullptr) {
        float bv = -1.f;
        int bi = 0;
#pragma unroll
        for (int nt = 0; nt < C::NKT; ++nt) {
          if (L == 8 && nt != hf) continue;
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const float pv = s[nt][2 * hf + e];
            const int col = (L == 8 ? 0 : nt * 8) + 2 * t + e;
            if (C::RAGGED && col >= nf) continue;
            if (pv > bv) {
              bv = pv;
              bi = col;
            }
          }
        }
#pragma unroll
        for (int off = 1; off <= 2; off <<= 1) {
          const float ov = __shfl_xor_sync(0xffffffffu, bv, off);
          const int oi = __shfl_xor_sync(0xffffffffu, bi, off);
          if (ov > bv || (ov == bv && oi < bi)) {
            bv = ov;
            bi = oi;
          }
        }
        if (t == 0 && row_ok) {
          prm.top_val[R] = __float2half_rn(bv);
          prm.top_idx[R] = (uint8_t)bi;
        }
      }
      if (prm.gathered != nullptr && row_ok) {
        const int gi = prm.gather_idx[R];
#pragma unroll
        for (int nt = 0; nt < C::NKT; ++nt) {
          if (L == 8 && nt != hf) continue;
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int col = (L == 8 ? 0 : nt * 8) + 2 * t + e;
            if (col == gi) prm.gathered[R] = __float2half_rn(s[nt][2 * hf + e]);
          }
        }
      }
    }

    // ---- O = P V, written over this item's Q rows ----
    if (has_o) {
      if (!v_ready) {
        if (bar_v != nullptr) mbar_wait(bar_v, 0);
        v_ready = true;
      }
      uint32_t pa[C::KK][4];
      probs_to_afrag<C>(pa, s);
      float acc[C::NDT][4];
#pragma unroll
      for (int nd = 0; nd < C::NDT; ++nd)
#pragma unroll
        for (int e = 0; e < 4; ++e) acc[nd][e] = 0.f;
      mma_a_rowmajor_b<C>(acc, pa, sVa, pl0, colbase, g, lane);
      __syncwarp();  // every lane's ldmatrix of this tile's Q rows has completed before they are overwritten
      store_acc<C>(acc, 1.f, sQ, mt, pl0, colbase, g, lane);
    }
  }
}

template <typename G>
__device__ __forceinline__ G load_geom(const TAParams& prm) {
  if constexpr (std::is_same<G, TileGeom>::value) {
    return prm.g;
  } else {
    return G{};
  }
}

template <int DH, int L, int NW, typename G = TileGeom, bool RAGGED = false>
__global__ void __launch_bounds__(NW * 32) temporal_attn_fwd_kernel(const TAParams prm) {
  using C = TACfg<DH, L, RAGGED>;
  extern __shared__ __align__(128) uint8_t smem[];
  uint64_t* bar_qk = reinterpret_cast<uint64_t*>(smem);
  uint64_t* bar_v = bar_qk + 1;
  const G g = load_geom<G>(prm);
  const int nf = RAGGED ? prm.L : L;  // frames of the clip
  uint8_t* sQ = smem + kHeaderBytes;
  uint8_t* sK = g.fused ? sQ + g.W * 2 : sQ + g.tensor_bytes;       // fused: K, V are column offsets of one tile
  uint8_t* sV = g.fused ? sQ + g.W * 4 : sQ + 2 * g.tensor_bytes;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n_hg = prm.H / g.HG, n_pt = prm.D / g.P;
  int bid = blockIdx.x;
  const int hg = bid % n_hg;
  bid /= n_hg;
  const int pt = bid % n_pt;
  const int b = bid / n_pt;
  const int p0 = pt * g.P, h0 = hg * g.HG;
  const bool has_o = prm.o != nullptr;

  if (threadIdx.x == 0) {
    mbar_init(bar_qk, 1);
    mbar_init(bar_v, 1);
    fence_mbar_init();
  }
  if (RAGGED) zero_frames(sQ, g.fused ? 1 : 3, g.tensor_bytes, g.pitch, nf, L);
  __syncthreads();
  if (warp == 0) {
    const uint32_t tbytes = (uint32_t)nf * g.P * g.W * 2;  // exactly the bytes the copies below bring in
    const int64_t gbase = (int64_t)b * prm.in.stride_b + (int64_t)p0 * prm.in.stride_p + h0 * DH;
    if (g.fused) {
      if (lane == 0) mbar_arrive_expect_tx(bar_qk, 3 * tbytes);
      __syncwarp();
      stage_rows(nf, sQ, g.pitch, g.PS, 3 * g.W, g.P, prm.q, prm.in, gbase, bar_qk, lane);
    } else {
      if (lane == 0) {
        mbar_arrive_expect_tx(bar_qk, 2 * tbytes);
        if (has_o) mbar_arrive_expect_tx(bar_v, tbytes);
      }
      __syncwarp();
      stage_rows(nf, sQ, g.pitch, g.PS, g.W, g.P, prm.q, prm.in, gbase, bar_qk, lane);
      stage_rows(nf, sK, g.pitch, g.PS, g.W, g.P, prm.k, prm.in, gbase, bar_qk, lane);
      if (has_o) stage_rows(nf, sV, g.pitch, g.PS, g.W, g.P, prm.v, prm.in, gbase, bar_v, lane);
    }
  }
  mbar_wait(bar_qk, 0);

  const int n_items = ((g.P + C::PP - 1) / C::PP) * g.HG;
  const uint32_t sQa = smem_u32(sQ), sKa = smem_u32(sK), sVa = smem_u32(sV);
  bool v_ready = false;

  for (int item = warp; item < n_items; item += NW)
    fwd_item<C>(prm, g, sQ, sQa, sKa, sVa, b, p0, h0, item, lane, has_o, g.fused ? nullptr : bar_v, v_ready, nf);

  if (has_o) {
    fence_proxy_async();
    __syncthreads();
    if (warp == 0) {
      const int64_t obase = (int64_t)b * prm.out.stride_b + (int64_t)p0 * prm.out.stride_p + h0 * DH;
      store_rows(nf, prm.o, sQ, g.pitch, g.PS, g.W, g.P, prm.out, obase, lane);
      bulk_commit();
      bulk_wait_read_all();
    }
  }
}

// ================================================================================================================
// backward: dq, dk, dv from d_o and/or the probability branches. Staged: Q, K, V, dO; outputs reuse dead tiles
// (dV -> V, dQ -> dO, dK -> K).
// ================================================================================================================
template <int DH, int L, int NW, typename G = TileGeom, bool RAGGED = false>
__global__ void __launch_bounds__(NW * 32) temporal_attn_bwd_kernel(const TAParams prm) {
  using C = TACfg<DH, L, RAGGED>;
  static_assert(C::MT == 1 || L == 32, "");
  extern __shared__ __align__(128) uint8_t smem[];
  uint64_t* bar_qk = reinterpret_cast<uint64_t*>(smem);
  uint64_t* bar_v = bar_qk + 1;
  const G g = load_geom<G>(prm);
  const int nf = RAGGED ? prm.L : L;  // frames of the clip
  uint8_t* sQ = smem + kHeaderBytes;
  uint8_t* sK = g.fused ? sQ + g.W * 2 : sQ + g.tensor_bytes;
  uint8_t* sV = g.fused ? sQ + g.W * 4 : sQ + 2 * g.tensor_bytes;
  uint8_t* sD = sQ + (g.fused ? 1 : 3) * g.tensor_bytes;  // extra tile: dO, later dQ
  // outputs as one [.., 3C] buffer too: dQ is moved next to dK, dV and each frame leaves with ONE bulk store
  const bool fused_out = g.fused && prm.out.stride_p == 3 * g.W && prm.dk == prm.dq + g.W &&
                         (prm.dv == nullptr || prm.dv == prm.dq + 2 * g.W);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n_hg = prm.H / g.HG, n_pt = prm.D / g.P;
  int bid = blockIdx.x;
  const int hg = bid % n_hg;
  bid /= n_hg;
  const int pt = bid % n_pt;
  const int b = bid / n_pt;
  const int p0 = pt * g.P, h0 = hg * g.HG;
  const bool has_do = prm.d_o != nullptr;

  if (threadIdx.x == 0) {
    mbar_init(bar_qk, 1);
    mbar_init(bar_v, 1);
    fence_mbar_init();
  }
  if (RAGGED) {
    zero_frames(sQ, g.fused ? 1 : 3, g.tensor_bytes, g.pitch, nf, L);
    zero_frames(sD, 1, 0, g.pitch_x, nf, L);  // zero dO rows: padded queries add nothing to dV = P^T dO
  }
  __syncthreads();
  if (warp == 0) {
    const uint32_t tbytes = (uint32_t)nf * g.P * g.W * 2;  // exactly the bytes the copies below bring in
    const int64_t gbase = (int64_t)b * prm.in.stride_b + (int64_t)p0 * prm.in.stride_p + h0 * DH;
    const int64_t dbase = (int64_t)b * prm.dol.stride_b + (int64_t)p0 * prm.dol.stride_p + h0 * DH;
    if (g.fused) {
      if (lane == 0) {
        mbar_arrive_expect_tx(bar_qk, 3 * tbytes);
        if (has_do) mbar_arrive_expect_tx(bar_v, tbytes);
      }
      __syncwarp();
      stage_rows(nf, sQ, g.pitch, g.PS, 3 * g.W, g.P, prm.q, prm.in, gbase, bar_qk, lane);
      if (has_do) stage_rows(nf, sD, g.pitch_x, g.W, g.W, g.P, prm.d_o, prm.dol, dbase, bar_v, lane);
    } else {
      if (lane == 0) {
        mbar_arrive_expect_tx(bar_qk, 2 * tbytes);
        if (has_do) mbar_arrive_expect_tx(bar_v, 2 * tbytes);
      }
      __syncwarp();
      stage_rows(nf, sQ, g.pitch, g.PS, g.W, g.P, prm.q, prm.in, gbase, bar_qk, lane);
      stage_rows(nf, sK, g.pitch, g.PS, g.W, g.P, prm.k, prm.in, gbase, bar_qk, lane);
      if (has_do) {
        stage_rows(nf, sV, g.pitch, g.PS, g.W, g.P, prm.v, prm.in, gbase, bar_v, lane);
        stage_rows(nf, sD, g.pitch_x, g.W, g.W, g.P, prm.d_o, prm.dol, dbase, bar_v, lane);
      }
    }
  }
  mbar_wait(bar_qk, 0);
  if (has_do) mbar_wait(bar_v, 0);

  const int n_items = ((g.P + C::PP - 1) / C::PP) * g.HG;
  const uint32_t sQa = smem_u32(sQ), sKa = smem_u32(sK), sVa = smem_u32(sV), sDa = smem_u32(sD);
  const int gq = lane >> 2, t = lane & 3;

  for (int item = warp; item < n_items; item += NW) {
    const int pl0 = (item / g.HG) * C::PP;
    const int hl = item % g.HG;
    const int colbase = hl * DH;
    const int h = h0 + hl;

    // P and dS for every query tile, kept as A fragments (rows = queries)
    uint32_t pfrag[C::MT][C::KK][4];
    uint32_t dsfrag[C::MT][C::KK][4];
#pragma unroll
    for (int mt = 0; mt < C::MT; ++mt) {
      float p[C::NKT][4];
      qk_scores<C>(p, sQa, sKa, mt, pl0, colbase, g, lane);
      softmax_rows<C>(p, prm.scale, nf, lane);
      probs_to_afrag<C>(pfrag[mt], p);

      // dP = dO V^T  (+ dense d_probs, + one-hot d_gathered)
      float dp[C::NKT][4];
      if (has_do) {
        qk_scores<C, true, false>(dp, sDa, sVa, mt, pl0, colbase, g, lane);
#pragma unroll
        for (int nt = 0; nt < C::NKT; ++nt)
#pragma unroll
          for (int e = 0; e < 4; ++e) dp[nt][e] = round_half(dp[nt][e]);  // bmm backward output is fp16
      } else {
#pragma unroll
        for (int nt = 0; nt < C::NKT; ++nt)
#pragma unroll
          for (int e = 0; e < 4; ++e) dp[nt][e] = 0.f;
      }
#pragma unroll
      for (int hf = 0; hf < 2; ++hf) {
        const int64_t R = out_row<C>(b, p0 + pl0, p0 + g.P - 1, h, mt, gq, hf, prm.D, prm.H, nf);
        const bool row_ok = !C::RAGGED || row_frame<C>(mt, gq, hf) < nf;
        int gi = -1;
        float gv = 0.f;
        if (prm.d_gathered != nullptr && row_ok) {
          gi = prm.gather_idx[R];
          gv = __half2float(prm.d_gathered[R]);
        }
        float dot = 0.f;
#pragma unroll
        for (int nt = 0; nt < C::NKT; ++nt) {
          if (L == 8 && nt != hf) continue;
          const int col0 = (L == 8 ? 0 : nt * 8) + 2 * t;
          if (prm.d_probs != nullptr && row_ok) {
            if (C::RAGGED) {  // row R starts at R*nf halves: any parity, so 2-byte loads, columns < nf only
              const __half* drow = prm.d_probs + R * nf;
              if (col0 < nf) dp[nt][2 * hf] += __half2float(drow[col0]);
              if (col0 + 1 < nf) dp[nt][2 * hf + 1] += __half2float(drow[col0 + 1]);
            } else {
              const __half2 dd = *reinterpret_cast<const __half2*>(prm.d_probs + R * L + col0);
              dp[nt][2 * hf] += __low2float(dd);
              dp[nt][2 * hf + 1] += __high2float(dd);
            }
          }
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            if (col0 + e == gi) dp[nt][2 * hf + e] += gv;
            dot += dp[nt][2 * hf + e] * p[nt][2 * hf + e];
          }
        }
        dot += __shfl_xor_sync(0xffffffffu, dot, 1);
        dot += __shfl_xor_sync(0xffffffffu, dot, 2);
#pragma unroll
        for (int nt = 0; nt < C::NKT; ++nt) {
          const bool valid = (L != 8) || (nt == hf);
#pragma unroll
          for (int e = 0; e < 2; ++e)
            dp[nt][2 * hf + e] = valid ? p[nt][2 * hf + e] * (dp[nt][2 * hf + e] - dot) : 0.f;  // dS (softmax bwd)
        }
      }
      probs_to_afrag<C>(dsfrag[mt], dp);  // rounds dS to fp16, as the eager softmax backward does
    }
    __syncwarp();

    // ---- dV[key tile] = sum over query tiles of P^T dO ; A = P^T built with movmatrix ----
    if (has_do && prm.dv != nullptr) {
#pragma unroll
      for (int kt = 0; kt < C::MT; ++kt) {  // 16-key output tiles
        float acc[C::NDT][4];
#pragma unroll
        for (int nd = 0; nd < C::NDT; ++nd)
#pragma unroll
          for (int e = 0; e < 4; ++e) acc[nd][e] = 0.f;
        uint32_t at[C::KK][4];  // A = P^T: rows = keys of tile kt, k = queries; k16 step index = query tile
#pragma unroll
        for (int mt = 0; mt < C::MT; ++mt) {
          at[mt][0] = movmatrix_t(pfrag[mt][kt][0]);
          at[mt][1] = movmatrix_t(pfrag[mt][kt][2]);
          at[mt][2] = movmatrix_t(pfrag[mt][kt][1]);
          at[mt][3] = movmatrix_t(pfrag[mt][kt][3]);
        }
        mma_a_rowmajor_b<C, true>(acc, at, sDa, pl0, colbase, g, lane);
        // dV tile kt goes over V rows [kt*16, +16); V is still needed by nobody (dP done for all tiles above)
        store_acc<C>(acc, 1.f, sV, kt, pl0, colbase, g, lane);
      }
    }
    __syncwarp();

    // ---- dQ[query tile] = scale * dS K  -> over the dO rows of that tile (dO is dead: dP and dV are done) ----
#pragma unroll
    for (int mt = 0; mt < C::MT; ++mt) {
      float acc[C::NDT][4];
#pragma unroll
      for (int nd = 0; nd < C::NDT; ++nd)
#pragma unroll
        for (int e = 0; e < 4; ++e) acc[nd][e] = 0.f;
      mma_a_rowmajor_b<C>(acc, dsfrag[mt], sKa, pl0, colbase, g, lane);
      store_acc<C, true>(acc, prm.scale, sD, mt, pl0, colbase, g, lane);
    }
    __syncwarp();

    // ---- dK[key tile] = scale * dS^T Q -> over K rows (K is dead: every dQ tile of this item is done) ----
#pragma unroll
    for (int kt = 0; kt < C::MT; ++kt) {
      float acc[C::NDT][4];
#pragma unroll
      for (int nd = 0; nd < C::NDT; ++nd)
#pragma unroll
        for (int e = 0; e < 4; ++e) acc[nd][e] = 0.f;
      uint32_t at[C::KK][4];
#pragma unroll
      for (int mt = 0; mt < C::MT; ++mt) {
        at[mt][0] = movmatrix_t(dsfrag[mt][kt][0]);
        at[mt][1] = movmatrix_t(dsfrag[mt][kt][2]);
        at[mt][2] = movmatrix_t(dsfrag[mt][kt][1]);
        at[mt][3] = movmatrix_t(dsfrag[mt][kt][3]);
      }
      mma_a_rowmajor_b<C>(acc, at, sQa, pl0, colbase, g, lane);
      store_acc<C>(acc, prm.scale, sK, kt, pl0, colbase, g, lane);
    }
    if (fused_out) {  // Q is dead now: move this item's dQ rows (extra tile) over its Q columns, 16 B per lane-step
      __syncwarp();
      constexpr int kChunks = DH / 8;
      constexpr int kRows = (L == 8) ? 16 : L;
      for (int i = lane; i < kRows * kChunks; i += 32) {
        const int r = i / kChunks, ch = i % kChunks;
        const uint4 val = *reinterpret_cast<const uint4*>(sD + xrow_off<L>(r, pl0, g) + (colbase + ch * 8) * 2);
        *reinterpret_cast<uint4*>(sQ + vrow_off<L>(r, pl0, g) + (colbase + ch * 8) * 2) = val;
      }
    }
  }

  fence_proxy_async();
  __syncthreads();
  if (warp == 0) {
    const int64_t obase = (int64_t)b * prm.out.stride_b + (int64_t)p0 * prm.out.stride_p + h0 * DH;
    if (fused_out && (prm.dv != nullptr && has_do)) {
      store_rows(nf, prm.dq, sQ, g.pitch, g.PS, 3 * g.W, g.P, prm.out, obase, lane);  // dQ | dK | dV per frame
    } else if (fused_out) {  // no dV: two column blocks per (frame, position)
      store_rows(nf, prm.dq, sQ, g.pitch, g.PS, 2 * g.W, g.P, prm.out, obase, lane);
    } else {
      store_rows(nf, prm.dq, sD, g.pitch_x, g.W, g.W, g.P, prm.out, obase, lane);
      store_rows(nf, prm.dk, sK, g.pitch, g.PS, g.W, g.P, prm.out, obase, lane);
      if (has_do && prm.dv != nullptr) store_rows(nf, prm.dv, sV, g.pitch, g.PS, g.W, g.P, prm.out, obase, lane);
    }
    bulk_commit();
    bulk_wait_read_all();
  }
}

// ================================================================================================================
// host side
// ================================================================================================================
static int pad16(int row_bytes) { return row_bytes + ((16 - (row_bytes % 128)) + 128) % 128; }

// ntensors: 3 (fwd: Q,K,V) or 4 (bwd: + dO). `fusable`: q, k, v are the three column blocks of one [.., 3C] buffer.
static bool choose_geom(int D, int L, int H, int DH, int ntensors, bool need_even_p, bool fusable, TileGeom* g,
                        int n_batch = 0) {
  // Tile size: ~32 KB per Q/K/V set keeps 6-7 CTAs resident per SM (227 KB), which is what de-synchronises their
  // load / math / store phases.
  // Tiles that would hold fewer than 4 (position, head) items get twice the budget instead of idle warps.
  const int base = 32 * 1024 * ntensors / 3;
  auto tbytes = [&](int P, int hg) { return (int64_t)ntensors * L * P * hg * DH * 2; };
  const int Pmin = (need_even_p && D % 2 == 0) ? 2 : 1;  // L == 8 packs two positions per item; odd D: tail pairs with itself
  const int pp = need_even_p ? 2 : 1;
  int HG = H, P = Pmin, target = base;
  for (int attempt = 0; attempt < 2; ++attempt, target *= 2) {
    HG = H;
    while (HG > 1 && tbytes(Pmin, HG) > target && (HG % 2 == 0)) HG /= 2;
    P = Pmin;
    if (HG == H) {  // whole positions are contiguous runs: grow P while the tile stays within budget
      while (D % (P * 2) == 0 && tbytes(P * 2, HG) <= target && P < 8) P *= 2;
    }
    if (((P + pp - 1) / pp) * HG >= 4) break;
  }
  // Small layers (16x16 / 8x8 latent positions at C = 1280: 10-40 MB per launch) are bound by latency, not bandwidth: a
  // grid of less than two waves leaves SMs with one tile in flight. Halve the head group (down to 2 heads: half the
  // warps of a CTA then idle, which costs nothing here) until the launch has at least two waves of resident CTAs.
  if (n_batch > 0) {
    auto ctas = [&](int hg) { return (int64_t)n_batch * (D / P) * (H / hg); };
    auto resident = [&](int hg) { return (int64_t)132 * (227 * 1024 / (tbytes(P, hg) + 2048)); };
    while (HG > 2 && HG % 2 == 0 && ctas(HG) < 2 * resident(HG)) HG /= 2;
  }
  g->P = P;
  g->HG = HG;
  g->W = HG * DH;
  g->fused = (fusable && HG == H) ? 1 : 0;
  g->PS = g->fused ? 3 * g->W : g->W;
  g->pitch = pad16(P * g->PS * 2);
  g->pitch_x = pad16(P * g->W * 2);
  g->tensor_bytes = ((L * g->pitch) + 127) / 128 * 128;
  g->x_bytes = ((L * g->pitch_x) + 127) / 128 * 128;
  return true;
}

static int tile_smem(const TileGeom& g, int ntensors) {
  const int qkv = g.fused ? g.tensor_bytes : 3 * g.tensor_bytes;
  return kHeaderBytes + qkv + (ntensors == 4 ? g.x_bytes : 0);
}

static bool is_fusable(const TAParams& prm, int C) {
  return prm.v != nullptr && prm.k == prm.q + C && prm.v == prm.q + 2 * C && prm.in.stride_p == 3 * C;
}

static bool layout_ok(const mc_temporal_layout& l) {
  return l.stride_b % 8 == 0 && l.stride_f % 8 == 0 && l.stride_p % 8 == 0;
}

// Does the runtime geometry equal the compile-time one (then the constant-address kernel can take the launch)?
template <typename G>
static bool geom_matches(const TileGeom& g) {
  return g.P == G::P && g.HG == G::HG && g.W == G::W && g.PS == G::PS && g.fused == G::fused && g.pitch == G::pitch &&
         g.pitch_x == G::pitch_x && g.tensor_bytes == G::tensor_bytes && g.x_bytes == G::x_bytes;
}

// The tile shapes of the SD1.5 + motion-module UNet (8 heads; DH = 40 / 80 / 160; L = 16 or 32), see CGeom.
template <int DH, int L>
struct CGeomSet {
  static constexpr bool enabled = (DH == 40 || DH == 80 || DH == 160) && (L == 16 || L == 32);
  using Fused8 = CGeom<DH, L, 1, 8, true>;   // all 8 heads, one Q|K|V run per frame
  using Sep4 = CGeom<DH, L, 1, 4, false>;    // 4-head group, Q / K / V staged separately
  using Sep2 = CGeom<DH, L, 1, 2, false>;
};

template <int DH, int L, typename G, bool BWD>
static void launch_cgeom(const TAParams& prm, unsigned grid, int smem, cudaStream_t st) {
  if constexpr (BWD) {
    auto kern = temporal_attn_bwd_kernel<DH, L, 4, G>;
    cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    kern<<<grid, 4 * 32, smem, st>>>(prm);
  } else {
    auto kern = temporal_attn_fwd_kernel<DH, L, 4, G>;
    cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    kern<<<grid, 4 * 32, smem, st>>>(prm);
  }
}

// true if a constant-geometry instantiation took the launch (4-warp CTAs only: these tiles hold <= 8 items)
template <int DH, int L, bool BWD>
static bool try_launch_cgeom(const TAParams& prm, unsigned grid, int smem, int n_items, cudaStream_t st) {
  if constexpr (CGeomSet<DH, L>::enabled) {
    using S = CGeomSet<DH, L>;
    if (n_items >= 16 || prm.H != 8) return false;
    if (geom_matches<typename S::Fused8>(prm.g)) {
      launch_cgeom<DH, L, typename S::Fused8, BWD>(prm, grid, smem, st);
      return true;
    }
    if (geom_matches<typename S::Sep4>(prm.g)) {
      launch_cgeom<DH, L, typename S::Sep4, BWD>(prm, grid, smem, st);
      return true;
    }
    if (geom_matches<typename S::Sep2>(prm.g)) {
      launch_cgeom<DH, L, typename S::Sep2, BWD>(prm, grid, smem, st);
      return true;
    }
  }
  return false;
}

// L: the tile length; RAGGED: the clip has prm.L < L frames (runtime TileGeom only)
template <int DH, int L, bool RAGGED = false>
static int launch_fwd(TAParams& prm, cudaStream_t st) {
  choose_geom(prm.D, L, prm.H, DH, 3, L == 8, is_fusable(prm, prm.H * DH) && prm.o != nullptr, &prm.g, prm.B);
  const int smem = tile_smem(prm.g, 3);
  const int64_t grid = (int64_t)prm.B * (prm.D / prm.g.P) * (prm.H / prm.g.HG);
  const int n_items = ((prm.g.P + TACfg<DH, L>::PP - 1) / TACfg<DH, L>::PP) * prm.g.HG;
  bool launched = false;
  if constexpr (!RAGGED) launched = try_launch_cgeom<DH, L, false>(prm, (unsigned)grid, smem, n_items, st);
  if (launched) {
  } else if (n_items >= 16) {
    auto kern = temporal_attn_fwd_kernel<DH, L, 8, TileGeom, RAGGED>;
    cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    kern<<<(unsigned)grid, 8 * 32, smem, st>>>(prm);
  } else {
    auto kern = temporal_attn_fwd_kernel<DH, L, 4, TileGeom, RAGGED>;
    cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    kern<<<(unsigned)grid, 4 * 32, smem, st>>>(prm);
  }
  count_launch();
  return check_launch("temporal_attn_fwd");
}

template <int DH, int L, bool RAGGED = false>
static int launch_bwd(TAParams& prm, cudaStream_t st) {
  choose_geom(prm.D, L, prm.H, DH, 4, L == 8, is_fusable(prm, prm.H * DH), &prm.g, prm.B);
  const int smem = tile_smem(prm.g, 4);
  const int64_t grid = (int64_t)prm.B * (prm.D / prm.g.P) * (prm.H / prm.g.HG);
  const int n_items = ((prm.g.P + TACfg<DH, L>::PP - 1) / TACfg<DH, L>::PP) * prm.g.HG;
  bool launched = false;
  if constexpr (!RAGGED) launched = try_launch_cgeom<DH, L, true>(prm, (unsigned)grid, smem, n_items, st);
  if (launched) {
  } else if (n_items >= 16) {
    auto kern = temporal_attn_bwd_kernel<DH, L, 8, TileGeom, RAGGED>;
    cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    kern<<<(unsigned)grid, 8 * 32, smem, st>>>(prm);
  } else {
    auto kern = temporal_attn_bwd_kernel<DH, L, 4, TileGeom, RAGGED>;
    cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    kern<<<(unsigned)grid, 4 * 32, smem, st>>>(prm);
  }
  count_launch();
  return check_launch("temporal_attn_bwd");
}

#define MC_DISPATCH_DH(L_, FN, RG)                          \
  switch (DH) {                                             \
    case 8: return FN<8, L_, RG>(prm, st);                  \
    case 16: return FN<16, L_, RG>(prm, st);                \
    case 32: return FN<32, L_, RG>(prm, st);                \
    case 40: return FN<40, L_, RG>(prm, st);                \
    case 64: return FN<64, L_, RG>(prm, st);                \
    case 80: return FN<80, L_, RG>(prm, st);                \
    case 128: return FN<128, L_, RG>(prm, st);              \
    case 160: return FN<160, L_, RG>(prm, st);              \
    default: break;                                         \
  }

// Ragged launches (1 <= L <= 32, L not a tile length); they live in their own translation units (MC_TA_PART 3 / 4).
// MC_E_UNSUPPORTED (error message left to the caller) for a head dim without an instantiation.
int dispatch_fwd_ragged(TAParams& prm, int L, int DH, cudaStream_t st);
int dispatch_bwd_ragged(TAParams& prm, int L, int DH, cudaStream_t st);

#if MC_TA_PART == 0 || MC_TA_PART == 1
static int dispatch_fwd(TAParams& prm, int L, int DH, cudaStream_t st) {
  if (L == 8) { MC_DISPATCH_DH(8, launch_fwd, false) }
  if (L == 16) { MC_DISPATCH_DH(16, launch_fwd, false) }
  if (L == 32) { MC_DISPATCH_DH(32, launch_fwd, false) }
  if (L != 8 && L != 16 && L != 32) {
    const int rc = dispatch_fwd_ragged(prm, L, DH, st);
    if (rc != MC_E_UNSUPPORTED) return rc;
  }
  set_error("temporal_attn_fwd: unsupported L=%d / DH=%d (L in 1..32; DH in {8,16,32,40,64,80,128,160})", L, DH);
  return MC_E_UNSUPPORTED;
}

#endif
#if MC_TA_PART == 0 || MC_TA_PART == 2
static int dispatch_bwd(TAParams& prm, int L, int DH, cudaStream_t st) {
  if (L == 8) { MC_DISPATCH_DH(8, launch_bwd, false) }
  if (L == 16) { MC_DISPATCH_DH(16, launch_bwd, false) }
  if (L == 32) { MC_DISPATCH_DH(32, launch_bwd, false) }
  if (L != 8 && L != 16 && L != 32) {
    const int rc = dispatch_bwd_ragged(prm, L, DH, st);
    if (rc != MC_E_UNSUPPORTED) return rc;
  }
  set_error("temporal_attn_bwd: unsupported L=%d / DH=%d (L in 1..32; DH in {8,16,32,40,64,80,128,160})", L, DH);
  return MC_E_UNSUPPORTED;
}

#endif
#if MC_TA_PART == 0 || MC_TA_PART >= 3
// tile length a clip of L frames runs in
static int tile_len(int L) { return L <= 8 ? 8 : (L <= 16 ? 16 : 32); }

#endif
#if MC_TA_PART == 0 || MC_TA_PART == 3
int dispatch_fwd_ragged(TAParams& prm, int L, int DH, cudaStream_t st) {
  switch (tile_len(L)) {
    case 8: { MC_DISPATCH_DH(8, launch_fwd, true) } break;
    case 16: { MC_DISPATCH_DH(16, launch_fwd, true) } break;
    default: { MC_DISPATCH_DH(32, launch_fwd, true) } break;
  }
  return MC_E_UNSUPPORTED;
}

#endif
#if MC_TA_PART == 0 || MC_TA_PART == 4
int dispatch_bwd_ragged(TAParams& prm, int L, int DH, cudaStream_t st) {
  switch (tile_len(L)) {
    case 8: { MC_DISPATCH_DH(8, launch_bwd, true) } break;
    case 16: { MC_DISPATCH_DH(16, launch_bwd, true) } break;
    default: { MC_DISPATCH_DH(32, launch_bwd, true) } break;
  }
  return MC_E_UNSUPPORTED;
}

#endif
}  // namespace mc

#if MC_TA_PART == 0 || MC_TA_PART == 1
extern "C" int mc_temporal_attn_fwd(const void* q, const void* k, const void* v, mc_temporal_layout qkv_layout,
                                    void* o, mc_temporal_layout o_layout, void* probs, void* top_val,
                                    uint8_t* top_idx, const uint8_t* gather_idx, void* gathered, int B, int D, int L,
                                    int H, int DH, float scale, void* stream) {
  using namespace mc;
  if (L < 1 || L > 32) {  // the motion module's positional encoding has 32 entries (max_len)
    set_error("temporal_attn_fwd: L=%d frames outside the supported range 1..32", L);
    return MC_E_UNSUPPORTED;
  }
  if (!q || !k || (o && !v) || B <= 0 || D <= 0 || H <= 0) {
    set_error("temporal_attn_fwd: null q/k (or o without v) or non-positive dims");
    return MC_E_INVALID;
  }
  if ((top_val == nullptr) != (top_idx == nullptr) || (gathered != nullptr && gather_idx == nullptr)) {
    set_error("temporal_attn_fwd: top_val/top_idx must come together; gathered needs gather_idx");
    return MC_E_INVALID;
  }
  if (!layout_ok(qkv_layout) || (o && !layout_ok(o_layout))) {
    set_error("temporal_attn_fwd: strides must be multiples of 8 elements (16 B bulk-copy alignment)");
    return MC_E_INVALID;
  }
  TAParams prm{};
  prm.q = (const __half*)q;
  prm.k = (const __half*)k;
  prm.v = (const __half*)v;
  prm.o = (__half*)o;
  prm.in = qkv_layout;
  prm.out = o_layout;
  prm.probs = (__half*)probs;
  prm.top_val = (__half*)top_val;
  prm.top_idx = top_idx;
  prm.gather_idx = gather_idx;
  prm.gathered = (__half*)gathered;
  prm.B = B;
  prm.D = D;
  prm.H = H;
  prm.scale = scale;
  prm.L = L;
  return dispatch_fwd(prm, L, DH, (cudaStream_t)stream);
}

#endif
#if MC_TA_PART == 0 || MC_TA_PART == 2
extern "C" int mc_temporal_attn_bwd(const void* q, const void* k, const void* v, mc_temporal_layout qkv_layout,
                                    const void* d_o, mc_temporal_layout do_layout, const void* d_probs,
                                    const uint8_t* gather_idx, const void* d_gathered, void* dq, void* dk, void* dv,
                                    mc_temporal_layout g_layout, int B, int D, int L, int H, int DH, float scale,
                                    void* stream) {
  using namespace mc;
  if (L < 1 || L > 32) {  // the motion module's positional encoding has 32 entries (max_len)
    set_error("temporal_attn_bwd: L=%d frames outside the supported range 1..32", L);
    return MC_E_UNSUPPORTED;
  }
  if (!q || !k || !dq || !dk || (d_o && !v) || B <= 0 || D <= 0 || H <= 0) {
    set_error("temporal_attn_bwd: null q/k/dq/dk (or d_o without v) or non-positive dims");
    return MC_E_INVALID;
  }
  if (d_gathered != nullptr && gather_idx == nullptr) {
    set_error("temporal_attn_bwd: d_gathered needs gather_idx");
    return MC_E_INVALID;
  }
  if (!layout_ok(qkv_layout) || !layout_ok(g_layout) || (d_o && !layout_ok(do_layout))) {
    set_error("temporal_attn_bwd: strides must be multiples of 8 elements (16 B bulk-copy alignment)");
    return MC_E_INVALID;
  }
  TAParams prm{};
  prm.q = (const __half*)q;
  prm.k = (const __half*)k;
  prm.v = (const __half*)v;
  prm.d_o = (const __half*)d_o;
  prm.dq = (__half*)dq;
  prm.dk = (__half*)dk;
  prm.dv = (__half*)dv;
  prm.in = qkv_layout;
  prm.out = g_layout;
  prm.dol = do_layout;
  prm.d_probs = (const __half*)d_probs;
  prm.gather_idx = gather_idx;
  prm.d_gathered = (const __half*)d_gathered;
  prm.B = B;
  prm.D = D;
  prm.H = H;
  prm.scale = scale;
  prm.L = L;
  return dispatch_bwd(prm, L, DH, (cudaStream_t)stream);
}
#endif
