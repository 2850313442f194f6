// Attention forward on Hopper tensor cores (wgmma with register accumulators), operands staged by tensor-map TMA
// (cp.async.bulk.tensor), sm_90a. Serves two seams of the reference:
//   * spatial self-attention `attn1` (models/attention.py:190-192, :271-278 -> :535-542,
//     xformers.ops.memory_efficient_attention(q, k, v, attn_bias=None)): O = softmax(scale Q K^T) V per (frame, head)
//     over the N = h*w tokens of one frame; N = 4096 / 1024 / 256 / 64 and DH = 40 / 80 / 160 / 160 at 16 x 512 x 512;
//     the natural-log sum-exp of every query row is kept for the backward (csrc/spatial_attn_bwd_tc.cu);
//   * text cross-attention `attn2` (models/attention.py:193-201, :280-285): Q [b, f*N, C] (all frames of one prompt)
//     against the 77 text tokens K / V [b, 77, C].
// fp32 softmax statistics, one rounding of the output (xformers / flash semantics - SURVEY.md appendix "Attention
// numerics").
//
// One CTA = one (frame or batch, head, 128-query tile); 288 threads = 2 consumer warpgroups (64 query rows each) + 1
// producer warp whose lane 0 issues every TMA load. The Q tile is loaded once; K and V tiles of 64 keys stream through an
// NS-stage ring (full barriers: TMA transaction bytes; empty barriers: one arrival per consumer warp). Per key tile j a
// consumer warpgroup computes
//   S = Q K_j^T      wgmma m64n64k16, A = its 64 Q rows and B = K_j, both K-major from shared memory
//   online softmax   row max / sum across the 4 threads of a row quad, O rescaled in registers, P -> fp16 A fragments
//   O += P V_j       wgmma m64nWk16 with A = P from registers, B = V_j read MN-major straight from its TMA tile
// Keys past the end of the sequence are zero-filled by the TMA unit and masked to -inf in S.
#include <math.h>

#include "tma_common.cuh"

namespace mc {

constexpr int kFM = 128;                    // query rows per CTA
constexpr int kFBN = 64;                    // keys per tile
constexpr int kFWG = kFM / 64;              // consumer warpgroups
constexpr int kFThreads = kFWG * 128 + 32;  // + producer warp
constexpr int kFProducerWarp = kFWG * 4;

struct FAParams {
  float* lse;        // [B][H][Nq] natural-log sum-exp of the scaled scores (nullable)
  __half* o;
  int64_t o_sb, o_sr;
  int B, Nq, Nk, H;
  float scale_log2e;  // scale * log2(e)
};

template <int DH>
struct FACfg {
  using TQ = TileParts<DH, kFM>;
  using TK = TileParts<DH, kFBN>;
  static constexpr int ACC = AccW<DH>::REGS;       // O accumulator registers per thread
  static constexpr int NS = DH <= 80 ? 4 : 3;      // K / V ring depth
  static constexpr int QB = align1k(TQ::BYTES), KB = align1k(TK::BYTES);
  static constexpr int OFF_Q = 0, OFF_K = QB, OFF_V = OFF_K + NS * KB, OFF_BAR = OFF_V + NS * KB;
  static constexpr int SMEM = OFF_BAR + 256 + 1024;  // + alignment slack (dynamic smem base is 16 B aligned)
};

template <int DH>
__global__ void __launch_bounds__(kFThreads, 1)
attn_fwd_kernel(const __grid_constant__ CUtensorMap mq128, const __grid_constant__ CUtensorMap mk128,
                const __grid_constant__ CUtensorMap mv128, const __grid_constant__ CUtensorMap mq32,
                const __grid_constant__ CUtensorMap mk32, const __grid_constant__ CUtensorMap mv32, const FAParams prm) {
  using X = FACfg<DH>;
  using TQ = typename X::TQ;
  using TK = typename X::TK;
  constexpr int BN = kFBN, NS = X::NS;

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint8_t* sQ = smem + X::OFF_Q;
  uint8_t* sK = smem + X::OFF_K;  // NS stages
  uint8_t* sV = smem + X::OFF_V;  // NS stages
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + X::OFF_BAR);
  uint64_t* bar_q = bars;           // Q landed (tx)
  uint64_t* full = bars + 1;        // [NS] K_j, V_j landed (tx)
  uint64_t* empty = bars + 1 + NS;  // [NS] every consumer warp is done with stage j % NS

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int h = blockIdx.y, b = blockIdx.z;
  const int q0 = blockIdx.x * kFM;
  const int T_tiles = (prm.Nk + BN - 1) / BN;

  if (tid == 0) {
    mbar_init(bar_q, 1);
    for (int i = 0; i < NS; ++i) mbar_init(full + i, 1), mbar_init(empty + i, kFWG * 4);
    fence_mbar_init();
  }
  __syncthreads();

  if (warp == kFProducerWarp) {
    if (lane == 0) {
      tma_prefetch_desc(&mq128), tma_prefetch_desc(&mk128), tma_prefetch_desc(&mv128);
      mbar_arrive_expect_tx(bar_q, TQ::BYTES);
      tma_load_tile<DH, kFM>(sQ, &mq128, &mq32, bar_q, q0, h, b);
      for (int j = 0; j < T_tiles; ++j) {
        const int st = j % NS;
        if (j >= NS) mbar_wait(empty + st, ((j / NS) - 1) & 1);
        mbar_arrive_expect_tx(full + st, 2 * TK::BYTES);
        tma_load_tile<DH, BN>(sK + st * X::KB, &mk128, &mk32, full + st, j * BN, h, b);
        tma_load_tile<DH, BN>(sV + st * X::KB, &mv128, &mv32, full + st, j * BN, h, b);
      }
    }
    return;
  }

  // ================= consumers: warpgroup wg owns query rows wg*64 .. wg*64 + 63 =================
  const int wg = warp >> 2, g = lane >> 2, t = lane & 3;
  const int row0 = q0 + wg * 64 + (warp & 3) * 16 + g;  // the thread's rows: row0, row0 + 8
  const float c = prm.scale_log2e;
  float o[X::ACC];
#pragma unroll
  for (int i = 0; i < X::ACC; ++i) o[i] = 0.f;
  float m_[2] = {-INFINITY, -INFINITY}, l_[2] = {0.f, 0.f};  // running max (scaled, log2 units) and sum per row
  mbar_wait(bar_q, 0);
  const uint32_t aQ = smem_u32(sQ);

  for (int j = 0; j < T_tiles; ++j) {
    const int st = j % NS;
    mbar_wait(full + st, (j / NS) & 1);
    float s[BN / 2];
    wg_fence();
    gemm_kk<DH, kFM, BN>(s, aQ, wg * 64, smem_u32(sK + st * X::KB));
    wg_commit();
    wg_wait<0>();

    const int kvalid = prm.Nk - j * BN;  // keys of this tile that exist (>= 1)
    if (kvalid < BN) {
#pragma unroll
      for (int i = 0; i < BN / 2; ++i)
        if ((i >> 2) * 8 + 2 * t + (i & 1) >= kvalid) s[i] = -INFINITY;
    }
    float negm[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      float mx = -INFINITY;
#pragma unroll
      for (int i = 0; i < BN / 8; ++i) mx = fmaxf(mx, fmaxf(s[4 * i + 2 * r], s[4 * i + 2 * r + 1]));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
      const float m_new = fmaxf(m_[r], mx * c);
      const float alpha = ex2_approx(m_[r] - m_new);  // 0 on the first tile
      m_[r] = m_new;
      l_[r] *= alpha;
#pragma unroll
      for (int i = 0; i < X::ACC / 4; ++i) o[4 * i + 2 * r] *= alpha, o[4 * i + 2 * r + 1] *= alpha;
      negm[r] = -m_new;
    }
#pragma unroll
    for (int i = 0; i < BN / 8; ++i) {
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        float p0, p1;
        ex2_pair(i, s[4 * i + 2 * r], s[4 * i + 2 * r + 1], c, negm[r], p0, p1);
        l_[r] += p0 + p1;
        s[4 * i + 2 * r] = p0, s[4 * i + 2 * r + 1] = p1;
      }
    }
    uint32_t pa[BN / 4];
    acc_to_afrag<BN>(s, pa);
    wg_fence();
    gemm_rmn<DH, BN>(o, pa, smem_u32(sV + st * X::KB));
    wg_commit();
    wg_wait<0>();
    __syncwarp();
    if (lane == 0) mbar_arrive(empty + st);
  }

  // ---- epilogue: O / l -> fp16 -> global; log-sum-exp for the backward ----
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    float l = l_[r];
    l += __shfl_xor_sync(0xffffffffu, l, 1);
    l += __shfl_xor_sync(0xffffffffu, l, 2);
    const float inv = 1.f / l;
    const int row = row0 + 8 * r;
    if (row < prm.Nq) {
      __half* orow = prm.o + (int64_t)b * prm.o_sb + (int64_t)row * prm.o_sr + h * DH;
#pragma unroll
      for (int i = 0; i < X::ACC / 4; ++i) {
        const int col = 8 * i + 2 * t;
        if (col < DH) *reinterpret_cast<uint32_t*>(orow + col) = pack_half2(o[4 * i + 2 * r] * inv, o[4 * i + 2 * r + 1] * inv);
      }
      if (prm.lse != nullptr && t == 0) prm.lse[((int64_t)b * prm.H + h) * prm.Nq + row] = (m_[r] + log2f(l)) * 0.6931471805599453f;
    }
  }
}

template <int DH>
static int launch_attn_fwd(const void* q, const void* k, const void* v, const FAParams& prm, int64_t q_sb, int64_t q_sr,
                           int64_t k_sb, int64_t k_sr, int64_t v_sb, int64_t v_sr, cudaStream_t st) {
  using X = FACfg<DH>;
  AttnMaps mq, mk, mv;
  if (make_attn_maps<DH>(mq, q, prm.H, prm.Nq, prm.B, q_sr, q_sb, kFM) ||
      make_attn_maps<DH>(mk, k, prm.H, prm.Nk, prm.B, k_sr, k_sb, kFBN) ||
      make_attn_maps<DH>(mv, v, prm.H, prm.Nk, prm.B, v_sr, v_sb, kFBN)) {
    return MC_E_CUDA;
  }
  const int q_tiles = (prm.Nq + kFM - 1) / kFM;
  auto kern = attn_fwd_kernel<DH>;
  cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, X::SMEM);
  dim3 grid(q_tiles, prm.H, prm.B);
  kern<<<grid, kFThreads, X::SMEM, st>>>(mq.m128, mk.m128, mv.m128, mq.m32, mk.m32, mv.m32, prm);
  count_launch();
  return check_launch("attn_fwd");
}

static int attn_fwd_dispatch(const char* what, int DH, const void* q, const void* k, const void* v, const FAParams& prm,
                             int64_t q_sb, int64_t q_sr, int64_t k_sb, int64_t k_sr, int64_t v_sb, int64_t v_sr,
                             cudaStream_t st) {
#define MC_FA_CASE(D) \
  case D: return launch_attn_fwd<D>(q, k, v, prm, q_sb, q_sr, k_sb, k_sr, v_sb, v_sr, st);
  switch (DH) {
    MC_FA_CASE(8) MC_FA_CASE(16) MC_FA_CASE(32) MC_FA_CASE(40) MC_FA_CASE(64) MC_FA_CASE(80) MC_FA_CASE(160)
    default: break;
  }
#undef MC_FA_CASE
  set_error("%s: unsupported head dim %d (8, 16, 32, 40, 64, 80, 160)", what, DH);
  return MC_E_UNSUPPORTED;
}

}  // namespace mc

extern "C" int mc_spatial_attn_fwd(const void* q, const void* k, const void* v, void* o, float* lse, int B, int N, int H,
                                   int DH, int64_t q_stride_b, int64_t q_stride_row, int64_t k_stride_b,
                                   int64_t k_stride_row, int64_t v_stride_b, int64_t v_stride_row, int64_t o_stride_b,
                                   int64_t o_stride_row, float scale, void* stream) {
  using namespace mc;
  if (!q || !k || !v || !o || B <= 0 || N <= 0 || H <= 0) {
    set_error("spatial_attn_fwd: null pointer or non-positive dims");
    return MC_E_INVALID;
  }
  if (B > 65535 || H > 65535) {
    set_error("spatial_attn_fwd: at most 65535 frames / heads");
    return MC_E_UNSUPPORTED;
  }
  if ((q_stride_b | q_stride_row | k_stride_b | k_stride_row | v_stride_b | v_stride_row | o_stride_b | o_stride_row) % 8 ||
      ((uintptr_t)q | (uintptr_t)k | (uintptr_t)v | (uintptr_t)o) % 16) {
    set_error("spatial_attn_fwd: pointers must be 16-byte aligned and strides multiples of 8 elements");
    return MC_E_INVALID;
  }
  FAParams prm{};
  prm.lse = lse, prm.o = (__half*)o, prm.o_sb = o_stride_b, prm.o_sr = o_stride_row;
  prm.B = B, prm.Nq = N, prm.Nk = N, prm.H = H;
  prm.scale_log2e = scale * 1.44269504088896340736f;
  return attn_fwd_dispatch("spatial_attn_fwd", DH, q, k, v, prm, q_stride_b, q_stride_row, k_stride_b, k_stride_row,
                           v_stride_b, v_stride_row, (cudaStream_t)stream);
}

extern "C" int mc_cross_attn_fwd(const void* q, const void* k, const void* v, void* o, int B, int Nq, int Nk, int H, int DH,
                                 int64_t q_stride_b, int64_t q_stride_row, int64_t kv_stride_b, int64_t kv_stride_row,
                                 int64_t o_stride_b, int64_t o_stride_row, float scale, void* stream) {
  using namespace mc;
  if (!q || !k || !v || !o || B <= 0 || Nq <= 0 || Nk <= 0 || H <= 0) {
    set_error("cross_attn_fwd: null pointer or non-positive dims");
    return MC_E_INVALID;
  }
  if (Nk > kMaxTextKeys) {
    set_error("cross_attn_fwd: at most %d keys (text tokens), got %d", kMaxTextKeys, Nk);
    return MC_E_UNSUPPORTED;
  }
  if (B > 65535 || H > 65535) {
    set_error("cross_attn_fwd: at most 65535 batches / heads");
    return MC_E_UNSUPPORTED;
  }
  if ((q_stride_row | kv_stride_row | o_stride_row | q_stride_b | kv_stride_b | o_stride_b) % 8 ||
      ((uintptr_t)q | (uintptr_t)k | (uintptr_t)v | (uintptr_t)o) % 16) {
    set_error("cross_attn_fwd: pointers must be 16-byte aligned and strides multiples of 8 elements");
    return MC_E_INVALID;
  }
  FAParams prm{};
  prm.lse = nullptr, prm.o = (__half*)o, prm.o_sb = o_stride_b, prm.o_sr = o_stride_row;
  prm.B = B, prm.Nq = Nq, prm.Nk = Nk, prm.H = H;
  prm.scale_log2e = scale * 1.44269504088896340736f;
  return attn_fwd_dispatch("cross_attn_fwd", DH, q, k, v, prm, q_stride_b, q_stride_row, kv_stride_b, kv_stride_row,
                           kv_stride_b, kv_stride_row, (cudaStream_t)stream);
}
