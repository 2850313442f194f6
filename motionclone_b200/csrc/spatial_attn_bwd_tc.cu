// Backward of the attention forward (csrc/spatial_attn_tc.cu) on Hopper tensor cores (wgmma, register accumulators)
// with tensor-map TMA operand loads, sm_90a: the autograd of the xformers seams (reference models/attention.py:535-542)
// that torch.autograd.grad traverses at utils/motionclone_functions.py:236.
//
// With P = softmax(scale S), S = Q K^T, D_r = sum_e dO_re O_re:
//     dV = P^T dO      dP = dO V^T      dS = scale * P o (dP - D)      dQ = dS K      dK = dS^T Q
// Spatial self-attention, three launches; P is recomputed from the forward's log-sum-exp (no N x N tensor is stored):
//   prep       : lse2 = lse * log2(e) and Dsc = scale * D per (frame, head, token), padded to a multiple of 64 tokens
//   dQ kernel  : CTA = 128 queries (2 warpgroups x 64), streams 64-key tiles:  S, dP -> dS (registers) -> dQ += dS K
//   dKV kernel : CTA = 128 keys (64 at DH = 160), streams 64-query tiles (32 at DH = 160):  S^T = K Q^T, dP^T = V dO^T
//                -> P^T, dS^T (registers) -> dV += P^T dO, dK += dS^T Q
// Text cross-attention needs dQ only (the text K / V come from frozen projections of a constant prompt embedding,
// reference t2v_video_sample.py:67-68): the dQ kernel with the whole key axis (77 -> 80 keys) as ONE tile, the softmax
// and D = sum_j P_j dP_j computed in place (exact, no statistics from the forward).
// Every streamed [rows][DH] tile serves two GEMMs through two descriptors - K-major where DH is contracted (S, dP),
// MN-major where the rows are (dS K, P^T dO, dS^T Q) - so nothing is transposed or copied twice; the tiles the threads
// produce (P^T, dS, dS^T) are register A operands of the next wgmma and never touch shared memory. Rows past the end of
// the sequence are zero-filled by the TMA unit. In the dK/dV kernel a padded query row needs no mask: its statistics are
// padded with lse2 = Dsc = 0, so P^T = 1 and dS^T = 0 stay finite, and its zero Q / dO row adds nothing. The dQ kernel
// scores a padded KEY against a real row's statistics, P = exp(-lse), which overflows for very negative lse: it zeroes
// dS of the keys past the end of the last tile, as the forward and the SINGLE path mask them to -inf. The two-kernel split
// recomputes S and dP once more than a fused kernel would but needs no atomics on dQ: results are deterministic.
#include <math.h>

#include "tma_common.cuh"

namespace mc {

constexpr int kBM = 128;  // query rows per dQ CTA (2 warpgroups)
constexpr int kBT = 64;   // key tile of the spatial dQ kernel

struct FABwdParams {
  const float* lse2;   // [B][H][Npad]  lse * log2(e)      (padding: 0)
  const float* dsc;    // [B][H][Npad]  scale * rowsum(dO o O)   (padding: 0)
  __half *dq, *dk, *dv;
  int64_t g_sb, g_sr;  // dq / dk / dv share one stride pattern (column blocks of one fused gradient buffer, or separate)
  int B, Nq, Nk, H, Npad;
  float scale, scale_log2e;
};


// lse2[b][h][r] = lse * log2 e;  dsc[b][h][r] = scale * sum_e dO[b][r][h][e] * O[b][r][h][e];  zeros for N <= r < Npad
template <int DH>
__global__ void __launch_bounds__(256) attn_bwd_prep_kernel(const __half* __restrict__ o, const __half* __restrict__ d_o,
                                                            const float* __restrict__ lse, float* __restrict__ lse2,
                                                            float* __restrict__ dsc, int64_t o_sb, int64_t o_sr,
                                                            int64_t do_sb, int64_t do_sr, int B, int N, int Npad, int H,
                                                            float scale) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;  // ((b * Npad) + r) * H + h
  if (i >= (int64_t)B * Npad * H) return;
  const int h = (int)(i % H);
  const int64_t br = i / H;
  const int r = (int)(br % Npad), b = (int)(br / Npad);
  const int64_t dst = ((int64_t)b * H + h) * Npad + r;
  if (r >= N) {
    lse2[dst] = 0.f, dsc[dst] = 0.f;
    return;
  }
  const uint4* po = reinterpret_cast<const uint4*>(o + b * o_sb + (int64_t)r * o_sr + h * DH);
  const uint4* pd = reinterpret_cast<const uint4*>(d_o + b * do_sb + (int64_t)r * do_sr + h * DH);
  float acc = 0.f;
#pragma unroll
  for (int c = 0; c < DH / 8; ++c) {
    const uint4 a = po[c], g = pd[c];
    const __half2* ah = reinterpret_cast<const __half2*>(&a);
    const __half2* gh = reinterpret_cast<const __half2*>(&g);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 x = __half22float2(ah[j]), y = __half22float2(gh[j]);
      acc = fmaf(x.x, y.x, acc);
      acc = fmaf(x.y, y.y, acc);
    }
  }
  lse2[dst] = lse[((int64_t)b * H + h) * N + r] * 1.44269504088896340736f;
  dsc[dst] = acc * scale;
}


// rows row0 and row0 + 8 of the calling thread in a warpgroup accumulator (columns < DH) -> fp16 -> global
template <int DH>
__device__ __forceinline__ void store_acc_rows(const float* acc, __half* base, int64_t sr, int row0, int nrows, int t) {
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int row = row0 + 8 * r;
    if (row >= nrows) continue;
    __half* p = base + (int64_t)row * sr;
#pragma unroll
    for (int i = 0; i < AccW<DH>::REGS / 4; ++i) {
      const int col = 8 * i + 2 * t;
      if (col < DH) *reinterpret_cast<uint32_t*>(p + col) = pack_half2(acc[4 * i + 2 * r], acc[4 * i + 2 * r + 1]);
    }
  }
}

template <int DH, bool SINGLE>
struct DQCfg {
  static constexpr int BN = SINGLE ? kMaxTextKeys : kBT;  // keys per tile
  using TQ = TileParts<DH, kBM>;
  using TK = TileParts<DH, BN>;
  static constexpr int ACC = AccW<DH>::REGS;
  static constexpr int NS = SINGLE ? 1 : 2;  // K / V ring depth
  static constexpr int THREADS = 2 * 128 + 32;
  static constexpr int QB = align1k(TQ::BYTES), KB = align1k(TK::BYTES);
  static constexpr int OFF_Q = 0, OFF_DO = QB, OFF_K = 2 * QB, OFF_V = OFF_K + NS * KB, OFF_BAR = OFF_V + NS * KB;
  static constexpr int SMEM = OFF_BAR + 256 + 1024;
};

// dQ for 128 queries: warpgroups 0, 1 own 64 rows each; warp 8 lane 0 issues the TMA loads (Q and dO resident, K and V
// streamed). SINGLE: the whole key axis (<= kMaxTextKeys) is one tile and the softmax statistics are computed here.
// RAGGED (spatial only, launched when Nk % 64 != 0): dS of the keys past the end of the last tile is zeroed; a separate
// instantiation so that the 64-aligned token counts run the unmasked code unchanged.
template <int DH, bool SINGLE, bool RAGGED>
__global__ void __launch_bounds__(DQCfg<DH, SINGLE>::THREADS, 1)
attn_bwd_dq_kernel(const __grid_constant__ CUtensorMap mq128, const __grid_constant__ CUtensorMap mq32,
                   const __grid_constant__ CUtensorMap mdo128, const __grid_constant__ CUtensorMap mdo32,
                   const __grid_constant__ CUtensorMap mk128, const __grid_constant__ CUtensorMap mk32,
                   const __grid_constant__ CUtensorMap mv128, const __grid_constant__ CUtensorMap mv32,
                   const FABwdParams prm) {
  using X = DQCfg<DH, SINGLE>;
  using TQ = typename X::TQ;
  using TK = typename X::TK;
  constexpr int BN = X::BN, NS = X::NS;

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint8_t* sQ = smem + X::OFF_Q;
  uint8_t* sDO = smem + X::OFF_DO;
  uint8_t* sK = smem + X::OFF_K;  // NS stages
  uint8_t* sV = smem + X::OFF_V;  // NS stages
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + X::OFF_BAR);
  uint64_t* bar_q = bars;           // Q and dO landed (tx)
  uint64_t* full = bars + 1;        // [NS] K_j, V_j landed (tx)
  uint64_t* empty = bars + 1 + NS;  // [NS] every consumer warp is done with stage j % NS

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int h = blockIdx.y, b = blockIdx.z;
  const int q0 = blockIdx.x * kBM;
  const int T_tiles = (prm.Nk + BN - 1) / BN;

  if (tid == 0) {
    mbar_init(bar_q, 1);
    for (int i = 0; i < NS; ++i) mbar_init(full + i, 1), mbar_init(empty + i, 8);
    fence_mbar_init();
  }
  __syncthreads();

  if (warp == 8) {
    if (lane == 0) {
      mbar_arrive_expect_tx(bar_q, 2 * TQ::BYTES);
      tma_load_tile<DH, kBM>(sQ, &mq128, &mq32, bar_q, q0, h, b);
      tma_load_tile<DH, kBM>(sDO, &mdo128, &mdo32, bar_q, q0, h, b);
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

  const int wg = warp >> 2, g = lane >> 2, t = lane & 3;
  const int row0 = q0 + wg * 64 + (warp & 3) * 16 + g;  // the thread's rows: row0, row0 + 8
  const float c = prm.scale_log2e, scale = prm.scale;
  float neg_lse2[2] = {0.f, 0.f}, dscr[2] = {0.f, 0.f};
  if constexpr (!SINGLE) {
    const int64_t base = ((int64_t)b * prm.H + h) * prm.Npad;
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const int row = row0 + 8 * r;
      if (row < prm.Npad) neg_lse2[r] = -prm.lse2[base + row], dscr[r] = prm.dsc[base + row];
    }
  }
  float dq[X::ACC];
#pragma unroll
  for (int i = 0; i < X::ACC; ++i) dq[i] = 0.f;
  mbar_wait(bar_q, 0);

  for (int j = 0; j < T_tiles; ++j) {
    const int st = j % NS;
    mbar_wait(full + st, (j / NS) & 1);
    float s[BN / 2], dp[BN / 2];
    wg_fence();
    gemm_kk<DH, kBM, BN>(s, smem_u32(sQ), wg * 64, smem_u32(sK + st * X::KB));
    gemm_kk<DH, kBM, BN>(dp, smem_u32(sDO), wg * 64, smem_u32(sV + st * X::KB));
    wg_commit();
    wg_wait<0>();

    if constexpr (SINGLE) {
#pragma unroll
      for (int i = 0; i < BN / 2; ++i)
        if ((i >> 2) * 8 + 2 * t + (i & 1) >= prm.Nk) s[i] = -INFINITY;  // keys past the end
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        float mx = -INFINITY;
#pragma unroll
        for (int i = 0; i < BN / 8; ++i) mx = fmaxf(mx, fmaxf(s[4 * i + 2 * r], s[4 * i + 2 * r + 1]));
        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
        const float negm = -mx * c;
        float sum = 0.f;
#pragma unroll
        for (int i = 0; i < BN / 8; ++i)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int k = 4 * i + 2 * r + e;
            s[k] = ex2_approx(fmaf(s[k], c, negm));
            sum += s[k];
          }
        sum += __shfl_xor_sync(0xffffffffu, sum, 1);
        sum += __shfl_xor_sync(0xffffffffu, sum, 2);
        const float inv = 1.f / sum;
        float d = 0.f;  // D = sum_j P_j dP_j
#pragma unroll
        for (int i = 0; i < BN / 8; ++i)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int k = 4 * i + 2 * r + e;
            s[k] *= inv;
            d = fmaf(s[k], dp[k], d);
          }
        d += __shfl_xor_sync(0xffffffffu, d, 1);
        d += __shfl_xor_sync(0xffffffffu, d, 2);
#pragma unroll
        for (int i = 0; i < BN / 8; ++i)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int k = 4 * i + 2 * r + e;
            dp[k] = scale * s[k] * (dp[k] - d);
          }
      }
    } else {
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) {
        const int r = (i >> 1) & 1;
        const float p = ex2_approx(fmaf(s[i], c, neg_lse2[r]));
        dp[i] = p * fmaf(dp[i], scale, -dscr[r]);
      }
      if constexpr (RAGGED) {
        // Keys past the end of the sequence: the zero-filled K row scores s = 0 against this row's statistics, so
        // p = exp(-lse) overflows fp16 (or fp32) when lse is very negative, and inf x 0 in dS K would be NaN.
        const int kvalid = prm.Nk - j * BN;
        if (kvalid < BN) {
#pragma unroll
          for (int i = 0; i < BN / 2; ++i)
            if ((i >> 2) * 8 + 2 * t + (i & 1) >= kvalid) dp[i] = 0.f;
        }
      }
    }
    uint32_t da[BN / 4];
    acc_to_afrag<BN>(dp, da);
    wg_fence();
    gemm_rmn<DH, BN>(dq, da, smem_u32(sK + st * X::KB));
    wg_commit();
    wg_wait<0>();
    __syncwarp();
    if (lane == 0) mbar_arrive(empty + st);
  }
  store_acc_rows<DH>(dq, prm.dq + (int64_t)b * prm.g_sb + h * DH, prm.g_sr, row0, prm.Nq, t);
}

template <int DH>
struct KVCfg {
  static constexpr int WG = DH > 96 ? 1 : 2;   // consumer warpgroups (one at DH = 160: dK + dV take 160 registers)
  static constexpr int KM = WG * 64;           // keys per CTA
  static constexpr int BT = DH > 96 ? 32 : 64; // streamed query tile
  using TK = TileParts<DH, KM>;
  using TQ = TileParts<DH, BT>;
  static constexpr int ACC = AccW<DH>::REGS;
  static constexpr int NS = 2;
  static constexpr int THREADS = WG * 128 + 32;
  static constexpr int KB = align1k(TK::BYTES), QB = align1k(TQ::BYTES);
  static constexpr int OFF_K = 0, OFF_V = KB, OFF_Q = 2 * KB, OFF_DO = OFF_Q + NS * QB, OFF_BAR = OFF_DO + NS * QB;
  static constexpr int SMEM = OFF_BAR + 256 + 1024;
};

template <int DH>
__global__ void __launch_bounds__(KVCfg<DH>::THREADS, 1)
attn_bwd_dkv_kernel(const __grid_constant__ CUtensorMap mk128, const __grid_constant__ CUtensorMap mk32,
                    const __grid_constant__ CUtensorMap mv128, const __grid_constant__ CUtensorMap mv32,
                    const __grid_constant__ CUtensorMap mq128, const __grid_constant__ CUtensorMap mq32,
                    const __grid_constant__ CUtensorMap mdo128, const __grid_constant__ CUtensorMap mdo32,
                    const FABwdParams prm) {
  using X = KVCfg<DH>;
  using TK = typename X::TK;
  using TQ = typename X::TQ;
  constexpr int KM = X::KM, BT = X::BT, NS = X::NS;

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint8_t* sK = smem + X::OFF_K;
  uint8_t* sV = smem + X::OFF_V;
  uint8_t* sQ = smem + X::OFF_Q;    // NS stages
  uint8_t* sDO = smem + X::OFF_DO;  // NS stages
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + X::OFF_BAR);
  uint64_t* bar_kv = bars;          // K and V landed (tx)
  uint64_t* full = bars + 1;        // [NS] Q_j, dO_j landed (tx)
  uint64_t* empty = bars + 1 + NS;  // [NS] every consumer warp is done with stage j % NS

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int h = blockIdx.y, b = blockIdx.z;
  const int k0 = blockIdx.x * KM;
  const int T_tiles = (prm.Nq + BT - 1) / BT;

  if (tid == 0) {
    mbar_init(bar_kv, 1);
    for (int i = 0; i < NS; ++i) mbar_init(full + i, 1), mbar_init(empty + i, X::WG * 4);
    fence_mbar_init();
  }
  __syncthreads();

  if (warp == X::WG * 4) {
    if (lane == 0) {
      mbar_arrive_expect_tx(bar_kv, 2 * TK::BYTES);
      tma_load_tile<DH, KM>(sK, &mk128, &mk32, bar_kv, k0, h, b);
      tma_load_tile<DH, KM>(sV, &mv128, &mv32, bar_kv, k0, h, b);
      for (int j = 0; j < T_tiles; ++j) {
        const int st = j % NS;
        if (j >= NS) mbar_wait(empty + st, ((j / NS) - 1) & 1);
        mbar_arrive_expect_tx(full + st, 2 * TQ::BYTES);
        tma_load_tile<DH, BT>(sQ + st * X::QB, &mq128, &mq32, full + st, j * BT, h, b);
        tma_load_tile<DH, BT>(sDO + st * X::QB, &mdo128, &mdo32, full + st, j * BT, h, b);
      }
    }
    return;
  }

  const int wg = warp >> 2, g = lane >> 2, t = lane & 3;
  const int krow0 = k0 + wg * 64 + (warp & 3) * 16 + g;  // the thread's key rows: krow0, krow0 + 8
  const float c = prm.scale_log2e, scale = prm.scale;
  const float* lse2 = prm.lse2 + ((int64_t)b * prm.H + h) * prm.Npad;
  const float* dsc = prm.dsc + ((int64_t)b * prm.H + h) * prm.Npad;
  float dk[X::ACC], dv[X::ACC];
#pragma unroll
  for (int i = 0; i < X::ACC; ++i) dk[i] = 0.f, dv[i] = 0.f;
  mbar_wait(bar_kv, 0);

  for (int j = 0; j < T_tiles; ++j) {
    const int st = j % NS;
    mbar_wait(full + st, (j / NS) & 1);
    const uint32_t aQ = smem_u32(sQ + st * X::QB), aDO = smem_u32(sDO + st * X::QB);
    float s[BT / 2], dp[BT / 2];
    wg_fence();
    gemm_kk<DH, KM, BT>(s, smem_u32(sK), wg * 64, aQ);    // S^T = K Q^T
    gemm_kk<DH, KM, BT>(dp, smem_u32(sV), wg * 64, aDO);  // dP^T = V dO^T
    wg_commit();
    wg_wait<0>();
#pragma unroll
    for (int i = 0; i < BT / 8; ++i)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int qc = j * BT + 8 * i + 2 * t + e;  // query column (< Npad: BT divides 64)
        const float nl = -lse2[qc], d = dsc[qc];
#pragma unroll
        for (int r = 0; r < 2; ++r) {
          const int k = 4 * i + 2 * r + e;
          s[k] = ex2_approx(fmaf(s[k], c, nl));     // P^T
          dp[k] = s[k] * fmaf(dp[k], scale, -d);    // dS^T
        }
      }
    uint32_t pa[BT / 4], da[BT / 4];
    acc_to_afrag<BT>(s, pa);
    acc_to_afrag<BT>(dp, da);
    wg_fence();
    gemm_rmn<DH, BT>(dv, pa, aDO);  // dV += P^T dO
    gemm_rmn<DH, BT>(dk, da, aQ);   // dK += dS^T Q
    wg_commit();
    wg_wait<0>();
    __syncwarp();
    if (lane == 0) mbar_arrive(empty + st);
  }
  store_acc_rows<DH>(dk, prm.dk + (int64_t)b * prm.g_sb + h * DH, prm.g_sr, krow0, prm.Nk, t);
  store_acc_rows<DH>(dv, prm.dv + (int64_t)b * prm.g_sb + h * DH, prm.g_sr, krow0, prm.Nk, t);
}

template <int DH, bool SINGLE>
static int launch_dq(const AttnMaps& q, const AttnMaps& d_o, const AttnMaps& k, const AttnMaps& v, const FABwdParams& prm,
                     cudaStream_t st) {
  using X = DQCfg<DH, SINGLE>;
  auto kern = attn_bwd_dq_kernel<DH, SINGLE, false>;
  if constexpr (!SINGLE) {
    if (prm.Nk % kBT) kern = attn_bwd_dq_kernel<DH, false, true>;
  }
  cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, X::SMEM);
  dim3 grid((prm.Nq + kBM - 1) / kBM, prm.H, prm.B);
  kern<<<grid, X::THREADS, X::SMEM, st>>>(q.m128, q.m32, d_o.m128, d_o.m32, k.m128, k.m32, v.m128, v.m32, prm);
  count_launch();
  return check_launch(SINGLE ? "cross_attn_bwd_dq" : "spatial_attn_bwd_dq");
}

template <int DH>
static int launch_spatial_bwd(const void* q, const void* k, const void* v, const void* o, const void* d_o, const float* lse,
                              float* workspace, FABwdParams prm, int64_t q_sb, int64_t q_sr, int64_t k_sb, int64_t k_sr,
                              int64_t v_sb, int64_t v_sr, int64_t o_sb, int64_t o_sr, int64_t do_sb, int64_t do_sr,
                              cudaStream_t st) {
  using KV = KVCfg<DH>;
  const int B = prm.B, N = prm.Nq, H = prm.H, Npad = prm.Npad;
  AttnMaps q128, do128, k64, v64, kres, vres, qs, dos;
  int rc = make_attn_maps<DH>(q128, q, H, N, B, q_sr, q_sb, kBM) | make_attn_maps<DH>(do128, d_o, H, N, B, do_sr, do_sb, kBM) |
           make_attn_maps<DH>(k64, k, H, N, B, k_sr, k_sb, kBT) | make_attn_maps<DH>(v64, v, H, N, B, v_sr, v_sb, kBT) |
           make_attn_maps<DH>(kres, k, H, N, B, k_sr, k_sb, KV::KM) | make_attn_maps<DH>(vres, v, H, N, B, v_sr, v_sb, KV::KM) |
           make_attn_maps<DH>(qs, q, H, N, B, q_sr, q_sb, KV::BT) | make_attn_maps<DH>(dos, d_o, H, N, B, do_sr, do_sb, KV::BT);
  if (rc) return MC_E_CUDA;
  float* lse2 = workspace;
  float* dsc = workspace + (int64_t)B * H * Npad;
  prm.lse2 = lse2, prm.dsc = dsc;
  {
    const int64_t total = (int64_t)B * Npad * H;
    attn_bwd_prep_kernel<DH><<<(unsigned)((total + 255) / 256), 256, 0, st>>>((const __half*)o, (const __half*)d_o, lse, lse2,
                                                                            dsc, o_sb, o_sr, do_sb, do_sr, B, N, Npad, H,
                                                                            prm.scale);
    count_launch();
    if (int e = check_launch("attn_bwd_prep")) return e;
  }
  if (int e = launch_dq<DH, false>(q128, do128, k64, v64, prm, st)) return e;
  {
    auto kern = attn_bwd_dkv_kernel<DH>;
    cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, KV::SMEM);
    dim3 grid((N + KV::KM - 1) / KV::KM, H, B);
    kern<<<grid, KV::THREADS, KV::SMEM, st>>>(kres.m128, kres.m32, vres.m128, vres.m32, qs.m128, qs.m32, dos.m128, dos.m32, prm);
    count_launch();
    if (int e = check_launch("spatial_attn_bwd_dkv")) return e;
  }
  return MC_OK;
}

template <int DH>
static int launch_cross_bwd(const void* q, const void* k, const void* v, const void* d_o, const FABwdParams& prm,
                            int64_t q_sb, int64_t q_sr, int64_t kv_sb, int64_t kv_sr, int64_t do_sb, int64_t do_sr,
                            cudaStream_t st) {
  AttnMaps mq, mdo, mk, mv;
  if (make_attn_maps<DH>(mq, q, prm.H, prm.Nq, prm.B, q_sr, q_sb, kBM) ||
      make_attn_maps<DH>(mdo, d_o, prm.H, prm.Nq, prm.B, do_sr, do_sb, kBM) ||
      make_attn_maps<DH>(mk, k, prm.H, prm.Nk, prm.B, kv_sr, kv_sb, kMaxTextKeys) ||
      make_attn_maps<DH>(mv, v, prm.H, prm.Nk, prm.B, kv_sr, kv_sb, kMaxTextKeys))
    return MC_E_CUDA;
  return launch_dq<DH, true>(mq, mdo, mk, mv, prm, st);
}

static inline int npad64(int N) { return (N + 63) / 64 * 64; }

}  // namespace mc

extern "C" int64_t mc_spatial_attn_bwd_workspace_bytes(int B, int N, int H) {
  return (int64_t)2 * B * H * mc::npad64(N) * 4;
}

extern "C" int mc_spatial_attn_bwd(const void* q, const void* k, const void* v, const void* o, const void* d_o,
                                   const float* lse, void* dq, void* dk, void* dv, void* workspace, int B, int N, int H,
                                   int DH, int64_t q_stride_b, int64_t q_stride_row, int64_t k_stride_b,
                                   int64_t k_stride_row, int64_t v_stride_b, int64_t v_stride_row, int64_t o_stride_b,
                                   int64_t o_stride_row, int64_t do_stride_b, int64_t do_stride_row, int64_t g_stride_b,
                                   int64_t g_stride_row, float scale, void* stream) {
  using namespace mc;
  if (!q || !k || !v || !o || !d_o || !lse || !dq || !dk || !dv || !workspace || B <= 0 || N <= 0 || H <= 0) {
    set_error("spatial_attn_bwd: null pointer or non-positive dims");
    return MC_E_INVALID;
  }
  if (B > 65535 || H > 65535) {
    set_error("spatial_attn_bwd: at most 65535 frames / heads");
    return MC_E_UNSUPPORTED;
  }
  if ((q_stride_b | q_stride_row | k_stride_b | k_stride_row | v_stride_b | v_stride_row | o_stride_b | o_stride_row |
       do_stride_b | do_stride_row | g_stride_b | g_stride_row) % 8 ||
      ((uintptr_t)q | (uintptr_t)k | (uintptr_t)v | (uintptr_t)o | (uintptr_t)d_o | (uintptr_t)dq | (uintptr_t)dk |
       (uintptr_t)dv | (uintptr_t)workspace) % 16) {
    set_error("spatial_attn_bwd: pointers must be 16-byte aligned and strides multiples of 8 elements");
    return MC_E_INVALID;
  }
  FABwdParams prm{};
  prm.dq = (__half*)dq, prm.dk = (__half*)dk, prm.dv = (__half*)dv, prm.g_sb = g_stride_b, prm.g_sr = g_stride_row;
  prm.B = B, prm.Nq = N, prm.Nk = N, prm.H = H, prm.Npad = npad64(N), prm.scale = scale, prm.scale_log2e = scale * 1.44269504088896340736f;
  cudaStream_t st = (cudaStream_t)stream;
#define MC_SB_CASE(D)                                                                                                      \
  case D:                                                                                                                  \
    return launch_spatial_bwd<D>(q, k, v, o, d_o, lse, (float*)workspace, prm, q_stride_b, q_stride_row, k_stride_b,       \
                                 k_stride_row, v_stride_b, v_stride_row, o_stride_b, o_stride_row, do_stride_b, do_stride_row, st);
  switch (DH) {
    MC_SB_CASE(8) MC_SB_CASE(16) MC_SB_CASE(32) MC_SB_CASE(40) MC_SB_CASE(64) MC_SB_CASE(80) MC_SB_CASE(160)
    default: break;
  }
#undef MC_SB_CASE
  set_error("spatial_attn_bwd: unsupported head dim %d (8, 16, 32, 40, 64, 80, 160)", DH);
  return MC_E_UNSUPPORTED;
}

extern "C" int mc_cross_attn_bwd_dq(const void* q, const void* k, const void* v, const void* d_o, void* dq, int B, int Nq,
                                    int Nk, int H, int DH, int64_t q_stride_b, int64_t q_stride_row, int64_t kv_stride_b,
                                    int64_t kv_stride_row, int64_t do_stride_b, int64_t do_stride_row,
                                    int64_t dq_stride_b, int64_t dq_stride_row, float scale, void* stream) {
  using namespace mc;
  if (!q || !k || !v || !d_o || !dq || B <= 0 || Nq <= 0 || Nk <= 0 || H <= 0) {
    set_error("cross_attn_bwd_dq: null pointer or non-positive dims");
    return MC_E_INVALID;
  }
  if (Nk > kMaxTextKeys) {
    set_error("cross_attn_bwd_dq: at most %d keys (text tokens) per tile, got %d", kMaxTextKeys, Nk);
    return MC_E_UNSUPPORTED;
  }
  if (B > 65535 || H > 65535) {
    set_error("cross_attn_bwd_dq: at most 65535 batches / heads");
    return MC_E_UNSUPPORTED;
  }
  if ((q_stride_row | kv_stride_row | dq_stride_row | q_stride_b | kv_stride_b | dq_stride_b | do_stride_b | do_stride_row) % 8 ||
      ((uintptr_t)q | (uintptr_t)k | (uintptr_t)v | (uintptr_t)d_o | (uintptr_t)dq) % 16) {
    set_error("cross_attn_bwd_dq: pointers must be 16-byte aligned and strides multiples of 8 elements");
    return MC_E_INVALID;
  }
  FABwdParams prm{};
  prm.dq = (__half*)dq, prm.g_sb = dq_stride_b, prm.g_sr = dq_stride_row;
  prm.B = B, prm.Nq = Nq, prm.Nk = Nk, prm.H = H;
  prm.scale = scale, prm.scale_log2e = scale * 1.44269504088896340736f;
  cudaStream_t st = (cudaStream_t)stream;
#define MC_XB_CASE(D)                                                                                                    \
  case D:                                                                                                                \
    return launch_cross_bwd<D>(q, k, v, d_o, prm, q_stride_b, q_stride_row, kv_stride_b, kv_stride_row, do_stride_b,    \
                               do_stride_row, st);
  switch (DH) {
    MC_XB_CASE(8) MC_XB_CASE(16) MC_XB_CASE(32) MC_XB_CASE(40) MC_XB_CASE(64) MC_XB_CASE(80) MC_XB_CASE(160)
    default: break;
  }
#undef MC_XB_CASE
  set_error("cross_attn_bwd_dq: unsupported head dim %d (8, 16, 32, 40, 64, 80, 160)", DH);
  return MC_E_UNSUPPORTED;
}
