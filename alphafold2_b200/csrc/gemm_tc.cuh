// Generic batched bf16 GEMM on sm_90a warpgroup tensor cores (wgmma) with TMA-staged operands and a programmable
// epilogue applied to the register accumulators.
// One kernel serves every dense contraction of the Evoformer block:
//
//   K-major mode  : C[b][m][n] = sum_k A[b][m][k] * B[b][n][k]      (Linear layers: B = weight [out,in];
//                                                                    triangle "outgoing" per channel)
//   MN-major mode : C[b][m][n] = sum_k A[b][k][m] * B[b][k][n]      (triangle "ingoing", outer-mean:
//                                                                    channel-major operands, k = row axis)
//
// Tiling: BM = 128 rows, BN in {64,128,256} accumulator columns, BK = 64.
// Warp roles (384 threads, three warpgroups):
//   warpgroup 0     TMA producer of the A/B stages (one thread issues; the warpgroup hands its registers to the others)
//   warpgroups 1, 2 MMA + epilogue, rows 0..63 / 64..127 of the tile: wgmma m64nBNk16 into registers, then
//                   (bias, activation, gate, row scale, residual) -> global stores straight from the accumulator fragment
// Persistent over tiles; the producer runs ahead across tiles, so the loads of tile i+1 overlap the epilogue of tile i.
#pragma once
#include "common.cuh"

namespace af2 {

constexpr int GEMM_BM = 128;
constexpr int GEMM_BK = 64;

enum EpiMode : int { EPI_STORE_BF16 = 0, EPI_GATED_BF16 = 1, EPI_RESID_F32 = 2, EPI_STORE_F32 = 3 };
enum EpiAct : int { ACT_NONE = 0, ACT_SIGMOID = 1, ACT_GELU = 2 };
enum EpiLayout : int { LAYOUT_TOKEN = 0, LAYOUT_CHANNEL = 1 };

// Epilogue program (identical for every column tile).
struct NTile {
  int mode;        // EpiMode
  int act;         // EpiAct (applied to the value for STORE, to the gate half for GATED)
  int layout;      // EpiLayout
  int use_rowscale;
  void* out;
  const float* bias;   // [N] accumulator-column bias, or nullptr
  long long ld;        // token-major: row stride (elements); channel-major: channel stride (elements)
};

// Tile nt produces output columns [nt*W, nt*W + W) with W = BN (BN/2 for EPI_GATED, whose weight rows are
// packed per tile as [value rows of the tile | gate rows of the tile]), clipped to out_cols.
struct GemmParams {
  int M, N, K, batch;          // N = accumulator columns = rows of the B operand
  int num_ntiles;
  int out_cols;                // valid output columns (N, or N/2 for EPI_GATED)
  int direct;                  // unused: the epilogue always stores from registers
  const float* rowscale;       // [batch*M] multiplier per row (mask), or nullptr
  const float* resid;          // EPI_RESID_F32: fp32 [M, ld_resid]
  long long ld_resid;
  long long out_batch_stride;  // elements
  int cm_inner, cm_pitch;      // channel-major: row r -> (r / cm_inner) * cm_pitch + r % cm_inner
  // Split-bf16 (strict precision) operands: every fp32 operand value v is stored as bf16 planes p0 = bf16(v),
  // p1 = bf16(v - p0) [, p2 = bf16(v - p0 - p1)] (tensor maps of rank 4: k, row, plane, batch) and the k loop makes nseg passes
  // over K, one per plane pair (A plane, B plane), smallest products first, all into the same fp32 accumulator:
  //   nseg = 3 (two planes,   ~16 mantissa bits): (0,1) (1,0) (0,0)
  //   nseg = 6 (three planes,  24 mantissa bits): (0,2) (2,0) (1,1) (0,1) (1,0) (0,0)      <- strict mode
  // nseg = 1: plain bf16 operands, rank-3 maps.
  int nseg;
  // Operands gathered from several ranks ("pieces", alphafold2_b200/parallel.py): an all-gather concatenates the per-rank
  // shards [c][rows_p][k] along the outermost axis, so rows r = p * pr + rr of one channel are pr-row pieces piece_stride
  // apart.  Rank-4 maps (k | mn, row | k, piece, batch) address them in place -- one launch instead of one per piece.
  //   a_pr / b_pr: rows (K-major) or columns (MN-major) per piece of A / B; 0 = plain rank-3 map.
  int a_pr, b_pr;
  int x_evict_last;            // 1: residual loads / output stores of the fp32 stream carry an L2 evict_last hint
  NTile tile;
};

template <int BN, int STAGES>
struct GemmSmem {
  static constexpr int A_BYTES = GEMM_BM * GEMM_BK * 2;   // 16 KB
  static constexpr int B_BYTES = BN * GEMM_BK * 2;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr int BAR_OFF = STAGES * STAGE_BYTES;
  static constexpr int TOTAL = BAR_OFF + 256;
  static_assert(TOTAL <= 232448, "exceeds the 227 KB of shared memory a CTA can use");
};

__device__ __forceinline__ float apply_act(float x, int act) {
  if (act == ACT_SIGMOID) return sigmoidf_fast(x);
  if (act == ACT_GELU) return gelu_erf(x);
  return x;
}

// Compile-time epilogue specialisations (EK_GENERIC reads mode / act / layout from the params at run time; it is
// used for the small-tile instantiations where speed does not matter).
enum EpiKind : int {
  EK_GENERIC = 0,
  EK_STORE_TOK = 1,       // bf16 token-major, optional bias                       (q|k|v projection)
  EK_STORE_TOK_SIG = 2,   // bf16 token-major, sigmoid(acc + bias)                  (attention gate, out_gate)
  EK_STORE_CH = 3,        // bf16 channel-major, (acc + bias) * rowscale            (outer-mean left|right)
  EK_GATED_TOK_GELU = 4,  // bf16 token-major, (u + b) * gelu(g + b)                (FeedForward first Linear)
  EK_GATED_CH_SIG = 5,    // bf16 channel-major, (u + b) * sigmoid(g + b) * rowscale (triangle left / right)
  EK_RESID_F32 = 6,       // fp32 token-major, acc + bias + residual                (every output projection)
  EK_STORE_F32 = 7,       // fp32 token-major                                       (per-channel contractions)
  EK_STORE_CH_SIG = 8,    // bf16 channel-major, sigmoid(acc + bias)                (triangle out_gate for the fused tail)
  EK_RESID_F32_W = 9      // EK_RESID_F32 for a single full 256-column tile (same epilogue)
};
template <int EK> struct EpiTraits { static constexpr int mode = -1, act = -1, layout = -1; static constexpr bool rowscale = true; };
template <> struct EpiTraits<EK_STORE_TOK> { static constexpr int mode = EPI_STORE_BF16, act = ACT_NONE, layout = LAYOUT_TOKEN; static constexpr bool rowscale = false; };
template <> struct EpiTraits<EK_STORE_TOK_SIG> { static constexpr int mode = EPI_STORE_BF16, act = ACT_SIGMOID, layout = LAYOUT_TOKEN; static constexpr bool rowscale = false; };
template <> struct EpiTraits<EK_STORE_CH> { static constexpr int mode = EPI_STORE_BF16, act = ACT_NONE, layout = LAYOUT_CHANNEL; static constexpr bool rowscale = true; };
template <> struct EpiTraits<EK_GATED_TOK_GELU> { static constexpr int mode = EPI_GATED_BF16, act = ACT_GELU, layout = LAYOUT_TOKEN; static constexpr bool rowscale = false; };
template <> struct EpiTraits<EK_GATED_CH_SIG> { static constexpr int mode = EPI_GATED_BF16, act = ACT_SIGMOID, layout = LAYOUT_CHANNEL; static constexpr bool rowscale = true; };
template <> struct EpiTraits<EK_RESID_F32> { static constexpr int mode = EPI_RESID_F32, act = ACT_NONE, layout = LAYOUT_TOKEN; static constexpr bool rowscale = false; };
template <> struct EpiTraits<EK_RESID_F32_W> { static constexpr int mode = EPI_RESID_F32, act = ACT_NONE, layout = LAYOUT_TOKEN; static constexpr bool rowscale = false; };
template <> struct EpiTraits<EK_STORE_CH_SIG> { static constexpr int mode = EPI_STORE_BF16, act = ACT_SIGMOID, layout = LAYOUT_CHANNEL; static constexpr bool rowscale = false; };
template <> struct EpiTraits<EK_STORE_F32> { static constexpr int mode = EPI_STORE_F32, act = ACT_NONE, layout = LAYOUT_TOKEN; static constexpr bool rowscale = false; };

constexpr int GEMM_THREADS = 384;   // producer warpgroup + two MMA warpgroups

// stores the two values (col, col + 1) of one accumulator row, clipped to the valid columns
template <bool F32>
__device__ __forceinline__ void store_pair(void* base, long long off, float v0, float v1, bool two, bool vec) {
  if constexpr (F32) {
    float* o = reinterpret_cast<float*>(base) + off;
    if (two && vec) *reinterpret_cast<float2*>(o) = make_float2(v0, v1);
    else { o[0] = v0; if (two) o[1] = v1; }
  } else {
    __nv_bfloat16* o = reinterpret_cast<__nv_bfloat16*>(base) + off;
    if (two && vec) *reinterpret_cast<uint32_t*>(o) = pack_bf16x2(v0, v1);
    else { o[0] = __float2bfloat16(v0); if (two) o[1] = __float2bfloat16(v1); }
  }
}

template <int BN, int STAGES, bool MN_MAJOR, int EK>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_tc_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
               const __grid_constant__ CUtensorMap tmC, const __grid_constant__ CUtensorMap tmR,
               const __grid_constant__ GemmParams p) {
  using L = GemmSmem<BN, STAGES>;
  // 1024-byte aligned by declaration (128B-swizzle atoms); keeping the array symbol (no integer round-up of the pointer)
  // lets the compiler prove the shared address space and emit LDS/STS instead of generic LD/ST
  extern __shared__ __align__(1024) uint8_t smem[];
  if ((smem_u32(smem) & 1023u) != 0) __trap();
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + L::BAR_OFF);
  uint64_t* empty_bar = full_bar + STAGES;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int wg = warp >> 2;

  if (threadIdx.x == 0) {
    prefetch_tmap(&tmA);
    prefetch_tmap(&tmB);
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 2);     // one arrive per MMA warpgroup
    }
    fence_barrier_init();
  }
  __syncthreads();
  pdl_launch_dependents();
  pdl_wait();

  const int m_tiles = (p.M + GEMM_BM - 1) / GEMM_BM;
  const int n_tiles = p.num_ntiles;
  const int total_tiles = p.batch * m_tiles * n_tiles;
  const int num_kb = (p.K + GEMM_BK - 1) / GEMM_BK;
  const int nseg = p.nseg > 1 ? p.nseg : 1;
  const int num_kk = num_kb * nseg;                 // k-blocks consumed per tile

  if (wg == 0) {
    // ================================ TMA producer ================================
    regs_dealloc<40>();
    if (threadIdx.x == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
        const int nt = tile % n_tiles;
        const int mt = (tile / n_tiles) % m_tiles;
        const int b = tile / (n_tiles * m_tiles);
        for (int kk = 0; kk < num_kk; ++kk) {
          const int seg = kk / num_kb, kb = kk - seg * num_kb;
          mbar_wait(&empty_bar[stage], phase ^ 1);
          uint8_t* sa = smem + stage * L::STAGE_BYTES;
          uint8_t* sb = sa + L::A_BYTES;
          mbar_arrive_expect_tx(&full_bar[stage], L::STAGE_BYTES);
          if (nseg > 1) {
            // split operands (rank-4 maps): plane pair of this pass, small cross terms first, p0 x p0 last
            int ha, hb;
            if (nseg == 3) { ha = (seg == 1) ? 1 : 0; hb = (seg == 0) ? 1 : 0; }
            else { ha = (0x021010 >> (4 * (5 - seg))) & 0xf; hb = (0x201100 >> (4 * (5 - seg))) & 0xf; }
            if constexpr (!MN_MAJOR) {
              tma_load_4d(sa, &tmA, &full_bar[stage], kb * GEMM_BK, mt * GEMM_BM, ha, b);
              tma_load_4d(sb, &tmB, &full_bar[stage], kb * GEMM_BK, nt * BN, hb, b);
            } else {
#pragma unroll
              for (int h = 0; h < GEMM_BM / 64; ++h)
                tma_load_4d(sa + h * 8192, &tmA, &full_bar[stage], mt * GEMM_BM + h * 64, kb * GEMM_BK, ha, b);
#pragma unroll
              for (int h = 0; h < BN / 64; ++h)
                tma_load_4d(sb + h * 8192, &tmB, &full_bar[stage], nt * BN + h * 64, kb * GEMM_BK, hb, b);
            }
          } else if constexpr (!MN_MAJOR) {
            if (p.a_pr > 0) tma_load_4d(sa, &tmA, &full_bar[stage], kb * GEMM_BK, (mt * GEMM_BM) % p.a_pr, (mt * GEMM_BM) / p.a_pr, b);
            else tma_load_3d(sa, &tmA, &full_bar[stage], kb * GEMM_BK, mt * GEMM_BM, b);
            if (p.b_pr > 0) tma_load_4d(sb, &tmB, &full_bar[stage], kb * GEMM_BK, (nt * BN) % p.b_pr, (nt * BN) / p.b_pr, b);
            else tma_load_3d(sb, &tmB, &full_bar[stage], kb * GEMM_BK, nt * BN, b);
          } else if (p.a_pr > 0 || p.b_pr > 0) {
#pragma unroll
            for (int h = 0; h < GEMM_BM / 64; ++h) {
              const int m = mt * GEMM_BM + h * 64;
              if (p.a_pr > 0) tma_load_4d(sa + h * 8192, &tmA, &full_bar[stage], m % p.a_pr, kb * GEMM_BK, m / p.a_pr, b);
              else tma_load_3d(sa + h * 8192, &tmA, &full_bar[stage], m, kb * GEMM_BK, b);
            }
#pragma unroll
            for (int h = 0; h < BN / 64; ++h) {
              const int n = nt * BN + h * 64;
              if (p.b_pr > 0) tma_load_4d(sb + h * 8192, &tmB, &full_bar[stage], n % p.b_pr, kb * GEMM_BK, n / p.b_pr, b);
              else tma_load_3d(sb + h * 8192, &tmB, &full_bar[stage], n, kb * GEMM_BK, b);
            }
          } else {
            // operand stored [k][mn]: 64-wide mn boxes, each 64 k-rows x 128 B = 8 KB
#pragma unroll
            for (int h = 0; h < GEMM_BM / 64; ++h)
              tma_load_3d(sa + h * 8192, &tmA, &full_bar[stage], mt * GEMM_BM + h * 64, kb * GEMM_BK, b);
#pragma unroll
            for (int h = 0; h < BN / 64; ++h)
              tma_load_3d(sb + h * 8192, &tmB, &full_bar[stage], nt * BN + h * 64, kb * GEMM_BK, b);
          }
          if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
      }
    }
    return;
  }

  // ===================== MMA + epilogue (warpgroup 1: rows 0..63, warpgroup 2: rows 64..127) =====================
  regs_alloc<232>();
  const int h = wg - 1;
  const int wq = warp & 3;
  const int e_mode = (EK == EK_GENERIC) ? p.tile.mode : EpiTraits<EK>::mode;
  const int e_act = (EK == EK_GENERIC) ? p.tile.act : EpiTraits<EK>::act;
  const int e_layout = (EK == EK_GENERIC) ? p.tile.layout : EpiTraits<EK>::layout;
  const bool gated = e_mode == EPI_GATED_BF16;
  const bool out_f32 = (e_mode == EPI_RESID_F32) || (e_mode == EPI_STORE_F32);
  const int W = gated ? BN / 2 : BN;                                           // output columns per tile
  const NTile t = p.tile;
  // paired (8-byte fp32 / 4-byte bf16) stores need an even row pitch and an aligned base
  const bool vec_out = (t.ld % 2 == 0) && (p.out_batch_stride % 2 == 0) &&
                       (reinterpret_cast<uintptr_t>(t.out) & (out_f32 ? 7 : 3)) == 0;
  const bool vec_res = (p.ld_resid % 2 == 0) && (reinterpret_cast<uintptr_t>(p.resid) & 7) == 0;
  int stage = 0;
  uint32_t phase = 0;
  float acc[BN / 2];
  for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
    const int nt = tile % n_tiles;
    const int mt = (tile / n_tiles) % m_tiles;
    const int b = tile / (n_tiles * m_tiles);
    int prev = -1;
    for (int kk = 0; kk < num_kk; ++kk) {
      mbar_wait(&full_bar[stage], phase);
      const uint32_t sa = smem_u32(smem + stage * L::STAGE_BYTES);
      const uint32_t sb = sa + L::A_BYTES;
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < GEMM_BK / 16; ++k) {
        uint64_t adesc, bdesc;
        if constexpr (!MN_MAJOR) {
          // rows of 128 B (64 bf16 of K); 8-row swizzle atoms 1024 B apart; K step = 32 B; this warpgroup's 64 rows 8 KB in
          adesc = wgmma_desc(sa + h * 8192 + k * 32, 16, 1024, SWZ_128);
          bdesc = wgmma_desc(sb + k * 32, 16, 1024, SWZ_128);
        } else {
          // k-rows of 128 B (64 bf16 of M/N); 8 k-rows = 1024 B (SBO); next 64-wide mn block 8 KB (LBO); this warpgroup's
          // 64 rows are the h-th 64-wide box of A
          adesc = wgmma_desc(sa + h * 8192 + k * 2048, 8192, 1024, SWZ_128);
          bdesc = wgmma_desc(sb + k * 2048, 8192, 1024, SWZ_128);
        }
        const uint32_t scale_d = (kk | k) != 0 ? 1u : 0u;
        if constexpr (BN == 256) wgmma_m64n256k16_ss<MN_MAJOR ? 1 : 0, MN_MAJOR ? 1 : 0>(acc, adesc, bdesc, scale_d);
        else if constexpr (BN == 128) wgmma_m64n128k16_ss<MN_MAJOR ? 1 : 0, MN_MAJOR ? 1 : 0>(acc, adesc, bdesc, scale_d);
        else wgmma_m64n64k16_ss<MN_MAJOR ? 1 : 0, MN_MAJOR ? 1 : 0>(acc, adesc, bdesc, scale_d);
      }
      wgmma_commit();
      // keep one k-block in flight: the previous one has retired, so its stage goes back to the producer
      wgmma_wait<1>();
      if (prev >= 0 && lane == 0 && wq == 0) mbar_arrive(&empty_bar[prev]);
      prev = stage;
      if (++stage == STAGES) { stage = 0; phase ^= 1; }
    }
    wgmma_wait<0>();
    reg_fence(acc);
    if (prev >= 0 && lane == 0 && wq == 0) mbar_arrive(&empty_bar[prev]);

    // ------------------------------- epilogue from registers -------------------------------
    const int col0 = nt * W;
    const int ncols = min(W, p.out_cols - col0);
    const float* bias_tile = t.bias ? t.bias + nt * BN : nullptr;
#pragma unroll
    for (int half = 0; half < 2; ++half) {
      const int row = mt * GEMM_BM + h * 64 + wq * 16 + (lane >> 2) + half * 8;
      if (row >= p.M) continue;
      float rs = 1.0f;
      if (EpiTraits<EK>::rowscale && t.use_rowscale) rs = __ldg(p.rowscale + static_cast<long long>(b) * p.M + row);
      long long cm_off = 0;
      if (e_layout == LAYOUT_CHANNEL) cm_off = static_cast<long long>(row / p.cm_inner) * p.cm_pitch + row % p.cm_inner;
      const long long obase = static_cast<long long>(b) * p.out_batch_stride;
#pragma unroll
      for (int j = 0; j < BN / 8; ++j) {                    // fully unrolled: the accumulator stays in registers
        const int c = 8 * j + 2 * (lane & 3);                // tile-local output column of the pair
        if ((gated && j >= BN / 16) || c >= ncols) continue;
        const bool two = c + 1 < ncols;
        float v0 = acc[4 * j + 2 * half], v1 = acc[4 * j + 2 * half + 1];
        if (bias_tile) { v0 += __ldg(bias_tile + c); v1 += __ldg(bias_tile + c + 1); }
        if (gated) {
          // gate columns of the packed tile sit BN / 2 columns (BN / 16 fragment steps) to the right of their values
          constexpr int JM = BN / 8 - 1;
          const int jg = (j + BN / 16) & JM;
          float g0 = acc[4 * jg + 2 * half], g1 = acc[4 * jg + 2 * half + 1];
          if (bias_tile) { g0 += __ldg(bias_tile + BN / 2 + c); g1 += __ldg(bias_tile + BN / 2 + c + 1); }
          v0 *= apply_act(g0, e_act);
          v1 *= apply_act(g1, e_act);
        } else {
          v0 = apply_act(v0, e_act);
          v1 = apply_act(v1, e_act);
        }
        if (EpiTraits<EK>::rowscale && t.use_rowscale) { v0 *= rs; v1 *= rs; }
        const int col = col0 + c;
        if (e_layout == LAYOUT_CHANNEL) {
          __nv_bfloat16* o = reinterpret_cast<__nv_bfloat16*>(t.out) + obase + cm_off;
          o[static_cast<long long>(col) * t.ld] = __float2bfloat16(v0);
          if (two) o[static_cast<long long>(col + 1) * t.ld] = __float2bfloat16(v1);
        } else if (out_f32) {
          if (e_mode == EPI_RESID_F32) {
            const float* r = p.resid + static_cast<long long>(row) * p.ld_resid + col;
            if (two && vec_res) { const float2 r2 = *reinterpret_cast<const float2*>(r); v0 += r2.x; v1 += r2.y; }
            else { v0 += r[0]; if (two) v1 += r[1]; }
          }
          store_pair<true>(t.out, obase + static_cast<long long>(row) * t.ld + col, v0, v1, two, vec_out);
        } else {
          store_pair<false>(t.out, obase + static_cast<long long>(row) * t.ld + col, v0, v1, two, vec_out);
        }
      }
    }
  }
}

}  // namespace af2
