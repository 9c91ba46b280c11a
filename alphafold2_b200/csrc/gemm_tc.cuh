// Generic batched bf16 GEMM on sm_90a warpgroup tensor cores (wgmma) with TMA-staged operands and a programmable
// epilogue applied to the register accumulators.
// One kernel serves every dense contraction of the Evoformer block:
//
//   K-major mode  : C[b][m][n] = sum_k A[b][m][k] * B[b][n][k]      (Linear layers: B = weight [out,in];
//                                                                    triangle "outgoing" per channel)
//   MN-major mode : C[b][m][n] = sum_k A[b][k][m] * B[b][k][n]      (triangle "ingoing", outer-mean:
//                                                                    channel-major operands, k = row axis)
//
// Tiling: BM = 64 rows, BN in {64,128,256} accumulator columns, BK = 64.
// Warp roles (384 threads, three warpgroups):
//   warpgroup 0     TMA producers (the warpgroup hands its registers to the others):
//                     warp 0  A/B stages of every tile, in tile order
//                     warps 1, 2  residual sub-tiles of the tiles of MMA warpgroup 1 / 2 (EPI_RESID_F32 through TMA)
//   warpgroups 1, 2 "ping-pong" MMA + epilogue: the CTA's tiles alternate between them, each owns whole 64 x BN tiles.
//                   An ordered hand-off (named barriers 1, 2) lets one warpgroup issue its k loop only after the other
//                   has issued its own, so one warpgroup's epilogue runs while the other keeps the tensor cores busy.
// Epilogue (bias, activation, gate, row scale, residual): the fragment goes into 8 KB 128B-swizzled shared chunks (a ring
// per warpgroup) and leaves through TMA stores -- token-major [row][col] boxes, or channel-major [col][row] boxes (the
// transposing stage).  The residual arrives in the same chunks by TMA and is added in place.  Layouts TMA cannot express
// (odd pitches, unaligned bases, channel-major blocks that are not whole 64-row boxes) and the EK_GENERIC
// instantiations store straight from registers instead; the host chooses per call (GemmParams::epi_tma).
// The per-element k order is the same in both epilogues and for any tile size: results do not depend on the path.
#pragma once
#include "common.cuh"

namespace af2 {

constexpr int GEMM_BM = 64;
constexpr int GEMM_BK = 64;
constexpr int GEMM_EPI_BUFS = 4;          // epilogue chunks per MMA warpgroup
constexpr int GEMM_EPI_CHUNK = 8192;      // 64 rows x 128 B

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
  int epi_tma;                 // 1: epilogue through shared memory + TMA (tmC, and tmR for the residual); 0: register stores
  const float* rowscale;       // [batch*M] multiplier per row (mask), or nullptr
  const float* resid;          // EPI_RESID_F32: fp32 [M, ld_resid]
  long long ld_resid;
  long long out_batch_stride;  // elements
  int cm_inner, cm_pitch;      // channel-major: row r -> (r / cm_inner) * cm_pitch + r % cm_inner
  // Split-bf16 (strict precision) operands: every fp32 operand value v is stored as bf16 planes p0 = bf16(v),
  // p1 = bf16(v - p0), p2 = bf16(v - p0 - p1) (tensor maps of rank 4: k, row, plane, batch) and the k loop makes nseg = 6
  // passes over K, one per plane pair (A plane, B plane), smallest products first, all into the same fp32 accumulator:
  //   (0,2) (2,0) (1,1) (0,1) (1,0) (0,0)     (24 mantissa bits; (1,2) (2,1) (2,2) lie below 2^-24 and are dropped)
  // nseg = 1: plain bf16 operands, rank-3 maps.
  int nseg;
  // Operands gathered from several ranks ("pieces", alphafold2_b200/parallel.py): an all-gather concatenates the per-rank
  // shards [c][rows_p][k] along the outermost axis, so rows r = p * pr + rr of one channel are pr-row pieces piece_stride
  // apart.  Rank-4 maps (k | mn, row | k, piece, batch) address them in place -- one launch instead of one per piece.
  //   a_pr / b_pr: rows (K-major) or columns (MN-major) per piece of A / B; 0 = plain rank-3 map.
  int a_pr, b_pr;
  NTile tile;
};

template <int BN, int STAGES>
struct GemmSmem {
  static constexpr int A_BYTES = GEMM_BM * GEMM_BK * 2;   // 8 KB
  static constexpr int B_BYTES = BN * GEMM_BK * 2;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr int EPI_OFF = STAGES * STAGE_BYTES;                        // [2][GEMM_EPI_BUFS] chunks
  static constexpr int BIAS_OFF = EPI_OFF + 2 * GEMM_EPI_BUFS * GEMM_EPI_CHUNK;  // [2][BN] fp32
  static constexpr int BAR_OFF = BIAS_OFF + 2 * BN * 4;
  static constexpr int TOTAL = BAR_OFF + 256;
  static_assert(2 * STAGES + 4 * GEMM_EPI_BUFS <= 32, "mbarriers exceed their 256-byte region");
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
  uint64_t* efull_bar = empty_bar + STAGES;                 // [2][GEMM_EPI_BUFS] residual chunk landed
  uint64_t* eempty_bar = efull_bar + 2 * GEMM_EPI_BUFS;     // [2][GEMM_EPI_BUFS] chunk read out by its TMA store

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int wg = warp >> 2;

  const int e_mode = (EK == EK_GENERIC) ? p.tile.mode : EpiTraits<EK>::mode;
  const int e_act = (EK == EK_GENERIC) ? p.tile.act : EpiTraits<EK>::act;
  const int e_layout = (EK == EK_GENERIC) ? p.tile.layout : EpiTraits<EK>::layout;
  const bool epi_tma = EK != EK_GENERIC && p.epi_tma;

  if (threadIdx.x == 0) {
    prefetch_tmap(&tmA);
    prefetch_tmap(&tmB);
    if (epi_tma) prefetch_tmap(&tmC);
    if (epi_tma && e_mode == EPI_RESID_F32) prefetch_tmap(&tmR);
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 1);     // the one MMA warpgroup that consumed the stage
    }
    for (int s = 0; s < 2 * GEMM_EPI_BUFS; ++s) {
      mbar_init(&efull_bar[s], 1);
      mbar_init(&eempty_bar[s], 1);    // the storing thread, once the TMA store has read the chunk
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
  const bool gated = e_mode == EPI_GATED_BF16;
  const int W = gated ? BN / 2 : BN;                // output columns per tile

  if (wg == 0) {
    // ================================ TMA producers ================================
    regs_dealloc<40>();
    if (threadIdx.x == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
        const int nt = tile % n_tiles;
        const int mt = (tile / n_tiles) % m_tiles;
        const int b = tile / (n_tiles * m_tiles);
        const int m0 = mt * GEMM_BM;
        for (int kk = 0; kk < num_kk; ++kk) {
          const int seg = kk / num_kb, kb = kk - seg * num_kb;
          mbar_wait(&empty_bar[stage], phase ^ 1);
          uint8_t* sa = smem + stage * L::STAGE_BYTES;
          uint8_t* sb = sa + L::A_BYTES;
          mbar_arrive_expect_tx(&full_bar[stage], L::STAGE_BYTES);
          if (nseg > 1) {
            // split operands (rank-4 maps): plane pair of this pass, small cross terms first, p0 x p0 last
            const int ha = (0x021010 >> (4 * (5 - seg))) & 0xf, hb = (0x201100 >> (4 * (5 - seg))) & 0xf;
            if constexpr (!MN_MAJOR) {
              tma_load_4d(sa, &tmA, &full_bar[stage], kb * GEMM_BK, m0, ha, b);
              tma_load_4d(sb, &tmB, &full_bar[stage], kb * GEMM_BK, nt * BN, hb, b);
            } else {
              tma_load_4d(sa, &tmA, &full_bar[stage], m0, kb * GEMM_BK, ha, b);
#pragma unroll
              for (int h = 0; h < BN / 64; ++h)
                tma_load_4d(sb + h * 8192, &tmB, &full_bar[stage], nt * BN + h * 64, kb * GEMM_BK, hb, b);
            }
          } else if constexpr (!MN_MAJOR) {
            if (p.a_pr > 0) tma_load_4d(sa, &tmA, &full_bar[stage], kb * GEMM_BK, m0 % p.a_pr, m0 / p.a_pr, b);
            else tma_load_3d(sa, &tmA, &full_bar[stage], kb * GEMM_BK, m0, b);
            if (p.b_pr > 0) tma_load_4d(sb, &tmB, &full_bar[stage], kb * GEMM_BK, (nt * BN) % p.b_pr, (nt * BN) / p.b_pr, b);
            else tma_load_3d(sb, &tmB, &full_bar[stage], kb * GEMM_BK, nt * BN, b);
          } else {
            // operand stored [k][mn]: 64-wide mn boxes, each 64 k-rows x 128 B = 8 KB
            if (p.a_pr > 0) tma_load_4d(sa, &tmA, &full_bar[stage], m0 % p.a_pr, kb * GEMM_BK, m0 / p.a_pr, b);
            else tma_load_3d(sa, &tmA, &full_bar[stage], m0, kb * GEMM_BK, b);
#pragma unroll
            for (int h = 0; h < BN / 64; ++h) {
              const int n = nt * BN + h * 64;
              if (p.b_pr > 0) tma_load_4d(sb + h * 8192, &tmB, &full_bar[stage], n % p.b_pr, kb * GEMM_BK, n / p.b_pr, b);
              else tma_load_3d(sb + h * 8192, &tmB, &full_bar[stage], n, kb * GEMM_BK, b);
            }
          }
          if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
      }
    } else if ((warp == 1 || warp == 2) && lane == 0 && epi_tma && e_mode == EPI_RESID_F32) {
      // residual of MMA warpgroup (warp - 1)'s tiles, 64 x 32 fp32 chunks in the order its epilogue adds them; runs ahead
      // by up to GEMM_EPI_BUFS chunks, independently of the A/B stages
      const int hh = warp - 1;
      int e = 0;
      for (int i = hh; blockIdx.x + i * gridDim.x < total_tiles; i += 2) {
        const int tile = blockIdx.x + i * gridDim.x;
        const int nt = tile % n_tiles;
        const int mt = (tile / n_tiles) % m_tiles;
        for (int ch = 0; ch < BN / 32; ++ch, ++e) {
          const int buf = hh * GEMM_EPI_BUFS + e % GEMM_EPI_BUFS;
          mbar_wait(&eempty_bar[buf], ((e / GEMM_EPI_BUFS) & 1) ^ 1);
          mbar_arrive_expect_tx(&efull_bar[buf], GEMM_EPI_CHUNK);
          tma_load_2d(smem + L::EPI_OFF + buf * GEMM_EPI_CHUNK, &tmR, &efull_bar[buf], nt * W + ch * 32, mt * GEMM_BM);
        }
      }
    }
    return;
  }

  // ============== MMA + epilogue: warpgroup hh = wg - 1 owns the CTA's tiles i = hh, hh + 2, hh + 4, ... ==============
  regs_alloc<232>();
  const int hh = wg - 1;
  const int wq = warp & 3;
  const int tid = threadIdx.x & 127;
  const bool out_f32 = (e_mode == EPI_RESID_F32) || (e_mode == EPI_STORE_F32);
  const NTile t = p.tile;
  // paired (8-byte fp32 / 4-byte bf16) stores need an even row pitch and an aligned base
  const bool vec_out = (t.ld % 2 == 0) && (p.out_batch_stride % 2 == 0) &&
                       (reinterpret_cast<uintptr_t>(t.out) & (out_f32 ? 7 : 3)) == 0;
  const bool vec_res = (p.ld_resid % 2 == 0) && (reinterpret_cast<uintptr_t>(p.resid) & 7) == 0;
  float* sbias = reinterpret_cast<float*>(smem + L::BIAS_OFF) + hh * BN;
  uint8_t* sepi = smem + L::EPI_OFF + hh * GEMM_EPI_BUFS * GEMM_EPI_CHUNK;
  const int bar_self = 3 + hh;                       // this warpgroup's 128 threads
  int e = 0;                                         // epilogue chunks this warpgroup has used
  float acc[BN / 2];
  for (int i = hh; blockIdx.x + i * gridDim.x < total_tiles; i += 2) {
    const int tile = blockIdx.x + i * gridDim.x;
    const int nt = tile % n_tiles;
    const int mt = (tile / n_tiles) % m_tiles;
    const int b = tile / (n_tiles * m_tiles);
    // the bias of the tile goes to shared memory once (the previous epilogue has finished reading it)
    named_bar_sync(bar_self, 128);
    if (t.bias)
      for (int c = tid; c < BN; c += 128) sbias[c] = nt * BN + c < p.N ? __ldg(t.bias + nt * BN + c) : 0.0f;

    // k loop; stage ring position = k-blocks the producer issued for the CTA's tiles 0 .. i-1
    const int g0 = i * num_kk;
    int stage = g0 % STAGES;
    uint32_t phase = (g0 / STAGES) & 1;
    if (i > 0) named_bar_sync(1 + hh, 256);          // tile i - 1 (other warpgroup) has issued its k loop
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
          // rows of 128 B (64 bf16 of K); 8-row swizzle atoms 1024 B apart; K step = 32 B
          adesc = wgmma_desc(sa + k * 32, 16, 1024, SWZ_128);
          bdesc = wgmma_desc(sb + k * 32, 16, 1024, SWZ_128);
        } else {
          // k-rows of 128 B (64 bf16 of M/N); 8 k-rows = 1024 B (SBO); next 64-wide mn block 8 KB (LBO)
          adesc = wgmma_desc(sa + k * 2048, 8192, 1024, SWZ_128);
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
    if (blockIdx.x + (i + 1) * gridDim.x < total_tiles) named_bar_arrive(2 - hh, 256);   // tile i + 1 may start
    wgmma_wait<0>();
    reg_fence(acc);
    if (prev >= 0 && lane == 0 && wq == 0) mbar_arrive(&empty_bar[prev]);
    named_bar_sync(bar_self, 128);                   // bias of the tile visible

    const int col0 = nt * W;
    const int r_lo = wq * 16 + (lane >> 2);          // tile-local rows r_lo, r_lo + 8 of this thread
    if (epi_tma) {
      // ---------------- epilogue through 8 KB swizzled chunks + TMA stores (compile-time EK) ----------------
      constexpr int MODE = EpiTraits<EK>::mode, ACT = EpiTraits<EK>::act, LAYOUT = EpiTraits<EK>::layout;
      constexpr bool F32 = MODE == EPI_RESID_F32 || MODE == EPI_STORE_F32;
      constexpr bool GATED = MODE == EPI_GATED_BF16;
      constexpr int CJ = F32 ? 4 : 8;                // fragment column steps (8 columns) per chunk
      constexpr int NJ = GATED ? BN / 16 : BN / 8;
      constexpr int NCH = NJ / CJ >= 1 ? NJ / CJ : 1;
      float rs[2] = {1.0f, 1.0f};
      if (EpiTraits<EK>::rowscale && t.use_rowscale) {
#pragma unroll
        for (int half = 0; half < 2; ++half) {
          const int row = mt * GEMM_BM + r_lo + half * 8;
          if (row < p.M) rs[half] = __ldg(p.rowscale + static_cast<long long>(b) * p.M + row);
        }
      }
      const int q2 = 2 * (lane & 3);
#pragma unroll
      for (int ch = 0; ch < NCH; ++ch, ++e) {
        const int buf = e % GEMM_EPI_BUFS;
        const uint32_t par = (e / GEMM_EPI_BUFS) & 1;
        if (MODE == EPI_RESID_F32) mbar_wait(&efull_bar[hh * GEMM_EPI_BUFS + buf], par);
        else mbar_wait(&eempty_bar[hh * GEMM_EPI_BUFS + buf], par ^ 1);
        uint8_t* sc = sepi + buf * GEMM_EPI_CHUNK;
#pragma unroll
        for (int jj = 0; jj < CJ; ++jj) {
          const int j = ch * CJ + jj;
          if (j >= NJ) break;
          const int c = 8 * j + q2;                  // tile-local output column of the pair
          const int cl = 8 * jj + q2;                // chunk-local
#pragma unroll
          for (int half = 0; half < 2; ++half) {
            const int r = r_lo + half * 8;
            float v0 = acc[4 * j + 2 * half], v1 = acc[4 * j + 2 * half + 1];
            if (t.bias) { v0 += sbias[c]; v1 += sbias[c + 1]; }
            if constexpr (GATED) {
              const int jg = j + BN / 16;
              float g0 = acc[4 * jg + 2 * half], g1 = acc[4 * jg + 2 * half + 1];
              if (t.bias) { g0 += sbias[BN / 2 + c]; g1 += sbias[BN / 2 + c + 1]; }
              v0 *= apply_act(g0, ACT);
              v1 *= apply_act(g1, ACT);
            } else {
              v0 = apply_act(v0, ACT);
              v1 = apply_act(v1, ACT);
            }
            if (EpiTraits<EK>::rowscale && t.use_rowscale) { v0 *= rs[half]; v1 *= rs[half]; }
            if constexpr (LAYOUT == LAYOUT_CHANNEL) {
              // [col][row] box: 128-byte lines of 64 rows, 16-byte chunk (r / 8) swizzled by col % 8
              __nv_bfloat16* o0 = reinterpret_cast<__nv_bfloat16*>(sc + cl * 128 + (((r >> 3) ^ (cl & 7)) << 4)) + (r & 7);
              __nv_bfloat16* o1 = reinterpret_cast<__nv_bfloat16*>(sc + (cl + 1) * 128 + (((r >> 3) ^ ((cl + 1) & 7)) << 4)) + (r & 7);
              *o0 = __float2bfloat16(v0);
              *o1 = __float2bfloat16(v1);
            } else if constexpr (F32) {
              // [row][32 fp32] box
              float2* o = reinterpret_cast<float2*>(sc + r * 128 + (((cl >> 2) ^ (r & 7)) << 4) + (cl & 3) * 4);
              if constexpr (MODE == EPI_RESID_F32) { const float2 rv = *o; v0 += rv.x; v1 += rv.y; }
              *o = make_float2(v0, v1);
            } else {
              // [row][64 bf16] box
              *reinterpret_cast<uint32_t*>(sc + r * 128 + (((cl >> 3) ^ (r & 7)) << 4) + (cl & 7) * 2) = pack_bf16x2(v0, v1);
            }
          }
        }
        fence_proxy_async_smem();
        named_bar_sync(bar_self, 128);
        if (tid == 0) {
          const int m0 = mt * GEMM_BM;
          if constexpr (LAYOUT == LAYOUT_CHANNEL)
            tma_store_4d(&tmC, sc, m0 % p.cm_inner, m0 / p.cm_inner, col0 + ch * 64, b);
          else
            tma_store_3d(&tmC, sc, col0 + ch * (F32 ? 32 : 64), m0, b);
          tma_store_commit();
          if (ch > 0) {
            tma_store_wait_read<1>();
            mbar_arrive(&eempty_bar[hh * GEMM_EPI_BUFS + (e - 1) % GEMM_EPI_BUFS]);
          }
        }
      }
      if (tid == 0) {
        tma_store_wait_read<0>();
        mbar_arrive(&eempty_bar[hh * GEMM_EPI_BUFS + (e - 1) % GEMM_EPI_BUFS]);
      }
    } else {
      // ------------------------------- epilogue from registers -------------------------------
      const int ncols = min(W, p.out_cols - col0);
#pragma unroll
      for (int half = 0; half < 2; ++half) {
        const int row = mt * GEMM_BM + r_lo + half * 8;
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
          if (t.bias) { v0 += sbias[c]; v1 += sbias[c + 1]; }
          if (gated) {
            // gate columns of the packed tile sit BN / 2 columns (BN / 16 fragment steps) to the right of their values
            constexpr int JM = BN / 8 - 1;
            const int jg = (j + BN / 16) & JM;
            float g0 = acc[4 * jg + 2 * half], g1 = acc[4 * jg + 2 * half + 1];
            if (t.bias) { g0 += sbias[BN / 2 + c]; g1 += sbias[BN / 2 + c + 1]; }
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
  if (epi_tma && tid == 0) tma_store_wait<0>();
}

}  // namespace af2
