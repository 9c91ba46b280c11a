// Fused GEGLU feed-forward on sm_90a warpgroup tensor cores:
//
//   x[t] += W2 · h[t] + b2,   h[t] = (u + b_u) · gelu(g + b_g),   [u | g] = W1 · xn[t]        (xn = LayerNorm(x), bf16)
//
// The hidden activation h never leaves the SM: each MMA warpgroup computes it chunk by chunk (HC hidden units) into
// registers and feeds it straight back to the tensor cores as the register A operand of the second GEMM, whose fp32
// accumulator out[64 x D] stays in registers for the whole row tile.  Compared with two GEMM launches this removes the
// bf16 round trip of h through HBM (2 x 2 x T x hidden bytes) and reads each weight byte once per 128 rows instead of
// once per 64-row tile.
//
// Warp roles (384 threads, three warpgroups), one persistent CTA per SM, 128-row tiles:
//   warpgroup 0     TMA producer (one thread): per tile, the two 64 x D xn slices, then W1 / W2 chunk by chunk through a
//                   ring of 512 HC-byte slots that both MMA warpgroups read (a slot is free once both have retired it).
//   warpgroups 1, 2 rows 0-63 / 64-127 of the tile.  Per hidden chunk c:
//                     GEMM1  S[64 x 2 HC] = xn · [W1 value rows of c | W1 gate rows of c]ᵀ   (SS, K = D)
//                     GEGLU  h = (S_u + b_u) · gelu(S_g + b_g), rounded to bf16 in the m64k16 A-fragment layout
//                     GEMM2  out += h · W2[:, c]ᵀ                                            (RS, K = HC)
//                   GEMM2(c) and GEMM1(c + 1) are issued back to back as one unit; the two warpgroups' units take turns
//                   on the tensor cores (named barriers 1, 2), so one warpgroup's GEGLU runs under the other's MMAs.
//
// Results equal the two-GEMM path (gemm_tc.cuh, EK_GATED_TOK_GELU then EK_RESID_F32) bit for bit: the same k16 sequence
// over D for S, the same GEGLU expression and bf16 rounding of h, the same ascending k16 sequence over the hidden units
// into one fp32 accumulator, then + b2, then + x.
#pragma once
#include "common.cuh"

namespace af2 {

constexpr int FF_BM = 128;         // rows per tile, 64 per MMA warpgroup
constexpr int FF_THREADS = 384;

// HC: hidden units per chunk
template <int D, int HC>
struct FfSmem {
  static_assert(D == 128 || D == 256, "fused feed-forward: D must be 128 or 256");
  static_assert(HC == 32 || HC == 64, "fused feed-forward: HC must be 32 or 64");
  static constexpr int SLOT = HC * 512;                                // weight ring slot: W1 [2 HC rows x 128 k] or W2 [D rows x HC k]
  static constexpr int W1_BLOCK = HC * 256;                            // W1 [2 HC rows x 64 k]: value rows, then gate rows
  static constexpr int XN_BYTES = 64 * D * 2;                          // one warpgroup's xn slice: D / 64 boxes of 64 x 64
  static constexpr int RING_OFF = 2 * XN_BYTES;
  static constexpr int SLOTS = (232448 - RING_OFF - 256) / SLOT;
  static constexpr int W1_SLOTS = D / 128;                             // W1 slots per chunk (two 64-k blocks each)
  static constexpr int BAR_OFF = RING_OFF + SLOTS * SLOT;
  static constexpr int TOTAL = BAR_OFF + 256;
  static_assert(2 * SLOTS + 4 <= 32, "mbarriers exceed their 256-byte region");
  static_assert(SLOTS >= W1_SLOTS + 1, "a unit (GEMM2 + GEMM1) must fit the ring");
  static_assert(TOTAL <= 232448, "exceeds the 227 KB of shared memory a CTA can use");
};

struct FfParams {
  float* x;             // [T, D] fp32 residual stream, updated in place
  const float* b1;      // packed like W1: per 128 hidden units [128 value | 128 gate]
  const float* b2;      // [D]
  int T, hidden;        // hidden % 128 == 0
};

template <int D, int HC>
__global__ void __launch_bounds__(FF_THREADS, 1)
ff_fused_kernel(const __grid_constant__ CUtensorMap tmX, const __grid_constant__ CUtensorMap tmW1,
                const __grid_constant__ CUtensorMap tmW2, const __grid_constant__ FfParams p) {
  using L = FfSmem<D, HC>;
  constexpr int NS = L::SLOTS, W1S = L::W1_SLOTS, SLOT = L::SLOT, W1B = L::W1_BLOCK;
  constexpr int CPT = 128 / HC;                      // chunks per 256-row tile of the packed W1
  extern __shared__ __align__(1024) uint8_t smem[];
  if ((smem_u32(smem) & 1023u) != 0) __trap();
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + L::BAR_OFF);
  uint64_t* empty_bar = full_bar + NS;
  uint64_t* xfull_bar = empty_bar + NS;      // [2] xn slice of MMA warpgroup h landed
  uint64_t* xempty_bar = xfull_bar + 2;      // [2] its last GEMM1 of the tile has retired

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int wg = warp >> 2;

  if (threadIdx.x == 0) {
    prefetch_tmap(&tmX);
    prefetch_tmap(&tmW1);
    prefetch_tmap(&tmW2);
    for (int s = 0; s < NS; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 2);           // both MMA warpgroups read every slot
    }
    for (int h = 0; h < 2; ++h) {
      mbar_init(&xfull_bar[h], 1);
      mbar_init(&xempty_bar[h], 1);
    }
    fence_barrier_init();
  }
  __syncthreads();
  pdl_launch_dependents();
  pdl_wait();

  const int tiles = (p.T + FF_BM - 1) / FF_BM;
  const int nc = p.hidden / HC;

  if (wg == 0) {
    // ================================ TMA producer ================================
    regs_dealloc<24>();
    if (threadIdx.x == 0) {
      int slot = 0;
      uint32_t phase = 0;
      int it = 0;
      for (int tile = blockIdx.x; tile < tiles; tile += gridDim.x, ++it) {
        const int r0 = tile * FF_BM;
        // the residual rows the tile epilogue reads, into L2 a whole tile of MMAs ahead
        bulk_prefetch_l2(p.x + static_cast<long long>(r0) * D, static_cast<uint32_t>(min(FF_BM, p.T - r0) * D * 4));
        for (int h = 0; h < 2; ++h) {
          mbar_wait(&xempty_bar[h], (it & 1) ^ 1);
          mbar_arrive_expect_tx(&xfull_bar[h], L::XN_BYTES);
#pragma unroll
          for (int kb = 0; kb < D / 64; ++kb)
            tma_load_2d(smem + h * L::XN_BYTES + kb * 8192, &tmX, &xfull_bar[h], kb * 64, r0 + h * 64);
        }
        for (int c = 0; c < nc; ++c) {
          // value rows of chunk c in the packed W1 ([128 value | 128 gate] per 256 rows); its gate rows are 128 further
          const int rv = (c / CPT) * 256 + (c % CPT) * HC;
#pragma unroll
          for (int s = 0; s < W1S; ++s) {
            mbar_wait(&empty_bar[slot], phase ^ 1);
            uint8_t* dst = smem + L::RING_OFF + slot * SLOT;
            mbar_arrive_expect_tx(&full_bar[slot], SLOT);
#pragma unroll
            for (int q = 0; q < 2; ++q) {
              const int k0 = (2 * s + q) * 64;
              tma_load_2d(dst + q * W1B, &tmW1, &full_bar[slot], k0, rv);
              tma_load_2d(dst + q * W1B + W1B / 2, &tmW1, &full_bar[slot], k0, rv + 128);
            }
            if (++slot == NS) { slot = 0; phase ^= 1; }
          }
          mbar_wait(&empty_bar[slot], phase ^ 1);
          mbar_arrive_expect_tx(&full_bar[slot], D * HC * 2);
          tma_load_2d(smem + L::RING_OFF + slot * SLOT, &tmW2, &full_bar[slot], c * HC, 0);
          if (++slot == NS) { slot = 0; phase ^= 1; }
        }
      }
    }
    return;
  }

  // ==================== MMA + GEGLU + tile epilogue: warpgroup hh owns rows hh * 64 .. hh * 64 + 63 ====================
  // out (D / 2) + S (64) + h (16) registers are live across the MMAs: at D = 256 ptxas needs 240 to keep the wgmmas
  // asynchronous (at 232 it serialises them); the producer thread runs in 24
  regs_alloc<240>();
  const int hh = wg - 1;
  const int wq = warp & 3;
  const bool leader = wq == 0 && lane == 0;
  // descriptor of the warpgroup's xn slice; k steps add (byte offset >> 4) to the start-address field, which cannot carry
  // out of it below 256 KB.  opaque() keeps the compiler from precomputing every step's descriptor, which would hold
  // registers the accumulators need.
  const uint64_t xdesc = wgmma_desc(smem_u32(smem + hh * L::XN_BYTES), 16, 1024, SWZ_128);
  auto opaque = [](uint64_t v) { asm volatile("" : "+l"(v)); return v; };
  const uint32_t ring = smem_u32(smem + L::RING_OFF);
  const int r_lo = wq * 16 + (lane >> 2);            // tile-local rows r_lo, r_lo + 8 of this thread
  const int q2 = 2 * (lane & 3);
  // units issued per warpgroup: per tile GEMM1(0), then GEMM2(c) + GEMM1(c + 1) for c < nc - 1, then GEMM2(nc - 1)
  const int units = (tiles - static_cast<int>(blockIdx.x) + static_cast<int>(gridDim.x) - 1) / static_cast<int>(gridDim.x) * (nc + 1);
  int u = 0;
  int slot = 0;
  uint32_t phase = 0;
  float out[D / 2];
  float sacc[HC];                                    // m64n(2 HC): value columns 0 .. HC - 1, gate columns HC .. 2 HC - 1
  uint32_t ha[HC / 16][4];                           // h of the chunk as the m64k16 A fragments of GEMM2

  auto next_slot = [&]() { if (++slot == NS) { slot = 0; phase ^= 1; } };
  // The MMAs of the two warpgroups take turns: a warpgroup issues its unit once the other's previous unit has (all but) retired.
  // With both warpgroups' wgmmas in flight at once they would share the tensor cores and finish together, and the two
  // GEGLUs would then run together with the tensor cores idle.
  auto unit_begin = [&]() { if (u > 0 || hh == 1) named_bar_sync(1 + hh, 256); };
  auto unit_end = [&]() { if (hh == 0 || u + 1 < units) named_bar_arrive(2 - hh, 256); ++u; };
  auto release = [&](int s) { if (leader) mbar_arrive(&empty_bar[s]); };
  // out += h · W2[:, c]ᵀ: W2 chunk [D rows][HC k], rows of 2 HC bytes (128B / 64B swizzle), 8-row atoms 16 HC bytes apart
  auto issue_gemm2 = [&](int c) -> int {
    mbar_wait(&full_bar[slot], phase);
    wgmma_fence();
    const uint64_t b0 = opaque(wgmma_desc(ring + slot * SLOT, 16, 16 * HC, HC == 64 ? SWZ_128 : SWZ_64));
#pragma unroll
    for (int k = 0; k < HC / 16; ++k) {
      const uint64_t bdesc = b0 + (k * 32 >> 4);
      const uint32_t scale_d = (c | k) != 0 ? 1u : 0u;
      if constexpr (D == 256) wgmma_m64n256k16_rs<0>(out, ha[k], bdesc, scale_d);
      else wgmma_m64n128k16_rs<0>(out, ha[k], bdesc, scale_d);
    }
    wgmma_commit();
    const int s = slot;
    next_slot();
    return s;
  };
  // S = xn · [value rows | gate rows]ᵀ, one commit group per slot (two 64-k blocks of 128 W1 rows each)
  auto issue_gemm1 = [&](int (&w1slot)[W1S]) {
#pragma unroll
    for (int s = 0; s < W1S; ++s) {
      mbar_wait(&full_bar[slot], phase);
      wgmma_fence();
      const uint64_t a0 = opaque(xdesc), b0 = opaque(wgmma_desc(ring + slot * SLOT, 16, 1024, SWZ_128));
#pragma unroll
      for (int q = 0; q < 2; ++q) {
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const int kb = 2 * s + q;
          const uint64_t adesc = a0 + ((kb * 8192 + k * 32) >> 4);
          const uint64_t bdesc = b0 + ((q * W1B + k * 32) >> 4);
          if constexpr (HC == 64) wgmma_m64n128k16_ss<0, 0>(sacc, adesc, bdesc, (kb | k) != 0 ? 1u : 0u);
          else wgmma_m64n64k16_ss<0, 0>(sacc, adesc, bdesc, (kb | k) != 0 ? 1u : 0u);
        }
      }
      wgmma_commit();
      w1slot[s] = slot;
      next_slot();
    }
  };
  // retires GEMM1 (the only groups still pending), returns its slots, then GEGLU of chunk cn (the EK_GATED_TOK_GELU
  // epilogue) into GEMM2's A fragments
  auto finish_gemm1 = [&](const int (&w1slot)[W1S], int cn) {
    if constexpr (W1S == 2) {
      wgmma_wait<1>();
      release(w1slot[0]);
    }
    unit_end();                                      // the other warpgroup's unit queues behind the last k-blocks
    wgmma_wait<0>();
    release(w1slot[W1S - 1]);
    if (cn == nc - 1 && leader) mbar_arrive(&xempty_bar[hh]);   // last GEMM1 of the tile: the xn slice may be reloaded
    reg_fence(sacc);
#pragma unroll
    for (int i = 0; i < HC / 16; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) asm volatile("" : "+r"(ha[i][j])::"memory");     // GEMM2 read h until now
    const float* bu = p.b1 + (cn / CPT) * 256 + (cn % CPT) * HC;
#pragma unroll
    for (int j = 0; j < HC / 8; ++j) {
      const int col = 8 * j + q2;
      const float2 bv = __ldg(reinterpret_cast<const float2*>(bu + col));
      const float2 bg = __ldg(reinterpret_cast<const float2*>(bu + 128 + col));
#pragma unroll
      for (int half = 0; half < 2; ++half) {
        float v0 = sacc[4 * j + 2 * half] + bv.x, v1 = sacc[4 * j + 2 * half + 1] + bv.y;
        const float g0 = sacc[4 * (j + HC / 8) + 2 * half] + bg.x;
        const float g1 = sacc[4 * (j + HC / 8) + 2 * half + 1] + bg.y;
        v0 *= gelu_erf(g0);
        v1 *= gelu_erf(g1);
        // m64k16 A fragment of k-step j / 2: a0 / a1 = rows lo / hi of its first 8 columns, a2 / a3 of the next 8
        ha[j >> 1][(j & 1) * 2 + half] = pack_bf16x2(v0, v1);
      }
    }
  };

  int it = 0;
  for (int tile = blockIdx.x; tile < tiles; tile += gridDim.x, ++it) {
    mbar_wait(&xfull_bar[hh], it & 1);
    int w1slot[W1S];
    unit_begin();
    issue_gemm1(w1slot);
    finish_gemm1(w1slot, 0);
    for (int c = 0; c + 1 < nc; ++c) {
      unit_begin();
      const int w2slot = issue_gemm2(c);
      issue_gemm1(w1slot);
      wgmma_wait<W1S>();
      release(w2slot);
      finish_gemm1(w1slot, c + 1);
    }
    unit_begin();
    const int w2slot = issue_gemm2(nc - 1);
    wgmma_wait<0>();
    unit_end();
    release(w2slot);
    reg_fence(out);
#pragma unroll
    for (int i = 0; i < HC / 16; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) asm volatile("" : "+r"(ha[i][j])::"memory");

    // ---- tile epilogue: x = (out + b2) + x for the warpgroup's 64 rows (the EK_RESID_F32 order) ----
#pragma unroll
    for (int half = 0; half < 2; ++half) {
      const int row = tile * FF_BM + hh * 64 + r_lo + half * 8;
      if (row < p.T) {
        float* xr = p.x + static_cast<long long>(row) * D;
#pragma unroll
        for (int j = 0; j < D / 8; ++j) {
          const int col = 8 * j + q2;
          const float2 b = __ldg(reinterpret_cast<const float2*>(p.b2 + col));
          const float2 r = *reinterpret_cast<const float2*>(xr + col);
          float v0 = out[4 * j + 2 * half] + b.x, v1 = out[4 * j + 2 * half + 1] + b.y;
          v0 += r.x;
          v1 += r.y;
          *reinterpret_cast<float2*>(xr + col) = make_float2(v0, v1);
        }
      }
    }
  }
}

}  // namespace af2
