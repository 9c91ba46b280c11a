// Fused  LayerNorm -> multi-segment projection GEMM  for K = d in {128, 192, 256} on sm_90a wgmma.
//
//   out_seg = epilogue_seg( LN(x)[T, d] * Wcat[tiles of 256 rows, d]^T + bcat )
// x is the fp32 token-major residual stream; the LayerNorm affine is folded into the packed operands on the host
// (W' = W diag(gamma), b' = W beta + b, alphafold2_b200/ops.py _cat_segments), so the kernel computes (x - mean) * rstd
// only.  This is every LN -> Linear cluster of the reference: alphafold2.py:82-85, 210-217 + 114-118, 269-276 + 297-311,
// 330-340.  Against the unfused LayerNorm kernel + GEMM it saves the bf16 round trip of the normalised activations through
// HBM, and one launch serves several outputs with different epilogue programs (q|k|v + gate; left + right + out-gate ...).
//
// Work item = 128 rows.  The MMA warpgroups (1, 2) normalise the item's rows straight into the 128B-swizzled A tile in
// shared memory (one warp per row, one 16-byte chunk of 8 channels per lane); the tile then stays resident while EVERY
// 256-column weight tile of every segment streams past it through a TMA ring fed by warpgroup 0.  Each MMA warpgroup
// runs wgmma m64n256k16 on its 64 rows and applies the segment's epilogue from the register fragment (the same
// programs as gemm_tc.cuh: bias, sigmoid / erf-GELU, GEGLU gate, row mask, token- or channel-major bf16 store).
// Persistent CTAs; the producer runs ahead into the next item's weight tiles while the A tile is being rebuilt.
#pragma once
#include "gemm_tc.cuh"

namespace af2 {

constexpr int PROJ_THREADS = 384;
constexpr int PROJ_MAX_SEG = 3;
constexpr int PROJ_BN = 256;               // accumulator columns per weight tile
constexpr int PROJ_STAGES = 4;

struct ProjSeg {
  int tile0, ntiles;     // weight tiles (256 accumulator columns each) [tile0, tile0 + ntiles)
  int kind;              // EpiKind: EK_STORE_TOK, EK_STORE_TOK_SIG, EK_STORE_CH, EK_GATED_TOK_GELU, EK_GATED_CH_SIG
  int out_cols;          // valid output columns of the segment
  void* out;
  long long ld;          // token layout: row stride (elements); channel layout: channel stride (elements)
};

struct ProjParams {
  const float* x;                // [T, d] fp32 token-major residual stream
  long long T;
  int d;
  float inv_d, eps;
  const unsigned char* rowmask;  // [T] bool row scale (channel-major kinds) or nullptr
  const float* bcat;             // fp32 bias per accumulator column of Wcat (LayerNorm shift folded in)
  int nseg;
  ProjSeg seg[PROJ_MAX_SEG];
  int n_tiles_total;
  int m_tiles;                   // ceil(T / 128)
};

struct ProjSmem {
  static constexpr int A_BYTES = 128 * 256 * 2;                 // 128 rows x d <= 256, four 16 KB k-blocks
  static constexpr int B_STAGE = PROJ_BN * GEMM_BK * 2;          // 32 KB
  static constexpr int B_OFF = A_BYTES;
  static constexpr int BAR_OFF = B_OFF + PROJ_STAGES * B_STAGE;
  static constexpr int TOTAL = BAR_OFF + 128;
  static_assert(TOTAL <= 232448, "exceeds the 227 KB of shared memory a CTA can use");
};

__device__ __forceinline__ void proj_bar_sync() { asm volatile("bar.sync 1, 256;" ::: "memory"); }   // the two MMA warpgroups

// epilogue of one 256-column weight tile of segment sg, specialised on its kind (EpiTraits: mode, activation, layout)
template <int EK>
__device__ __forceinline__ void proj_epilogue(const float (&acc)[PROJ_BN / 2], const ProjParams& p, const ProjSeg& sg, int mt, int nt,
                                              int h, int wq, int lane) {
  constexpr bool gated = EpiTraits<EK>::mode == EPI_GATED_BF16;
  constexpr bool chan = EpiTraits<EK>::layout == LAYOUT_CHANNEL;
  constexpr int act = EpiTraits<EK>::act;
  constexpr int W = gated ? PROJ_BN / 2 : PROJ_BN;
  const int col0 = (nt - sg.tile0) * W;
  const int ncols = min(W, sg.out_cols - col0);
  const float* bias = p.bcat + static_cast<long long>(nt) * PROJ_BN;
#pragma unroll
  for (int half = 0; half < 2; ++half) {
    const long long row = static_cast<long long>(mt) * 128 + h * 64 + wq * 16 + (lane >> 2) + half * 8;
    if (row >= p.T) continue;
    const float rs = (chan && p.rowmask) ? (p.rowmask[row] ? 1.0f : 0.0f) : 1.0f;
#pragma unroll
    for (int j = 0; j < W / 8; ++j) {                      // fully unrolled: the accumulator stays in registers
      const int c = 8 * j + 2 * (lane & 3);
      if (c >= ncols) continue;
      const bool two = c + 1 < ncols;
      float v0 = acc[4 * j + 2 * half] + __ldg(bias + c), v1 = acc[4 * j + 2 * half + 1] + __ldg(bias + c + 1);
      if constexpr (gated) {
        // gate columns of the packed tile sit 128 columns (16 fragment steps) to the right of their values
        v0 *= apply_act(acc[4 * (j + PROJ_BN / 16) + 2 * half] + __ldg(bias + PROJ_BN / 2 + c), act);
        v1 *= apply_act(acc[4 * (j + PROJ_BN / 16) + 2 * half + 1] + __ldg(bias + PROJ_BN / 2 + c + 1), act);
      } else {
        v0 = apply_act(v0, act);
        v1 = apply_act(v1, act);
      }
      if constexpr (chan) { v0 *= rs; v1 *= rs; }
      const long long col = col0 + c;
      __nv_bfloat16* o = reinterpret_cast<__nv_bfloat16*>(sg.out);
      if constexpr (chan) {
        o[col * sg.ld + row] = __float2bfloat16(v0);
        if (two) o[(col + 1) * sg.ld + row] = __float2bfloat16(v1);
      } else {
        store_pair<false>(o, row * sg.ld + col, v0, v1, two, true);
      }
    }
  }
}

// tmB: 2-D map over Wcat (k = d contiguous, rows), box (64, 256), 128B swizzle
__global__ void __launch_bounds__(PROJ_THREADS, 1)
proj_tc_kernel(const __grid_constant__ CUtensorMap tmB, const __grid_constant__ ProjParams p) {
  using L = ProjSmem;
  extern __shared__ __align__(1024) uint8_t smem[];
  if ((smem_u32(smem) & 1023u) != 0) __trap();
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + L::BAR_OFF);
  uint64_t* empty_bar = full_bar + PROJ_STAGES;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, wg = warp >> 2;
  const int num_kb = p.d / GEMM_BK;

  if (threadIdx.x == 0) {
    prefetch_tmap(&tmB);
    for (int s = 0; s < PROJ_STAGES; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 2);     // one arrive per MMA warpgroup
    }
    fence_barrier_init();
  }
  __syncthreads();
  pdl_launch_dependents();
  pdl_wait();

  if (wg == 0) {
    // ================================ weight-tile TMA producer ================================
    regs_dealloc<40>();
    if (threadIdx.x == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int mt = blockIdx.x; mt < p.m_tiles; mt += gridDim.x)
        for (int nt = 0; nt < p.n_tiles_total; ++nt)
          for (int kb = 0; kb < num_kb; ++kb) {
            mbar_wait(&empty_bar[stage], phase ^ 1);
            mbar_arrive_expect_tx(&full_bar[stage], L::B_STAGE);
            tma_load_2d(smem + L::B_OFF + stage * L::B_STAGE, &tmB, &full_bar[stage], kb * GEMM_BK, nt * PROJ_BN);
            if (++stage == PROJ_STAGES) { stage = 0; phase ^= 1; }
          }
    }
    return;
  }

  regs_alloc<232>();
  const int h = wg - 1, wq = warp & 3;
  const int cw = warp - 4;                  // 0..7: LayerNorm row owner
  int stage = 0;
  uint32_t phase = 0;
  float acc[PROJ_BN / 2];
  for (int mt = blockIdx.x; mt < p.m_tiles; mt += gridDim.x) {
    // ---------------- LayerNorm of the item's 128 rows -> bf16 A tile (128B swizzle, 16 KB per 64 channels) ----------------
#pragma unroll 4                            // four rows' loads in flight per warp
    for (int r = cw; r < 128; r += 8) {
      const long long row = static_cast<long long>(mt) * 128 + r;
      const bool live = lane * 8 < p.d && row < p.T;
      float v[8];
      float s = 0.f;
      if (live) {
        const float4* src = reinterpret_cast<const float4*>(p.x + row * p.d + lane * 8);
        const float4 a = __ldg(src), b = __ldg(src + 1);
        v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
#pragma unroll
        for (int i = 0; i < 8; ++i) s += v[i];
      } else {
#pragma unroll
        for (int i = 0; i < 8; ++i) v[i] = 0.f;
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
      const float mean = s * p.inv_d;
      float q = 0.f;
      if (live) {
#pragma unroll
        for (int i = 0; i < 8; ++i) { v[i] -= mean; q += v[i] * v[i]; }
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o);
      const float rstd = rsqrtf(q * p.inv_d + p.eps);
      if (lane * 8 < p.d) {
        const uint4 pk = live ? make_uint4(pack_bf16x2(v[0] * rstd, v[1] * rstd), pack_bf16x2(v[2] * rstd, v[3] * rstd),
                                           pack_bf16x2(v[4] * rstd, v[5] * rstd), pack_bf16x2(v[6] * rstd, v[7] * rstd))
                              : make_uint4(0u, 0u, 0u, 0u);
        *reinterpret_cast<uint4*>(smem + (lane >> 3) * 16384 + swz128_off(r, lane & 7)) = pk;
      }
    }
    fence_proxy_async_smem();               // generic-proxy stores of the A tile -> wgmma (async proxy) reads
    proj_bar_sync();

    for (int nt = 0; nt < p.n_tiles_total; ++nt) {
      int prev = -1;
      for (int kb = 0; kb < num_kb; ++kb) {
        mbar_wait(&full_bar[stage], phase);
        const uint32_t sa = smem_u32(smem) + kb * 16384 + h * 8192;
        const uint32_t sb = smem_u32(smem + L::B_OFF + stage * L::B_STAGE);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < GEMM_BK / 16; ++k)
          wgmma_m64n256k16_ss<0, 0>(acc, wgmma_desc(sa + k * 32, 16, 1024, SWZ_128), wgmma_desc(sb + k * 32, 16, 1024, SWZ_128),
                                    (kb | k) != 0 ? 1u : 0u);
        wgmma_commit();
        wgmma_wait<1>();
        if (prev >= 0 && lane == 0 && wq == 0) mbar_arrive(&empty_bar[prev]);
        prev = stage;
        if (++stage == PROJ_STAGES) { stage = 0; phase ^= 1; }
      }
      wgmma_wait<0>();
      reg_fence(acc);
      if (lane == 0 && wq == 0) mbar_arrive(&empty_bar[prev]);

      // ------------------------------- epilogue of weight tile nt -------------------------------
      int si = 0;
      while (si + 1 < p.nseg && nt >= p.seg[si + 1].tile0) ++si;
      const ProjSeg& sg = p.seg[si];
      switch (sg.kind) {
        case EK_STORE_TOK: proj_epilogue<EK_STORE_TOK>(acc, p, sg, mt, nt, h, wq, lane); break;
        case EK_STORE_TOK_SIG: proj_epilogue<EK_STORE_TOK_SIG>(acc, p, sg, mt, nt, h, wq, lane); break;
        case EK_STORE_CH: proj_epilogue<EK_STORE_CH>(acc, p, sg, mt, nt, h, wq, lane); break;
        case EK_GATED_TOK_GELU: proj_epilogue<EK_GATED_TOK_GELU>(acc, p, sg, mt, nt, h, wq, lane); break;
        default: proj_epilogue<EK_GATED_CH_SIG>(acc, p, sg, mt, nt, h, wq, lane); break;
      }
    }
    proj_bar_sync();                         // both warpgroups are done with the A tile before it is rebuilt
  }
}

}  // namespace af2
