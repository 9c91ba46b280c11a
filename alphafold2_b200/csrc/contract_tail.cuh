// Tail of the triangle multiplications and the outer mean in one kernel (sm_90a):
//
//   x[t] += tail(O)[t] · W_outᵀ + b_out          (x fp32 token-major, updated in place)
//
// with O the fp32 channel-major contraction output [c][t] and
//   CT_GATE_PROJECT  tail = bf16(((O - mean) rstd γ + β) · gate),  gate = bf16(sigmoid(xn · W_ogateᵀ + b_ogate)) computed here
//   CT_GATE_LOAD     the same tail with the bf16 gate read from memory
//   CT_SCALE         tail = bf16(O · scale[t])  (or O · scale_const)
//
// It replaces the out-gate GEMM (EK_STORE_TOK_SIG), chan_to_token_tma_kernel and the to_out GEMM (EK_RESID_F32): the gate
// and the token-major tail never go through HBM.  Per token at D = 256 that is 4 D (O) + 2 D (xn) + 8 D (x) bytes instead
// of 2 D + 2 D, 4 D + 2 D + 2 D and 2 D + 8 D over three launches.
//
// Warp roles (384 threads), one persistent CTA per SM, 64-token tiles:
//   warp 0          TMA: per tile the O tile [D][64] fp32 and (gated variants) the xn or gate tile [64][D] bf16, 128B
//                   swizzle, into the A slot; L2 prefetch of the tile's residual rows
//   warp 1          TMA: W_ogate then W_out in k-chunks [D rows][64 k] through a ring both MMA warpgroups read
//   warpgroups 1, 2 output columns [0, D/2) / [D/2, D) of both GEMMs (m64n(D/2) accumulators) and, all 256 threads
//                   together, the LayerNorm over channels between them.  The A slot holds xn, then the gate (written over
//                   xn once both warpgroups' GEMM1 has retired), then the tail (written over the gate in place), in the
//                   128B-swizzled layout wgmma reads.  The residual values are loaded into registers before GEMM2, so
//                   their latency runs under it.
//
// Results equal the unfused sequence bit for bit: every projected element is one fp32 accumulator over the k16 steps
// 0 .. D/16 - 1 in order (as gemm_tc_kernel runs them), the gate is rounded to bf16 after + b and sigmoidf_fast, the
// LayerNorm statistics and the tail expression are chan_to_token_tma_kernel's (32-channel slices summed sequentially, slice
// partials added in slice order), and the output is (acc + b_out) + x.
#pragma once
#include "common.cuh"

namespace af2 {

enum CtailVariant : int { CT_GATE_PROJECT = 0, CT_GATE_LOAD = 1, CT_SCALE = 2 };

constexpr int CT_TOK = 64;          // tokens per tile (one wgmma M)
constexpr int CT_THREADS = 384;

template <int D>
struct CtailSmem {
  static_assert(D == 128 || D == 256, "contract tail: D must be 128 or 256");
  static constexpr int SL = D / 32;                         // 32-channel slices
  static constexpr int O_BYTES = D * CT_TOK * 4;            // fp32 [D][64]
  static constexpr int A_BYTES = CT_TOK * D * 2;            // bf16 D / 64 boxes [64 tok][64 ch], 128B swizzle
  static constexpr int SLOT = D * 64 * 2;                   // weight chunk [D rows][64 k]
  static constexpr int O_OFF = 0;
  static constexpr int A_OFF = O_OFF + O_BYTES;
  static constexpr int RING_OFF = A_OFF + A_BYTES;
  static constexpr int PAR_BYTES = 4 * D * 4 + 2 * SL * CT_TOK * 4;   // gamma, beta, b_ogate, b_out; moment partials
  static constexpr int FREE = 232448 - RING_OFF - PAR_BYTES - 256;
  static constexpr int SLOTS = FREE / SLOT < 8 ? FREE / SLOT : 8;
  static constexpr int PAR_OFF = RING_OFF + SLOTS * SLOT;
  static constexpr int BAR_OFF = PAR_OFF + PAR_BYTES;
  static constexpr int TOTAL = BAR_OFF + 256;
  static_assert(SLOTS >= 2, "the weight ring needs two slots");
  static_assert(2 * SLOTS + 4 <= 32, "mbarriers exceed their 256-byte region");
  static_assert(TOTAL <= 232448, "exceeds the 227 KB of shared memory a CTA can use");
};

struct CtailParams {
  float* x;                 // [T][D] fp32 residual stream, updated in place
  const float* b_ogate;     // [D] or nullptr
  const float* b_out;       // [D] or nullptr
  const float* gamma;       // [D] (gated variants)
  const float* beta;
  const float* scale;       // [T] or nullptr (CT_SCALE)
  float scale_const;
  float eps;
  int T;
};

// tmO: fp32 2-D (token [T], channel [D]), box (64, D), no swizzle.  tmG: bf16 2-D (channel [D], token [T]), box (64, 64),
// SW128.  tmWg / tmWo: bf16 2-D (k [D], row [D]), box (64, D), SW128.
template <int D, int V>
__global__ void __launch_bounds__(CT_THREADS, 1)
contract_tail_kernel(const __grid_constant__ CUtensorMap tmO, const __grid_constant__ CUtensorMap tmG,
                     const __grid_constant__ CUtensorMap tmWg, const __grid_constant__ CUtensorMap tmWo,
                     const __grid_constant__ CtailParams p) {
  using L = CtailSmem<D>;
  constexpr int SL = L::SL, NS = L::SLOTS, KC = D / 64;
  constexpr bool PROJECT = V == CT_GATE_PROJECT, GATED = V != CT_SCALE;
  extern __shared__ __align__(1024) uint8_t smem[];
  if ((smem_u32(smem) & 1023u) != 0) __trap();
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + L::BAR_OFF);
  uint64_t* empty_bar = full_bar + NS;       // count 2: both MMA warpgroups read every chunk
  uint64_t* ofull = empty_bar + NS;
  uint64_t* oempty = ofull + 1;              // count 1: the LayerNorm of the tile has read O
  uint64_t* afull = oempty + 1;
  uint64_t* aempty = afull + 1;              // count 2: both warpgroups' GEMM2 has retired
  float* par = reinterpret_cast<float*>(smem + L::PAR_OFF);
  float* s_gamma = par;
  float* s_beta = par + D;
  float* s_bog = par + 2 * D;
  float* s_bout = par + 3 * D;
  float* p1 = par + 4 * D;                   // [SL][64] slice sums
  float* p2 = p1 + SL * CT_TOK;              // [SL][64] centred slice sums of squares
  uint8_t* aslot = smem + L::A_OFF;
  const float* os = reinterpret_cast<const float*>(smem + L::O_OFF);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, wg = warp >> 2;
  const int tiles = (p.T + CT_TOK - 1) / CT_TOK;

  if (threadIdx.x == 0) {
    prefetch_tmap(&tmO);
    if (GATED) prefetch_tmap(&tmG);
    if (PROJECT) prefetch_tmap(&tmWg);
    prefetch_tmap(&tmWo);
    for (int s = 0; s < NS; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 2);
    }
    mbar_init(ofull, 1);
    mbar_init(oempty, 1);
    mbar_init(afull, 1);
    mbar_init(aempty, 2);
    fence_barrier_init();
  }
  __syncthreads();
  pdl_launch_dependents();
  pdl_wait();

  if (wg == 0) {
    regs_dealloc<40>();
    if (warp == 0 && lane == 0) {
      // ============================ tile producer ============================
      int it = 0;
      for (int tile = blockIdx.x; tile < tiles; tile += gridDim.x, ++it) {
        const int t0 = tile * CT_TOK;
        const uint32_t ph = static_cast<uint32_t>(it & 1);
        mbar_wait(oempty, ph ^ 1);
        mbar_arrive_expect_tx(ofull, L::O_BYTES);
        tma_load_2d(smem + L::O_OFF, &tmO, ofull, t0, 0);
        if (GATED) {
          mbar_wait(aempty, ph ^ 1);
          mbar_arrive_expect_tx(afull, L::A_BYTES);
#pragma unroll
          for (int q = 0; q < KC; ++q) tma_load_2d(aslot + q * 8192, &tmG, afull, q * 64, t0);
        }
        // the residual rows this tile's epilogue reads, into L2 while the tile's GEMMs run.  Prefetching the next tile's
        // O and xn / gate as well measured slower (118 against 126 us per C2 call without it, DESIGN §6).
        bulk_prefetch_l2(p.x + static_cast<long long>(t0) * D, static_cast<uint32_t>(min(CT_TOK, p.T - t0) * D * 4));
      }
    } else if (warp == 1 && lane == 0) {
      // ============================ weight producer ============================
      int slot = 0;
      uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
#pragma unroll 1
        for (int g = PROJECT ? 0 : 1; g < 2; ++g) {
          for (int kc = 0; kc < KC; ++kc) {
            mbar_wait(&empty_bar[slot], phase ^ 1);
            mbar_arrive_expect_tx(&full_bar[slot], L::SLOT);
            tma_load_2d(smem + L::RING_OFF + slot * L::SLOT, g == 0 ? &tmWg : &tmWo, &full_bar[slot], kc * 64, 0);
            if (++slot == NS) { slot = 0; phase ^= 1; }
          }
        }
      }
    }
    return;
  }

  // ============== MMA warpgroup hh: output columns n0 .. n0 + D/2 - 1; with the other, the LayerNorm ==============
  regs_alloc<232>();
  const int hh = wg - 1;
  const int wq = warp & 3;
  const int tid = threadIdx.x - 128;                 // 0 .. 255 over both MMA warpgroups
  const bool leader = wq == 0 && lane == 0;
  const int n0 = hh * (D / 2);
  const int r_lo = wq * 16 + (lane >> 2);            // tile-local rows r_lo, r_lo + 8 of this thread's fragment
  const int q2 = 2 * (lane & 3);
  for (int i = tid; i < D; i += 256) {
    if (GATED) { s_gamma[i] = p.gamma[i]; s_beta[i] = p.beta[i]; }
    if (PROJECT) s_bog[i] = p.b_ogate ? p.b_ogate[i] : 0.f;
    s_bout[i] = p.b_out ? p.b_out[i] : 0.f;
  }
  const uint32_t ring = smem_u32(smem + L::RING_OFF), abase = smem_u32(aslot);
  int slot = 0;
  uint32_t phase = 0;
  float acc[D / 4];

  // acc = A slot · (rows n0 .. n0 + D/2 of the next D / 64 weight chunks)ᵀ, k16 steps in order
  auto gemm = [&]() {
    int prev = -1;
#pragma unroll 1
    for (int kc = 0; kc < KC; ++kc) {
      mbar_wait(&full_bar[slot], phase);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const uint64_t adesc = wgmma_desc(abase + kc * 8192 + k * 32, 16, 1024, SWZ_128);
        const uint64_t bdesc = wgmma_desc(ring + slot * L::SLOT + n0 * 128 + k * 32, 16, 1024, SWZ_128);
        const uint32_t scale_d = (kc | k) != 0 ? 1u : 0u;
        if constexpr (D == 256) wgmma_m64n128k16_ss<0, 0>(acc, adesc, bdesc, scale_d);
        else wgmma_m64n64k16_ss<0, 0>(acc, adesc, bdesc, scale_d);
      }
      wgmma_commit();
      wgmma_wait<1>();
      if (prev >= 0 && leader) mbar_arrive(&empty_bar[prev]);
      prev = slot;
      if (++slot == NS) { slot = 0; phase ^= 1; }
    }
    wgmma_wait<0>();
    reg_fence(acc);
    if (leader) mbar_arrive(&empty_bar[prev]);
  };

  const int tok = tid & (CT_TOK - 1);                // LayerNorm: thread = (token, slices sg * SPT .. sg * SPT + SPT - 1)
  const int sg = tid >> 6;
  constexpr int SPT = SL / 4;
  int it = 0;
  for (int tile = blockIdx.x; tile < tiles; tile += gridDim.x, ++it) {
    const uint32_t ph = static_cast<uint32_t>(it & 1);
    const int t0 = tile * CT_TOK;
    if (PROJECT) {
      // ---- GEMM1: gate = bf16(sigmoid(xn · W_ogateᵀ + b)) (the EK_STORE_TOK_SIG epilogue), over xn in the slot ----
      mbar_wait(afull, ph);
      gemm();
      named_bar_sync(1, 256);                        // both warpgroups have read xn
#pragma unroll
      for (int j = 0; j < D / 16; ++j) {
        const int c = n0 + 8 * j + q2;
        const float b0 = s_bog[c], b1 = s_bog[c + 1];
#pragma unroll
        for (int half = 0; half < 2; ++half) {
          const int r = r_lo + half * 8;
          float v0 = acc[4 * j + 2 * half], v1 = acc[4 * j + 2 * half + 1];
          if (p.b_ogate) { v0 += b0; v1 += b1; }
          v0 = sigmoidf_fast(v0);
          v1 = sigmoidf_fast(v1);
          *reinterpret_cast<uint32_t*>(aslot + (c >> 6) * 8192 + swz128_off(r, (c & 63) >> 3) + (c & 7) * 2) = pack_bf16x2(v0, v1);
        }
      }
    } else if (GATED) {
      mbar_wait(afull, ph);
    } else {
      named_bar_sync(1, 256);                        // both warpgroups' previous GEMM2 has read the slot
    }

    // ---- the tail, written over the slot in place (chan_to_token_tma_kernel's arithmetic) ----
    mbar_wait(ofull, ph);
    if constexpr (GATED) {
#pragma unroll
      for (int u = 0; u < SPT; ++u) {
        const int sl = sg * SPT + u;
        float s1 = 0.f;
#pragma unroll
        for (int k = 0; k < 32; ++k) s1 += os[(sl * 32 + k) * CT_TOK + tok];
        p1[sl * CT_TOK + tok] = s1;
      }
      named_bar_sync(1, 256);
      float tot = 0.f;
#pragma unroll
      for (int k = 0; k < SL; ++k) tot += p1[k * CT_TOK + tok];
      const float mean = tot * (1.0f / D);
#pragma unroll
      for (int u = 0; u < SPT; ++u) {
        const int sl = sg * SPT + u;
        float s2 = 0.f;
#pragma unroll
        for (int k = 0; k < 32; ++k) {
          const float a = os[(sl * 32 + k) * CT_TOK + tok] - mean;
          s2 += a * a;
        }
        p2[sl * CT_TOK + tok] = s2;
      }
      named_bar_sync(1, 256);                        // also: every gate value of the tile is in the slot
      float var = 0.f;
#pragma unroll
      for (int k = 0; k < SL; ++k) var += p2[k * CT_TOK + tok];
      const float rstd = rsqrtf(var * (1.0f / D) + p.eps);
#pragma unroll
      for (int u = 0; u < SPT; ++u) {
        const int sl = sg * SPT + u, c0 = sl * 32;
        uint8_t* gs = aslot + (sl >> 1) * 8192 + tok * 128;
        const uint32_t ch0 = static_cast<uint32_t>((sl & 1) * 4), sw = static_cast<uint32_t>(tok & 7);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          uint4* gp = reinterpret_cast<uint4*>(gs + (((ch0 + j) ^ sw) << 4));
          const uint4 gq = *gp;
          const uint32_t gw[4] = {gq.x, gq.y, gq.z, gq.w};
          float o[8];
#pragma unroll
          for (int k = 0; k < 8; ++k) {
            const int c = c0 + j * 8 + k;
            const float g = (k & 1) ? bf16hi_to_f32(gw[k >> 1]) : bf16lo_to_f32(gw[k >> 1]);
            o[k] = ((os[c * CT_TOK + tok] - mean) * rstd * s_gamma[c] + s_beta[c]) * g;
          }
          *gp = make_uint4(pack_bf16x2(o[0], o[1]), pack_bf16x2(o[2], o[3]), pack_bf16x2(o[4], o[5]), pack_bf16x2(o[6], o[7]));
        }
      }
    } else {
      const int token = t0 + tok;
      const float sc = p.scale ? ((token < p.T) ? __ldg(p.scale + token) : 0.f) : p.scale_const;
#pragma unroll
      for (int u = 0; u < SPT; ++u) {
        const int sl = sg * SPT + u, c0 = sl * 32;
        uint8_t* gs = aslot + (sl >> 1) * 8192 + tok * 128;
        const uint32_t ch0 = static_cast<uint32_t>((sl & 1) * 4), sw = static_cast<uint32_t>(tok & 7);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          float xv[8];
#pragma unroll
          for (int k = 0; k < 8; ++k) xv[k] = os[(c0 + j * 8 + k) * CT_TOK + tok];
          *reinterpret_cast<uint4*>(gs + (((ch0 + j) ^ sw) << 4)) =
              make_uint4(pack_bf16x2(xv[0] * sc, xv[1] * sc), pack_bf16x2(xv[2] * sc, xv[3] * sc),
                         pack_bf16x2(xv[4] * sc, xv[5] * sc), pack_bf16x2(xv[6] * sc, xv[7] * sc));
        }
      }
    }
    fence_proxy_async_smem();                        // generic writes of the slot -> wgmma reads
    named_bar_sync(1, 256);
    if (tid == 0) mbar_arrive(oempty);

    // ---- GEMM2: x = (tail · W_outᵀ + b_out) + x (the EK_RESID_F32 order); the residual loads run under it ----
    float2 res[2][D / 16];
#pragma unroll
    for (int half = 0; half < 2; ++half) {
      const int row = t0 + r_lo + half * 8;
#pragma unroll
      for (int j = 0; j < D / 16; ++j)
        res[half][j] = row < p.T ? *reinterpret_cast<const float2*>(p.x + static_cast<long long>(row) * D + n0 + 8 * j + q2)
                                 : make_float2(0.f, 0.f);
    }
    gemm();
    if (GATED && leader) mbar_arrive(aempty);
#pragma unroll
    for (int half = 0; half < 2; ++half) {
      const int row = t0 + r_lo + half * 8;
      if (row < p.T) {
        float* xr = p.x + static_cast<long long>(row) * D;
#pragma unroll
        for (int j = 0; j < D / 16; ++j) {
          const int col = n0 + 8 * j + q2;
          float v0 = acc[4 * j + 2 * half], v1 = acc[4 * j + 2 * half + 1];
          if (p.b_out) { v0 += s_bout[col]; v1 += s_bout[col + 1]; }
          v0 += res[half][j].x;
          v1 += res[half][j].y;
          *reinterpret_cast<float2*>(xr + col) = make_float2(v0, v1);
        }
      }
    }
  }
}

}  // namespace af2
