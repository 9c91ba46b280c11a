// Axial self-attention with the q, k, v and gate projections inside the kernel: the LayerNorm output xn goes in, the gated
// attention output og comes out, and q|k|v and the gate never leave the SM.  Computes exactly what the two projection GEMMs
// (EK_STORE_TOK into q|k|v, EK_STORE_TOK_SIG into the gate) followed by attention_tc_kernel compute, bit for bit: every
// projected element is one fp32 accumulator over the k16 steps 0 .. d/16 - 1 in order (64-channel chunks, zero-filled past
// d, as the GEMM's k blocks), rounded to bf16 where the GEMM epilogue rounds it; the softmax, PV and epilogue code is the
// attention kernel's.
//
// Persistent: min(items, SMs) CTAs; CTA c computes the work items c, c + gridDim.x, ...  A work item is (folded batch
// element b', head h), numbered head fastest: the CTAs resident at one time read the same xn row from L2.
// Three warpgroups:
//   warpgroup 0, warp 0   TMA producer, running ahead across items through a ring of stages.  A stage is one 64-channel
//                         chunk of 128 xn tokens plus the same chunk of 2 DH weight rows: [W_k,h | W_v,h] while the item
//                         projects its keys, [W_q,h | W_g,h] while it projects its queries.  The weight rows are row windows
//                         of the packed w_qkv [3I, d] and w_gate [I, d]; no other packing is needed.
//   warpgroups 1, 2       64 of each 128 tokens each:
//     K|V phase   [K | V] = xn [W_k | W_v]^T     wgmma m64n(2 DH)k16 into fp32, rounded to bf16 and stored into the shared
//                                                K / V tiles of all kpad keys, laid out as attention_tc_kernel's K / V stages
//     query phase [q | g] = xn [W_q | W_g]^T     wgmma m64n(2 DH)k16; q rounded to bf16 stays in registers as the A fragment
//                                                of S = Q K^T, g = bf16(sigmoid(acc + b_gate)) as the epilogue's gate
//                 then S, bias, mask, online softmax, O += P V and O / l * gate as in attention_tc_kernel
// Both warpgroups release each stage (two arrivals); a named barrier separates an item's K / V stores from the reads of its
// query phase (after a generic -> async proxy fence), and the previous item's reads from the next item's stores.
// Keys and queries past n read zero xn rows (TMA fill), so pad keys are K = V = 0 exactly as the attention kernel's
// zero-filled K / V tiles; the key codes discard them.
// Head widths 32 and 64.  Shared memory holds the K / V of all kpad keys (4 DH bytes per key) and the stage ring
// (AttnProjSmem::stages_for): at DH 64 n <= 256 runs with 4 stages and 256 < n <= 384 with 3, at DH 32 n <= 896 with 4
// and 896 < n <= 1024 with 3 (attn_proj_max_n).
#pragma once
#include <float.h>
#include "common.cuh"

namespace af2 {

struct AttnProjParams {
  int n, heads, nbatch, d;
  int has_bias;
  const __nv_bfloat16* bias;  // [heads][n][npad] (log2 domain), or nullptr
  int npad;
  const uint8_t* mask;        // nullptr or bool mask; element (b', i) at mask[b'*mask_sb + i*mask_si]
  long long mask_sb, mask_si;
  const float* b_gate;        // [I] or nullptr
  __nv_bfloat16* out;         // [token, heads*DH]; token(b', i) = b'*tok_sb + i*tok_si
  long long tok_sb, tok_si;
  long long ld_out;
  int stages;                 // stage ring depth (AttnProjSmem::stages_for)
};

constexpr int APROJ_THREADS = 384;
constexpr int APROJ_CONSUMERS = 256;
constexpr int APROJ_TOK = 128;       // tokens per stage (64 per MMA warpgroup)
constexpr int APROJ_KB = 128;        // keys per S block

template <int DH>
struct AttnProjSmem {
  static_assert(DH == 32 || DH == 64, "attention_proj: DH must be 32 or 64");
  static constexpr int ROWB = DH * 2;                     // bytes per K / V row (one swizzle atom)
  static constexpr int XN_BYTES = APROJ_TOK * 128;        // 128 tokens x 64 channels
  static constexpr int W_BYTES = 2 * DH * 128;            // 2 DH weight rows x 64 channels
  static constexpr int STAGE_BYTES = XN_BYTES + W_BYTES;
  __host__ __device__ static constexpr int kpad(int n) { return (n + APROJ_KB - 1) / APROJ_KB * APROJ_KB; }
  __host__ __device__ static constexpr int kv_off(int stages) { return stages * STAGE_BYTES; }
  // the gate of each consumer thread's query fragment, bf16 pairs in a thread-private order ([pair][thread]): kept out of the
  // registers the softmax needs
  static constexpr int GATE_BYTES = APROJ_CONSUMERS * (DH / 4) * 4;
  static constexpr int Q_BYTES = 64 * ROWB;               // one warpgroup's 64 query rows, laid out as the K tile
  __host__ __device__ static constexpr int q_off(int n, int stages) { return kv_off(stages) + 2 * kpad(n) * ROWB; }
  __host__ __device__ static constexpr int gate_off(int n, int stages) { return q_off(n, stages) + 2 * Q_BYTES; }
  __host__ __device__ static constexpr int bar_off(int n, int stages) { return gate_off(n, stages) + GATE_BYTES; }
  __host__ __device__ static constexpr int code_off(int n, int stages) { return bar_off(n, stages) + 128; }
  __host__ __device__ static constexpr int bytes(int n, int stages) { return code_off(n, stages) + kpad(n); }
  static constexpr int MAX_SMEM = 232448;
  static constexpr int MIN_STAGES = 3, MAX_STAGES = 4;
  // the deepest ring that fits next to the K / V of n keys; 0 if not even MIN_STAGES fit
  static constexpr int stages_for(int n) {
    return bytes(n, MAX_STAGES) <= MAX_SMEM ? MAX_STAGES : (bytes(n, MIN_STAGES) <= MAX_SMEM ? MIN_STAGES : 0);
  }
};

// byte offset of (row, byte b) in a tile of ROWB-byte rows with the swizzle TMA / wgmma use for that row width (128B: 16-byte
// chunk c of row r at c ^ (r % 8); 64B: c ^ (r / 2 % 4)); the tile is aligned to its swizzle repeat
template <int ROWB>
__device__ __forceinline__ uint32_t swz_off(uint32_t row, uint32_t b) {
  constexpr uint32_t CMASK = ROWB == 128 ? 7u : 3u;
  const uint32_t off = row * ROWB + b;
  return off ^ (((off >> 7) & CMASK) << 4);
}

// xn [64 tokens of warpgroup wh] x [2 DH weight rows]^T over all of d into acc, consuming nkc stages from stage count g on:
// the GEMM's k order into one accumulator; `releaser` is the one thread of the warpgroup that hands stages back
template <int DH>
__device__ __forceinline__ void aproj_project(float (&acc)[DH], uint8_t* smem, uint64_t* full_bar, uint64_t* empty_bar, int& g,
                                              int S, int nkc, int wh, bool releaser) {
  using L = AttnProjSmem<DH>;
  int prev = -1;
  for (int c = 0; c < nkc; ++c, ++g) {
    const int s = g % S;
    mbar_wait(&full_bar[s], (g / S) & 1);
    const uint32_t sx = smem_u32(smem + s * L::STAGE_BYTES) + wh * 64 * 128;
    const uint32_t sw = smem_u32(smem + s * L::STAGE_BYTES + L::XN_BYTES);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const uint64_t adesc = wgmma_desc(sx + k * 32, 16, 1024, SWZ_128);
      const uint64_t bdesc = wgmma_desc(sw + k * 32, 16, 1024, SWZ_128);
      const uint32_t scale_d = (c | k) != 0 ? 1u : 0u;
      if constexpr (DH == 64) wgmma_m64n128k16_ss<0, 0>(acc, adesc, bdesc, scale_d);
      else wgmma_m64n64k16_ss<0, 0>(acc, adesc, bdesc, scale_d);
    }
    wgmma_commit();
    wgmma_wait<1>();   // keep one chunk in flight: the previous one has retired, so its stage goes back to the producer
    if (prev >= 0 && releaser) mbar_arrive(&empty_bar[prev]);
    prev = s;
  }
  wgmma_wait<0>();
  reg_fence(acc);
  if (releaser) mbar_arrive(&empty_bar[prev]);
}

__device__ __forceinline__ void st_shared_u32(uint32_t addr, uint32_t v) {
  asm volatile("st.shared.b32 [%0], %1;" ::"r"(addr), "r"(v) : "memory");
}

// tmX: 3-D map over xn, dims (c [d], i [n], b' [nbatch]), box (64, 128, 1), 128B swizzle.
// tmW / tmG: 2-D maps over w_qkv [3I, d] / w_gate [I, d], box (64, DH), 128B swizzle.
template <int DH>
__global__ void __launch_bounds__(APROJ_THREADS, 1)
attention_proj_kernel(const __grid_constant__ CUtensorMap tmX, const __grid_constant__ CUtensorMap tmW,
                      const __grid_constant__ CUtensorMap tmG, const __grid_constant__ AttnProjParams p) {
  using L = AttnProjSmem<DH>;
  constexpr uint32_t SWZ = DH == 64 ? SWZ_128 : SWZ_64;
  constexpr uint32_t ROWB = L::ROWB;
  constexpr uint32_t SBO = 8 * ROWB;
  constexpr int NACC = DH;                          // m64n(2 DH) accumulator floats per thread
  extern __shared__ __align__(1024) uint8_t smem[];
  if ((smem_u32(smem) & 1023u) != 0) __trap();
  const int n = p.n, S = p.stages;
  const int nkb = (n + APROJ_KB - 1) / APROJ_KB;
  const int kpad = nkb * APROJ_KB;
  const int ntile = (n + APROJ_TOK - 1) / APROJ_TOK;   // 128-token tiles (= nkb)
  const int nkc = (p.d + 63) / 64;                      // 64-channel chunks of d
  const int I = p.heads * DH;
  const int items = p.heads * p.nbatch;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + L::bar_off(n, S));
  uint64_t* empty_bar = full_bar + S;
  uint8_t* kcode = smem + L::code_off(n, S);
  uint32_t* gsm = reinterpret_cast<uint32_t*>(smem + L::gate_off(n, S));
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, wg = warp >> 2;

  if (threadIdx.x == 0) {
    prefetch_tmap(&tmX);
    prefetch_tmap(&tmW);
    prefetch_tmap(&tmG);
    for (int s = 0; s < S; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 2);   // one arrive per MMA warpgroup
    }
    fence_barrier_init();
  }
  __syncthreads();
  pdl_launch_dependents();
  pdl_wait();

  if (wg == 0) {
    // ================================ producer ================================
    regs_dealloc<40>();
    if (warp == 0 && lane == 0) {
      int g = 0;   // stages issued by this CTA so far: ring slot and phase
      for (int item = blockIdx.x; item < items; item += gridDim.x) {
        const int h = item % p.heads, b = item / p.heads;
        for (int ph = 0; ph < 2; ++ph) {   // 0: K|V rows of w_qkv; 1: q rows of w_qkv and gate rows of w_gate
          const int r0 = ph == 0 ? I + h * DH : h * DH;
          const int r1 = ph == 0 ? 2 * I + h * DH : h * DH;
          const CUtensorMap* m1 = ph == 0 ? &tmW : &tmG;
          for (int t = 0; t < ntile; ++t) {
            for (int c = 0; c < nkc; ++c, ++g) {
              const int s = g % S;
              mbar_wait(&empty_bar[s], ((g / S) & 1) ^ 1);
              uint8_t* st = smem + s * L::STAGE_BYTES;
              mbar_arrive_expect_tx(&full_bar[s], L::STAGE_BYTES);
              tma_load_3d(st, &tmX, &full_bar[s], c * 64, t * APROJ_TOK, b);
              tma_load_2d(st + L::XN_BYTES, &tmW, &full_bar[s], c * 64, r0);
              tma_load_2d(st + L::XN_BYTES + DH * 128, m1, &full_bar[s], c * 64, r1);
            }
          }
        }
      }
    }
    return;
  }

  // ========================= MMA warpgroups: 64 of each 128 tokens each =========================
  regs_alloc<232>();
  const int wh = wg - 1, wq = warp & 3;
  const int tid = threadIdx.x - 128;
  uint32_t* gw = gsm + tid;   // gate pair (i, hf) of this thread at gw[(2 i + hf) * APROJ_CONSUMERS]
  const uint32_t sq = smem_u32(smem + L::q_off(n, S) + wh * L::Q_BYTES);
  const uint32_t sk = smem_u32(smem + L::kv_off(S)), sv = sk + kpad * ROWB;
  int g = 0;   // stages consumed by this CTA so far

  for (int item = blockIdx.x; item < items; item += gridDim.x) {
    const int h = item % p.heads, b = item / p.heads;
    named_bar_sync(1, APROJ_CONSUMERS);   // both warpgroups are done reading the previous item's K / V and key codes
    // key codes of the folded row: 0 padding (k >= n), 1 masked, 2 valid
    {
      const uint8_t* mrow = p.mask ? p.mask + static_cast<long long>(b) * p.mask_sb : nullptr;
      for (int k = tid; k < kpad; k += APROJ_CONSUMERS)
        kcode[k] = k >= n ? 0 : ((mrow && !mrow[static_cast<long long>(k) * p.mask_si]) ? 1 : 2);
    }

    // phase 0 (K|V) then phase 1 (queries), one projection call site: both accumulators share the same registers
    for (int pt = 0; pt < 2 * ntile; ++pt) {
      const int t = pt < ntile ? pt : pt - ntile;
      if (pt == ntile) {
        fence_proxy_async_smem();              // the K / V stores are read by wgmma (async proxy)
        named_bar_sync(1, APROJ_CONSUMERS);    // and by the other warpgroup's queries too
      }
      {
        float acc[NACC];
        aproj_project<DH>(acc, smem, full_bar, empty_bar, g, S, nkc, wh, lane == 0 && wq == 0);
        if (pt < ntile) {
          // ------------------------------- K|V: bf16 into the resident K / V tiles -------------------------------
#pragma unroll
          for (int hf = 0; hf < 2; ++hf) {
            const uint32_t key = t * APROJ_TOK + wh * 64 + wq * 16 + (lane >> 2) + 8 * hf;
#pragma unroll
            for (int j = 0; j < NACC / 4; ++j) {
              // accumulator columns 8 j + 2 (lane % 4) + {0, 1}: K for j < DH / 8, V after
              const uint32_t col = (8 * j + 2 * (lane & 3)) % DH;
              st_shared_u32((j < DH / 8 ? sk : sv) + swz_off<ROWB>(key, col * 2), pack_bf16x2(acc[4 * j + 2 * hf], acc[4 * j + 2 * hf + 1]));
            }
          }
          continue;
        }
        // ------------------------------- queries: bf16 q tile, bf16 gate -------------------------------
        named_bar_sync(2 + wh, 128);   // the warpgroup's previous S = Q K^T has read its Q tile
#pragma unroll
        for (int hf = 0; hf < 2; ++hf) {
          const uint32_t r = wq * 16 + (lane >> 2) + 8 * hf;
#pragma unroll
          for (int i = 0; i < DH / 8; ++i)
            st_shared_u32(sq + swz_off<ROWB>(r, (8 * i + 2 * (lane & 3)) * 2), pack_bf16x2(acc[4 * i + 2 * hf], acc[4 * i + 2 * hf + 1]));
        }
#pragma unroll
        for (int i = 0; i < DH / 8; ++i) {
          const int e = 8 * i + 2 * (lane & 3);
          float b0 = 0.f, b1 = 0.f;
          if (p.b_gate) { b0 = __ldg(p.b_gate + h * DH + e); b1 = __ldg(p.b_gate + h * DH + e + 1); }
#pragma unroll
          for (int hf = 0; hf < 2; ++hf) {
            float g0 = acc[4 * (DH / 8 + i) + 2 * hf], g1 = acc[4 * (DH / 8 + i) + 2 * hf + 1];
            if (p.b_gate) { g0 += b0; g1 += b1; }
            gw[(2 * i + hf) * APROJ_CONSUMERS] = pack_bf16x2(sigmoidf_fast(g0), sigmoidf_fast(g1));
          }
        }
      }
      fence_proxy_async_smem();        // the Q stores are read by wgmma
      named_bar_sync(2 + wh, 128);
      int rows[2];
      bool qvalid[2];
      const __nv_bfloat16* brow[2];
#pragma unroll
      for (int hf = 0; hf < 2; ++hf) {
        rows[hf] = t * APROJ_TOK + wh * 64 + wq * 16 + (lane >> 2) + 8 * hf;
        qvalid[hf] = kcode[rows[hf]] != 1;   // rows < kpad; pad rows (code 0) count as valid queries
        // pad rows (>= n) read the bias of row n - 1: their results are never stored and never mix with other rows
        brow[hf] = p.has_bias ? p.bias + (static_cast<long long>(h) * n + min(rows[hf], n - 1)) * p.npad : nullptr;
      }
      float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
      float o[DH / 2];
#pragma unroll
      for (int i = 0; i < DH / 2; ++i) o[i] = 0.f;
      float s[APROJ_KB / 2];

      for (int kb = 0; kb < nkb; ++kb) {
        const uint32_t skb = sk + kb * APROJ_KB * ROWB;
        const uint32_t svb = sv + kb * APROJ_KB * ROWB;
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < DH / 16; ++k)
          wgmma_m64n128k16_ss<0, 0>(s, wgmma_desc(sq + k * 32, 16, SBO, SWZ), wgmma_desc(skb + k * 32, 16, SBO, SWZ),
                                    k != 0 ? 1u : 0u);
        wgmma_commit();
        wgmma_wait<0>();
        reg_fence(s);

        uint32_t bw[APROJ_KB / 8][2] = {};
        if (p.has_bias) {
#pragma unroll
          for (int j = 0; j < APROJ_KB / 8; ++j) {
            const int key = min(kb * APROJ_KB + 8 * j + 2 * (lane & 3), p.npad - 2);
#pragma unroll
            for (int hf = 0; hf < 2; ++hf) bw[j][hf] = __ldg(reinterpret_cast<const unsigned int*>(brow[hf] + key));
          }
        }

        float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
        for (int j = 0; j < APROJ_KB / 8; ++j) {
          const int key = kb * APROJ_KB + 8 * j + 2 * (lane & 3);
          const uint32_t c0 = kcode[key], c1 = kcode[key + 1];
#pragma unroll
          for (int hf = 0; hf < 2; ++hf) {
            const float b0 = bf16lo_to_f32(bw[j][hf]), b1 = bf16hi_to_f32(bw[j][hf]);
            float& v0 = s[4 * j + 2 * hf];
            float& v1 = s[4 * j + 2 * hf + 1];
            const float t0 = v0 + b0, t1 = v1 + b1;
            const float u0 = (c0 == 1 || !qvalid[hf]) ? -FLT_MAX : t0;
            const float u1 = (c1 == 1 || !qvalid[hf]) ? -FLT_MAX : t1;
            v0 = c0 == 0 ? -INFINITY : u0;
            v1 = c1 == 0 ? -INFINITY : u1;
            mx[hf] = fmaxf(mx[hf], fmaxf(v0, v1));
          }
        }
        float alpha[2];
#pragma unroll
        for (int hf = 0; hf < 2; ++hf) {
          mx[hf] = fmaxf(mx[hf], __shfl_xor_sync(0xffffffffu, mx[hf], 1));
          mx[hf] = fmaxf(mx[hf], __shfl_xor_sync(0xffffffffu, mx[hf], 2));
          const float m_new = fmaxf(m_run[hf], mx[hf]);
          alpha[hf] = fast_exp2(m_run[hf] - m_new);
          m_run[hf] = m_new;
          l_run[hf] *= alpha[hf];
        }
        uint32_t pa[APROJ_KB / 16][4];
#pragma unroll
        for (int j = 0; j < APROJ_KB / 8; ++j) {
#pragma unroll
          for (int hf = 0; hf < 2; ++hf) {
            const float e0 = fast_exp2(s[4 * j + 2 * hf] - m_run[hf]);
            const float e1 = fast_exp2(s[4 * j + 2 * hf + 1] - m_run[hf]);
            l_run[hf] += e0 + e1;
            pa[j >> 1][(j & 1) * 2 + hf] = pack_bf16x2(e0, e1);
          }
        }
#pragma unroll
        for (int i = 0; i < DH / 8; ++i) {
          o[4 * i] *= alpha[0]; o[4 * i + 1] *= alpha[0];
          o[4 * i + 2] *= alpha[1]; o[4 * i + 3] *= alpha[1];
        }
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < APROJ_KB / 16; ++kk) {
          const uint64_t vdesc = wgmma_desc(svb + kk * 16 * ROWB, 8192, SBO, SWZ);
          if constexpr (DH == 64) wgmma_m64n64k16_rs<1>(o, pa[kk], vdesc, 1u);
          else wgmma_m64n32k16_rs<1>(o, pa[kk], vdesc, 1u);
        }
        wgmma_commit();
        wgmma_wait<0>();
        reg_fence(o);
      }

      // ------------------------------- epilogue: O / l * gate -> bf16 -------------------------------
#pragma unroll
      for (int hf = 0; hf < 2; ++hf) {
        l_run[hf] += __shfl_xor_sync(0xffffffffu, l_run[hf], 1);
        l_run[hf] += __shfl_xor_sync(0xffffffffu, l_run[hf], 2);
        if (rows[hf] >= n) continue;
        const float inv = 1.0f / l_run[hf];
        const long long tok = static_cast<long long>(b) * p.tok_sb + static_cast<long long>(rows[hf]) * p.tok_si;
        __nv_bfloat16* out = p.out + tok * p.ld_out + h * DH;
#pragma unroll
        for (int i = 0; i < DH / 8; ++i) {
          const int e = 8 * i + 2 * (lane & 3);
          const uint32_t gv = gw[(2 * i + hf) * APROJ_CONSUMERS];
          *reinterpret_cast<uint32_t*>(out + e) =
              pack_bf16x2(o[4 * i + 2 * hf] * inv * bf16lo_to_f32(gv), o[4 * i + 2 * hf + 1] * inv * bf16hi_to_f32(gv));
        }
      }
    }
  }
}

}  // namespace af2
