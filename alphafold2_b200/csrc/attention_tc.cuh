// Axial self-attention with shared additive pair bias and the reference's two-sided mask, on sm_90a wgmma.
// Replaces Attention.forward (alphafold2.py:125-190) as driven by AxialAttention (alphafold2.py:219-255).
//
// One CTA per work item = (folded batch element b', head h, block of 128 queries); items are ordered so that the CTAs
// of one (h, b') pair are launched together and share its K / V tiles in L2.  Three warpgroups:
//   warpgroup 0     TMA producer: the Q tile once, then K / V tiles of 128 keys through an ATTN_STAGES-deep pipeline
//   warpgroups 1, 2 64 query rows each, flash-attention style with everything in registers:
//     S_j = Q K_j^T          wgmma m64n128k16, Q and K from shared memory (K-major)
//     softmax                + pair bias (bf16, read from global / L2 in the accumulator's fragment layout), key / query
//                            mask, online max / sum (the four lanes of a row reduce with two shuffles)
//     O  += P_j V_j          wgmma m64nDHk16 with A = P_j straight from registers (the S fragment of 16 keys IS the
//                            m64k16 A fragment), V consumed MN-major from its [key][dh] layout
//     epilogue               O / l * sigmoid-gate -> bf16 [token, h*DH + e]
// Logits are produced directly in the log2 domain: the host folds dim_head^-0.5 * log2(e) into to_q and
// log2(e) into edges_to_attn_bias, so the softmax is exp2(v - max) with no per-element scaling.
//
// Mask semantics (quirk Q1): logits where !(mask[q] & mask[k]) are REPLACED by -FLT_MAX.  For an unmasked
// query that gives probability exactly 0 on masked keys; for a masked query every logit is equal, i.e. a
// uniform distribution over all n keys (masked ones included).  Keys >= n (tile padding) never count.
#pragma once
#include <float.h>
#include "common.cuh"

namespace af2 {

struct AttnParams {
  int n;              // sequence length along the attended axis
  int heads;
  int nbatch;         // folded batch B'
  int has_bias;
  const __nv_bfloat16* bias;  // [heads][n][npad] (log2 domain), or nullptr
  int npad;                   // row pitch of the bias (n rounded up to 8; pad columns are zero)
  const uint8_t* mask;        // nullptr or bool mask; element (b', i) at mask[b'*mask_sb + i*mask_si]
  long long mask_sb, mask_si;
  const __nv_bfloat16* gate;  // sigmoid(gating) [token, heads*DH]; token(b', i) = b'*tok_sb + i*tok_si
  __nv_bfloat16* out;         // [token, heads*DH]
  long long tok_sb, tok_si;
  long long ld_gate, ld_out;
};

constexpr int ATTN_THREADS = 384;
constexpr int ATTN_STAGES = 3;
constexpr int ATTN_KB = 128;                        // keys per block

template <int DH>
struct AttnSmem {
  static constexpr int Q_BYTES = 128 * DH * 2;
  static constexpr int KV_BYTES = ATTN_KB * DH * 2;
  static constexpr int STAGE_BYTES = 2 * KV_BYTES;    // K | V
  static constexpr int STAGE_OFF = Q_BYTES;
  static constexpr int BAR_OFF = STAGE_OFF + ATTN_STAGES * STAGE_BYTES;
  static constexpr int KM_OFF = BAR_OFF + 128;        // key codes [nkb * 128]: 0 padding, 1 masked, 2 valid
  static constexpr int bytes(int n) { return KM_OFF + (n + ATTN_KB - 1) / ATTN_KB * ATTN_KB; }
};

// tmQ/tmK/tmV: 4-D maps over the projection buffer, dims (e [DH], i [n], h [heads], b' [nbatch]),
// box (DH, 128, 1, 1), swizzle = DH*2 bytes.  tmBias / tmG / tmO are not read (bias, gate and output go through the
// register fragments).
template <int DH>
__global__ void __launch_bounds__(ATTN_THREADS, 1)
attention_tc_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                    const __grid_constant__ CUtensorMap tmV, const __grid_constant__ CUtensorMap tmBias,
                    const __grid_constant__ CUtensorMap tmG, const __grid_constant__ CUtensorMap tmO,
                    const __grid_constant__ AttnParams p) {
  using L = AttnSmem<DH>;
  constexpr uint32_t SWZ = (DH == 64) ? SWZ_128 : SWZ_64;
  constexpr uint32_t ROWB = DH * 2;                 // bytes per Q/K/V row
  constexpr uint32_t SBO = 8 * ROWB;                // 8-row swizzle atom
  extern __shared__ __align__(1024) uint8_t smem[];
  if ((smem_u32(smem) & 1023u) != 0) __trap();
  uint64_t* q_bar = reinterpret_cast<uint64_t*>(smem + L::BAR_OFF);
  uint64_t* full_bar = q_bar + 1;
  uint64_t* empty_bar = full_bar + ATTN_STAGES;
  uint8_t* kcode = smem + L::KM_OFF;

  const int n = p.n;
  const int nqb = (n + 127) / 128;
  const int nkb = (n + ATTN_KB - 1) / ATTN_KB;
  const int qb = blockIdx.x % nqb;
  const int bb = (blockIdx.x / nqb) % p.nbatch;
  const int hh = blockIdx.x / (nqb * p.nbatch);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, wg = warp >> 2;

  if (threadIdx.x == 0) {
    prefetch_tmap(&tmQ);
    prefetch_tmap(&tmK);
    prefetch_tmap(&tmV);
    mbar_init(q_bar, 1);
    for (int s = 0; s < ATTN_STAGES; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 2);   // one arrive per softmax warpgroup
    }
    fence_barrier_init();
  }
  pdl_launch_dependents();
  pdl_wait();
  const uint8_t* mrow = p.mask ? p.mask + static_cast<long long>(bb) * p.mask_sb : nullptr;
  for (int k = threadIdx.x; k < nkb * ATTN_KB; k += ATTN_THREADS)
    kcode[k] = k >= n ? 0 : ((mrow && !mrow[static_cast<long long>(k) * p.mask_si]) ? 1 : 2);
  __syncthreads();

  if (wg == 0) {
    // ================================ TMA producer ================================
    regs_dealloc<40>();
    if (threadIdx.x == 0) {
      mbar_arrive_expect_tx(q_bar, L::Q_BYTES);
      tma_load_4d(smem, &tmQ, q_bar, 0, qb * 128, hh, bb);
      for (int kb = 0; kb < nkb; ++kb) {
        const int s = kb % ATTN_STAGES;
        mbar_wait(&empty_bar[s], ((kb / ATTN_STAGES) & 1) ^ 1);
        uint8_t* st = smem + L::STAGE_OFF + s * L::STAGE_BYTES;
        mbar_arrive_expect_tx(&full_bar[s], L::STAGE_BYTES);
        tma_load_4d(st, &tmK, &full_bar[s], 0, kb * ATTN_KB, hh, bb);
        tma_load_4d(st + L::KV_BYTES, &tmV, &full_bar[s], 0, kb * ATTN_KB, hh, bb);
      }
    }
    return;
  }

  // ========================= softmax warpgroups: 64 query rows each =========================
  regs_alloc<232>();
  const int h = wg - 1, wq = warp & 3;
  int rows[2];
  bool qvalid[2];
  const __nv_bfloat16* brow[2];
#pragma unroll
  for (int hf = 0; hf < 2; ++hf) {
    rows[hf] = qb * 128 + h * 64 + wq * 16 + (lane >> 2) + 8 * hf;
    const bool in = rows[hf] < n;
    qvalid[hf] = !(in && mrow && !mrow[static_cast<long long>(rows[hf]) * p.mask_si]);
    brow[hf] = (p.has_bias && in) ? p.bias + (static_cast<long long>(hh) * n + rows[hf]) * p.npad : nullptr;
  }
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
  float o[DH / 2];
#pragma unroll
  for (int i = 0; i < DH / 2; ++i) o[i] = 0.f;
  float s[ATTN_KB / 2];
  const uint32_t sq = smem_u32(smem) + h * 64 * ROWB;
  mbar_wait(q_bar, 0);

  for (int kb = 0; kb < nkb; ++kb) {
    const int st = kb % ATTN_STAGES;
    mbar_wait(&full_bar[st], (kb / ATTN_STAGES) & 1);
    const uint32_t sk = smem_u32(smem + L::STAGE_OFF + st * L::STAGE_BYTES);
    const uint32_t sv = sk + L::KV_BYTES;
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < DH / 16; ++k)
      wgmma_m64n128k16_ss<0, 0>(s, wgmma_desc(sq + k * 32, 16, SBO, SWZ), wgmma_desc(sk + k * 32, 16, SBO, SWZ), k != 0 ? 1u : 0u);
    wgmma_commit();
    wgmma_wait<0>();
    reg_fence(s);

    // logits -> probabilities (in place)
    float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int j = 0; j < ATTN_KB / 8; ++j) {
      const int key = kb * ATTN_KB + 8 * j + 2 * (lane & 3);
      const uint32_t c0 = kcode[key], c1 = kcode[key + 1];
#pragma unroll
      for (int hf = 0; hf < 2; ++hf) {
        float b0 = 0.f, b1 = 0.f;
        if (brow[hf] && c0 != 0) {
          const uint32_t bw = __ldg(reinterpret_cast<const unsigned int*>(brow[hf] + key));
          b0 = bf16lo_to_f32(bw);
          b1 = bf16hi_to_f32(bw);
        }
        float& v0 = s[4 * j + 2 * hf];
        float& v1 = s[4 * j + 2 * hf + 1];
        v0 = c0 == 0 ? -INFINITY : ((c0 == 1 || !qvalid[hf]) ? -FLT_MAX : v0 + b0);
        v1 = c1 == 0 ? -INFINITY : ((c1 == 1 || !qvalid[hf]) ? -FLT_MAX : v1 + b1);
        mx[hf] = fmaxf(mx[hf], fmaxf(v0, v1));
      }
    }
    float alpha[2];
#pragma unroll
    for (int hf = 0; hf < 2; ++hf) {
      mx[hf] = fmaxf(mx[hf], __shfl_xor_sync(0xffffffffu, mx[hf], 1));
      mx[hf] = fmaxf(mx[hf], __shfl_xor_sync(0xffffffffu, mx[hf], 2));
      const float m_new = fmaxf(m_run[hf], mx[hf]);    // finite: key 0 of block 0 is never padding
      alpha[hf] = fast_exp2(m_run[hf] - m_new);        // 0 on the first block (m_run = -inf)
      m_run[hf] = m_new;
      l_run[hf] *= alpha[hf];
    }
    uint32_t pa[ATTN_KB / 16][4];
#pragma unroll
    for (int j = 0; j < ATTN_KB / 8; ++j) {
#pragma unroll
      for (int hf = 0; hf < 2; ++hf) {
        const float e0 = fast_exp2(s[4 * j + 2 * hf] - m_run[hf]);
        const float e1 = fast_exp2(s[4 * j + 2 * hf + 1] - m_run[hf]);
        l_run[hf] += e0 + e1;
        // m64k16 A fragment of key chunk j / 2: a0 / a1 = rows lo / hi of keys 2t.., a2 / a3 = the same 8 keys further
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
    for (int kk = 0; kk < ATTN_KB / 16; ++kk) {
      // V tile [key][DH] is the MN-major B operand: 16 keys per step, 8-key groups SBO apart
      const uint64_t vdesc = wgmma_desc(sv + kk * 16 * ROWB, 8192, SBO, SWZ);
      if constexpr (DH == 64) wgmma_m64n64k16_rs<1>(o, pa[kk], vdesc, 1u);
      else wgmma_m64n32k16_rs<1>(o, pa[kk], vdesc, 1u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    reg_fence(o);
    if (lane == 0 && wq == 0) mbar_arrive(&empty_bar[st]);
  }

  // ------------------------------- epilogue: O / l * gate -> bf16 -------------------------------
#pragma unroll
  for (int hf = 0; hf < 2; ++hf) {
    l_run[hf] += __shfl_xor_sync(0xffffffffu, l_run[hf], 1);
    l_run[hf] += __shfl_xor_sync(0xffffffffu, l_run[hf], 2);
    if (rows[hf] >= n) continue;
    const float inv = 1.0f / l_run[hf];
    const long long tok = static_cast<long long>(bb) * p.tok_sb + static_cast<long long>(rows[hf]) * p.tok_si;
    const __nv_bfloat16* g = p.gate + tok * p.ld_gate + hh * DH;
    __nv_bfloat16* out = p.out + tok * p.ld_out + hh * DH;
#pragma unroll
    for (int i = 0; i < DH / 8; ++i) {
      const int e = 8 * i + 2 * (lane & 3);
      const uint32_t gw = __ldg(reinterpret_cast<const unsigned int*>(g + e));
      *reinterpret_cast<uint32_t*>(out + e) =
          pack_bf16x2(o[4 * i + 2 * hf] * inv * bf16lo_to_f32(gw), o[4 * i + 2 * hf + 1] * inv * bf16hi_to_f32(gw));
    }
  }
}

}  // namespace af2
