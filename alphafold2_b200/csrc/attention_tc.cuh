// Axial self-attention with shared additive pair bias and the reference's two-sided mask, on sm_90a wgmma.
// Replaces Attention.forward (alphafold2.py:125-190) as driven by AxialAttention (alphafold2.py:219-255).
//
// Persistent: min(items, SMs) CTAs; CTA c computes the work items c, c + gridDim.x, c + 2 gridDim.x, ...  A work item is
// (folded batch element b', block of 128 queries, head h), numbered head fastest, then query block, then b': the CTAs
// resident at one time read all heads of the same tokens, so whole q|k|v and gate rows come from DRAM together, and the
// query blocks of one (b', h) run close enough together to share its K / V tiles in L2.  An item's arithmetic does not
// depend on which CTA runs it or on what that CTA ran before, so results do not depend on the grid.
// Three warpgroups:
//   warpgroup 0, warp 0   TMA producer, running ahead across items: the Q and gate tiles of an item into one of two item
//                         slots, then its K / V tiles of 128 keys through an ATTN_STAGES-deep ring shared by all items
//   warpgroup 0, warp 1   the key codes of the item's folded row (from the global mask) into the same item slot
//   warpgroups 1, 2       64 query rows each, flash-attention style with everything in registers:
//     S_j = Q K_j^T          wgmma m64n128k16, Q and K from shared memory (K-major)
//     softmax                + pair bias (bf16, read from global / L2 in the accumulator's fragment layout), key / query
//                            mask, online max / sum (the four lanes of a row reduce with two shuffles)
//     O  += P_j V_j          wgmma m64nDHk16 with A = P_j straight from registers (the S fragment of 16 keys IS the
//                            m64k16 A fragment), V consumed MN-major from its [key][dh] layout
//     epilogue               O / l * sigmoid-gate (gate tile from shared memory) -> bf16 [token, h*DH + e]
// Slots and stages are handed over with phase-tracked mbarriers only: an item slot (Q | gate | key codes) is refilled once
// all 256 consumer threads have arrived on its `slot_empty` barrier after their epilogue.
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
  __nv_bfloat16* out;         // [token, heads*DH]; token(b', i) = b'*tok_sb + i*tok_si
  long long tok_sb, tok_si;
  long long ld_out;
};

constexpr int ATTN_THREADS = 384;
constexpr int ATTN_STAGES = 4;
constexpr int ATTN_KB = 128;                        // keys per block
constexpr int ATTN_CONSUMERS = 256;                 // threads of warpgroups 1 and 2

template <int DH>
struct AttnSmem {
  static constexpr int Q_BYTES = 128 * DH * 2;        // one Q or gate tile
  static constexpr int SLOT_BYTES = 2 * Q_BYTES;      // item slot: Q | gate
  static constexpr int KV_BYTES = ATTN_KB * DH * 2;
  static constexpr int STAGE_BYTES = 2 * KV_BYTES;    // K | V
  static constexpr int STAGE_OFF = 2 * SLOT_BYTES;
  static constexpr int BAR_OFF = STAGE_OFF + ATTN_STAGES * STAGE_BYTES;
  static constexpr int KM_OFF = BAR_OFF + 128;        // key codes of the two item slots, kpad(n) each: 0 padding, 1 masked, 2 valid
  static constexpr int kpad(int n) { return (n + ATTN_KB - 1) / ATTN_KB * ATTN_KB; }
  static constexpr int bytes(int n) { return KM_OFF + 2 * kpad(n); }
};

struct AttnItem {
  int h, qb, b;
};
__device__ __forceinline__ AttnItem attn_item(int item, int heads, int nqb) {
  const int r = item / heads;
  return {item - r * heads, r % nqb, r / nqb};
}

// tmQ/tmK/tmV/tmG: 4-D maps over the projection buffer (Q, K, V) and the gate, dims (e [DH], i [n], h [heads],
// b' [nbatch]), box (DH, 128, 1, 1), swizzle = DH*2 bytes.
template <int DH>
__global__ void __launch_bounds__(ATTN_THREADS, 1)
attention_tc_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                    const __grid_constant__ CUtensorMap tmV, const __grid_constant__ CUtensorMap tmG,
                    const __grid_constant__ AttnParams p) {
  using L = AttnSmem<DH>;
  constexpr uint32_t SWZ = (DH == 64) ? SWZ_128 : SWZ_64;
  constexpr uint32_t ROWB = DH * 2;                 // bytes per Q/K/V/gate row
  constexpr uint32_t SBO = 8 * ROWB;                // 8-row swizzle atom
  extern __shared__ __align__(1024) uint8_t smem[];
  if ((smem_u32(smem) & 1023u) != 0) __trap();
  uint64_t* slot_full = reinterpret_cast<uint64_t*>(smem + L::BAR_OFF);   // [2] Q and gate tiles landed
  uint64_t* code_full = slot_full + 2;                                   // [2] key codes written
  uint64_t* slot_empty = code_full + 2;                                  // [2] the consumers are done with the slot
  uint64_t* full_bar = slot_empty + 2;                                   // [ATTN_STAGES] K / V landed
  uint64_t* empty_bar = full_bar + ATTN_STAGES;                          // [ATTN_STAGES] K / V consumed

  const int n = p.n;
  const int nqb = (n + 127) / 128;
  const int nkb = (n + ATTN_KB - 1) / ATTN_KB;
  const int kpad = nkb * ATTN_KB;
  const int items = nqb * p.heads * p.nbatch;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, wg = warp >> 2;

  if (threadIdx.x == 0) {
    prefetch_tmap(&tmQ);
    prefetch_tmap(&tmK);
    prefetch_tmap(&tmV);
    prefetch_tmap(&tmG);
    for (int s = 0; s < 2; ++s) {
      mbar_init(&slot_full[s], 1);
      mbar_init(&code_full[s], 32);              // every lane of the key-code warp
      mbar_init(&slot_empty[s], ATTN_CONSUMERS);
    }
    for (int s = 0; s < ATTN_STAGES; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 2);   // one arrive per softmax warpgroup
    }
    fence_barrier_init();
  }
  __syncthreads();
  // The dependent grid (to_out in the trunk) is launched once every CTA of this one has passed this point, i.e. is resident.  The
  // grid is persistent, so no attention CTA is left waiting for an SM that a dependent CTA could take; the dependent
  // CTAs only fill SMs that attention CTAs have left, and run their set-up in the shadow of the attention tail.
  pdl_launch_dependents();
  pdl_wait();

  if (wg == 0) {
    // ================================ producer warpgroup ================================
    regs_dealloc<40>();
    if (warp == 0 && lane == 0) {
      // TMA: Q | gate into the item slot, then K / V into the ring; runs ahead by up to one item slot and ATTN_STAGES stages
      int kbg = 0;   // key blocks issued by this CTA so far: ring stage and phase
      for (int item = blockIdx.x, it = 0; item < items; item += gridDim.x, ++it) {
        const AttnItem w = attn_item(item, p.heads, nqb);
        const int slot = it & 1;
        mbar_wait(&slot_empty[slot], ((it >> 1) & 1) ^ 1);
        uint8_t* q = smem + slot * L::SLOT_BYTES;
        mbar_arrive_expect_tx(&slot_full[slot], L::SLOT_BYTES);
        tma_load_4d(q, &tmQ, &slot_full[slot], 0, w.qb * 128, w.h, w.b);
        tma_load_4d(q + L::Q_BYTES, &tmG, &slot_full[slot], 0, w.qb * 128, w.h, w.b);
        for (int kb = 0; kb < nkb; ++kb, ++kbg) {
          const int s = kbg % ATTN_STAGES;
          mbar_wait(&empty_bar[s], ((kbg / ATTN_STAGES) & 1) ^ 1);
          uint8_t* st = smem + L::STAGE_OFF + s * L::STAGE_BYTES;
          mbar_arrive_expect_tx(&full_bar[s], L::STAGE_BYTES);
          tma_load_4d(st, &tmK, &full_bar[s], 0, kb * ATTN_KB, w.h, w.b);
          tma_load_4d(st + L::KV_BYTES, &tmV, &full_bar[s], 0, kb * ATTN_KB, w.h, w.b);
        }
      }
    } else if (warp == 1) {
      // key codes of the item's folded row: 0 padding (k >= n), 1 masked, 2 valid
      for (int item = blockIdx.x, it = 0; item < items; item += gridDim.x, ++it) {
        const AttnItem w = attn_item(item, p.heads, nqb);
        const int slot = it & 1;
        mbar_wait(&slot_empty[slot], ((it >> 1) & 1) ^ 1);
        uint8_t* kcode = smem + L::KM_OFF + slot * kpad;
        const uint8_t* mrow = p.mask ? p.mask + static_cast<long long>(w.b) * p.mask_sb : nullptr;
        for (int k = lane; k < kpad; k += 32)
          kcode[k] = k >= n ? 0 : ((mrow && !mrow[static_cast<long long>(k) * p.mask_si]) ? 1 : 2);
        mbar_arrive(&code_full[slot]);
      }
    }
    return;
  }

  // ========================= softmax warpgroups: 64 query rows each =========================
  regs_alloc<232>();
  const int h = wg - 1, wq = warp & 3;
  int kbg = 0;   // key blocks consumed by this CTA so far: ring stage and phase
  for (int item = blockIdx.x, it = 0; item < items; item += gridDim.x, ++it) {
    const AttnItem w = attn_item(item, p.heads, nqb);
    const int slot = it & 1;
    const uint32_t use = (it >> 1) & 1;
    const uint8_t* kcode = smem + L::KM_OFF + slot * kpad;
    mbar_wait(&code_full[slot], use);
    int rows[2];
    bool qvalid[2];
    const __nv_bfloat16* brow[2];
#pragma unroll
    for (int hf = 0; hf < 2; ++hf) {
      rows[hf] = w.qb * 128 + h * 64 + wq * 16 + (lane >> 2) + 8 * hf;
      qvalid[hf] = kcode[rows[hf]] != 1;   // rows < nqb * 128 = kpad; pad rows (code 0) count as valid queries
      // pad rows (>= n) read the bias of row n - 1: their results are never stored and never mix with other rows
      brow[hf] = p.has_bias ? p.bias + (static_cast<long long>(w.h) * n + min(rows[hf], n - 1)) * p.npad : nullptr;
    }
    float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
    float o[DH / 2];
#pragma unroll
    for (int i = 0; i < DH / 2; ++i) o[i] = 0.f;
    float s[ATTN_KB / 2];
    const uint32_t sq = smem_u32(smem + slot * L::SLOT_BYTES) + h * 64 * ROWB;
    mbar_wait(&slot_full[slot], use);

    for (int kb = 0; kb < nkb; ++kb, ++kbg) {
      const int st = kbg % ATTN_STAGES;
      mbar_wait(&full_bar[st], (kbg / ATTN_STAGES) & 1);
      const uint32_t sk = smem_u32(smem + L::STAGE_OFF + st * L::STAGE_BYTES);
      const uint32_t sv = sk + L::KV_BYTES;
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < DH / 16; ++k)
        wgmma_m64n128k16_ss<0, 0>(s, wgmma_desc(sq + k * 32, 16, SBO, SWZ), wgmma_desc(sk + k * 32, 16, SBO, SWZ), k != 0 ? 1u : 0u);
      wgmma_commit();
      wgmma_wait<0>();
      reg_fence(s);

      // the pair bias of this key block, read without branches: pad keys (>= n) read a word inside the row, which the key
      // code then discards
      uint32_t bw[ATTN_KB / 8][2] = {};
      if (p.has_bias) {
#pragma unroll
        for (int j = 0; j < ATTN_KB / 8; ++j) {
          const int key = min(kb * ATTN_KB + 8 * j + 2 * (lane & 3), p.npad - 2);
#pragma unroll
          for (int hf = 0; hf < 2; ++hf) bw[j][hf] = __ldg(reinterpret_cast<const unsigned int*>(brow[hf] + key));
        }
      }

      // logits -> probabilities (in place)
      float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
      for (int j = 0; j < ATTN_KB / 8; ++j) {
        const int key = kb * ATTN_KB + 8 * j + 2 * (lane & 3);
        const uint32_t c0 = kcode[key], c1 = kcode[key + 1];
#pragma unroll
        for (int hf = 0; hf < 2; ++hf) {
          const float b0 = bf16lo_to_f32(bw[j][hf]), b1 = bf16hi_to_f32(bw[j][hf]);
          float& v0 = s[4 * j + 2 * hf];
          float& v1 = s[4 * j + 2 * hf + 1];
          // computed unconditionally and then selected, so that the compiler emits selects rather than branches
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
    const uint8_t* gtile = smem + slot * L::SLOT_BYTES + L::Q_BYTES;
#pragma unroll
    for (int hf = 0; hf < 2; ++hf) {
      l_run[hf] += __shfl_xor_sync(0xffffffffu, l_run[hf], 1);
      l_run[hf] += __shfl_xor_sync(0xffffffffu, l_run[hf], 2);
      if (rows[hf] >= n) continue;
      const float inv = 1.0f / l_run[hf];
      const long long tok = static_cast<long long>(w.b) * p.tok_sb + static_cast<long long>(rows[hf]) * p.tok_si;
      __nv_bfloat16* out = p.out + tok * p.ld_out + w.h * DH;
      const uint32_t r = rows[hf] - w.qb * 128;   // row of the gate tile
#pragma unroll
      for (int i = 0; i < DH / 8; ++i) {
        const int e = 8 * i + 2 * (lane & 3);
        // the TMA swizzle moves 16-byte chunk c of row r to chunk c ^ (r % 8) (128 B rows) or c ^ (r / 2 % 4) (64 B rows)
        const uint32_t off = r * ROWB + e * 2;
        const uint32_t gw = *reinterpret_cast<const uint32_t*>(gtile + (off ^ (((off >> 7) & (DH == 64 ? 7u : 3u)) << 4)));
        *reinterpret_cast<uint32_t*>(out + e) =
            pack_bf16x2(o[4 * i + 2 * hf] * inv * bf16lo_to_f32(gw), o[4 * i + 2 * hf + 1] * inv * bf16hi_to_f32(gw));
      }
    }
    mbar_arrive(&slot_empty[slot]);
  }
}

}  // namespace af2
