// Template embedder kernels (alphafold2.py:743-785).
//
// template_pointwise_kernel: the pointwise template attention of Alphafold2.forward.  At every pair position p = (b, i, j) ONE
// query from x attends over the T template vectors at the same position:
//   logit_t = q[p] . k[(b T + t) pairs + ij]   per head, -FLT_MAX where !(x_mask[p] & t_mask[b T + t][ij])
//   out[p]  = gate[p] * sum_t softmax_t(logit) v[(b T + t) pairs + ij]
//   pooled[p] = any_t t_mask[b T + t][ij]                 (exactly 0 or 1; NOT x_mask, quirk of alphafold2.py:779)
// A pair whose logits are all masked gets the uniform mean over all T templates, masked ones included (-FLT_MAX fill of the
// reference, alphafold2.py:162-167): the online softmax below reaches that without a branch (every -FLT_MAX logit then
// contributes 2^0 = 1).
//
// The kernel is memory-bound: per pair it reads q, gate (I elements each) and T rows of k|v (2I each), and writes I + 1
// values.  One thread owns VEC = 16 / sizeof(E) consecutive channels of one pair (one 16-byte load per operand row), the
// dh / VEC lanes of one head reduce the dot product with xor shuffles, and every k|v row is read exactly once.  There is no
// bound on T: the softmax is online (running max, running sum, rescaled accumulator), in fp32.
//   E = bf16 : q pre-scaled by dim_head^-0.5 * log2(e), logits in the log2 domain on ex2.approx, gate already sigmoid-ed.
//   E = float: strict mode -- q pre-scaled by dim_head^-0.5, expf, gate given as logits (sigmoid by expf here).
#pragma once
#include <cfloat>
#include "common.cuh"
#include "strict_kernels.cuh"

namespace af2 {

struct TplParams {
  const void* q; const void* gate; const void* kv;       // q [P][ld_q], gate [P][ld_gate], kv [B T pairs][2I] (k | v)
  const uint8_t* x_mask;                                  // [P] or nullptr (all valid)
  const uint8_t* t_mask;                                  // [B T pairs] or nullptr (all valid)
  void* out;                                              // [P][I]
  float* pooled;                                          // [P]
  long long pairs;                                        // pair positions per batch element (n * n)
  long long ld_q, ld_gate;                                // row strides of q / gate (elements)
  int B, T, heads, dh;
};

template <typename E> struct TplVec;
template <> struct TplVec<__nv_bfloat16> {
  static constexpr int N = 8;
  __device__ static void load(const void* p, float (&v)[8]) {
    const uint4 u = __ldcs(reinterpret_cast<const uint4*>(p));
    const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) { v[2 * i] = bf16lo_to_f32(w[i]); v[2 * i + 1] = bf16hi_to_f32(w[i]); }
  }
  __device__ static void store(void* p, const float (&v)[8]) {
    uint4 u;
    u.x = pack_bf16x2(v[0], v[1]); u.y = pack_bf16x2(v[2], v[3]); u.z = pack_bf16x2(v[4], v[5]); u.w = pack_bf16x2(v[6], v[7]);
    *reinterpret_cast<uint4*>(p) = u;
  }
  __device__ static float exp(float x) { return fast_exp2(x); }
  __device__ static float gate(float g) { return g; }
};
template <> struct TplVec<float> {
  static constexpr int N = 4;
  __device__ static void load(const void* p, float (&v)[4]) {
    const float4 u = __ldcs(reinterpret_cast<const float4*>(p));
    v[0] = u.x; v[1] = u.y; v[2] = u.z; v[3] = u.w;
  }
  __device__ static void store(void* p, const float (&v)[4]) { *reinterpret_cast<float4*>(p) = make_float4(v[0], v[1], v[2], v[3]); }
  __device__ static float exp(float x) { return expf(x); }
  __device__ static float gate(float g) { return 1.0f / (1.0f + expf(-g)); }
};

// grid-stride over warps: all 32 lanes of a warp step together, so the head groups (dh / VEC lanes, a power of two that
// divides 32, starting at a multiple of its size) always shuffle inside one warp
template <typename E>
__global__ void __launch_bounds__(256) template_pointwise_kernel(const TplParams p) {
  using V = TplVec<E>;
  constexpr int VEC = V::N;
  const int I = p.heads * p.dh;
  const int C = I / VEC;                       // work items per pair
  const int G = p.dh / VEC;                    // lanes per head
  const long long P = (long long)p.B * p.pairs;
  const long long total = P * C;
  const int lane = threadIdx.x & 31;
  const long long stride = (long long)gridDim.x * blockDim.x;
  pdl_wait();
  for (long long base = (long long)blockIdx.x * blockDim.x + (threadIdx.x & ~31); base < total; base += stride) {
    const long long idx = base + lane;
    const bool active = idx < total;
    const long long pr = active ? idx / C : 0;
    const int c = active ? (int)(idx - pr * C) : 0;
    const long long b = pr / p.pairs, ij = pr - b * p.pairs;
    float q[VEC], g[VEC], acc[VEC];
#pragma unroll
    for (int e = 0; e < VEC; ++e) { q[e] = 0.f; g[e] = 0.f; acc[e] = 0.f; }
    if (active) {
      V::load(static_cast<const E*>(p.q) + pr * p.ld_q + (long long)c * VEC, q);
      V::load(static_cast<const E*>(p.gate) + pr * p.ld_gate + (long long)c * VEC, g);
    }
    const bool xm = !p.x_mask || (active && p.x_mask[pr]);
    float mx = -INFINITY, l = 0.f;
    bool any = false;
    const long long row0 = b * p.T * p.pairs + ij;
#pragma unroll 4
    for (int t = 0; t < p.T; ++t) {
      const long long row = row0 + (long long)t * p.pairs;
      float k[VEC], v[VEC];
      bool tv = true;
      if (active) {
        const E* kr = static_cast<const E*>(p.kv) + row * 2 * I + (long long)c * VEC;
        V::load(kr, k);
        V::load(kr + I, v);
        if (p.t_mask) tv = p.t_mask[row] != 0;
      } else {
#pragma unroll
        for (int e = 0; e < VEC; ++e) { k[e] = 0.f; v[e] = 0.f; }
      }
      float s = 0.f;
#pragma unroll
      for (int e = 0; e < VEC; ++e) s = fmaf(q[e], k[e], s);
      for (int o = 1; o < G; o <<= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
      any |= tv;
      if (!(xm && tv)) s = -FLT_MAX;
      const float mn = fmaxf(mx, s);
      const float alpha = V::exp(mx - mn);     // 0 on the first template (mx = -inf)
      const float pt = V::exp(s - mn);
      l = fmaf(l, alpha, pt);
#pragma unroll
      for (int e = 0; e < VEC; ++e) acc[e] = fmaf(acc[e], alpha, pt * v[e]);
      mx = mn;
    }
    if (active) {
      const float inv = 1.0f / l;
#pragma unroll
      for (int e = 0; e < VEC; ++e) acc[e] = acc[e] * inv * V::gate(g[e]);
      V::store(static_cast<E*>(p.out) + pr * I + (long long)c * VEC, acc);
      if (c == 0) p.pooled[pr] = any ? 1.0f : 0.0f;
    }
  }
  pdl_launch_dependents();
}

// y[r][c] = bf16(x[r][c]) for c < K, 0 for K <= c < P   (x fp32 [rows][K], y [rows][P])
__global__ void __launch_bounds__(256) f32_to_bf16_pad_kernel(const float* __restrict__ x, __nv_bfloat16* __restrict__ y,
                                                              long long rows, int K, int P) {
  const long long total = rows * P;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / P;
    const int c = (int)(i - r * P);
    y[i] = __float2bfloat16(c < K ? x[r * K + c] : 0.f);
  }
}

// the same for K == P, K % 4 == 0: 16-byte loads, 8-byte stores
__global__ void __launch_bounds__(256) f32_to_bf16_vec_kernel(const float4* __restrict__ x, uint2* __restrict__ y, long long n4) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
    const float4 v = __ldcs(x + i);
    y[i] = make_uint2(pack_bf16x2(v.x, v.y), pack_bf16x2(v.z, v.w));
  }
}

// strict angle MLP: y split [rows][SPL][P] = exact erf-GELU of h fp32 [rows][d] (pad columns zero)
__global__ void __launch_bounds__(256) strict_gelu_split_kernel(const float* __restrict__ h, __nv_bfloat16* __restrict__ y,
                                                                long long rows, int d, int P) {
  const long long total = rows * P;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / P;
    const int c = (int)(i - r * P);
    split_store(y + r * SPL * P + c, P, c < d ? gelu_acc(h[r * d + c]) : 0.f);
  }
}

}  // namespace af2
