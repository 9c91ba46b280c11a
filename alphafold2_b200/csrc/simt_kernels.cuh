// Bandwidth-bound helper kernels (no tensor-core work): row LayerNorm with optional fused pair-bias
// projection, channel-major -> token-major LayerNorm*gate, pair-mask counts, rotary embedding.
// All are coalesced / vectorised and sized as grid-stride loops over (SM count) x k CTAs.
#pragma once
#include "common.cuh"

namespace af2 {

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// ------------------------------------------------------------------------------------------------
// y = LayerNorm(x) * gamma + beta  -> bf16 [T, d]          (nn.LayerNorm, eps inside sqrt)
// optionally  bias[h][(t / n_inner) * pitch + t % n_inner] = <x_raw[t, :], Wb[h, :]>   (bf16)
//   (edges_to_attn_bias of alphafold2.py:214-217,245-247 acts on the RAW, un-normalised pair tensor)
// One warp per row; the row lives in registers (d <= 1024, d % 4 == 0).
// ------------------------------------------------------------------------------------------------
struct LnParams {
  const float* x;
  const float* gamma;
  const float* beta;
  __nv_bfloat16* y;        // may be nullptr (bias only)
  long long T;
  int d;
  float eps;
  const float* wb;         // [H, d] or nullptr
  __nv_bfloat16* bias_out; // [H][bias_hs]
  int heads;
  long long bias_hs;       // elements between heads
  int n_inner, pitch;      // token t -> (t / n_inner) * pitch + t % n_inner
};

template <int MAXC>
__global__ void __launch_bounds__(256) layernorm_rows_kernel(const LnParams p) {
  const int lane = threadIdx.x & 31;
  const int warps_per_block = blockDim.x >> 5;
  const long long warp_global = static_cast<long long>(blockIdx.x) * warps_per_block + (threadIdx.x >> 5);
  const long long nwarps = static_cast<long long>(gridDim.x) * warps_per_block;
  const int nchunk = p.d >> 2;   // float4 chunks per row
  for (long long t = warp_global; t < p.T; t += nwarps) {
    const float4* xr = reinterpret_cast<const float4*>(p.x + t * p.d);
    float4 v[MAXC];
    float sum = 0.f;
#pragma unroll
    for (int c = 0; c < MAXC; ++c) {
      const int idx = lane + 32 * c;
      if (idx < nchunk) {
        v[c] = __ldg(xr + idx);
        sum += v[c].x + v[c].y + v[c].z + v[c].w;
      } else {
        v[c] = make_float4(0.f, 0.f, 0.f, 0.f);
      }
    }
    const float mean = warp_sum(sum) / p.d;
    float sq = 0.f;
#pragma unroll
    for (int c = 0; c < MAXC; ++c) {
      const int idx = lane + 32 * c;
      if (idx < nchunk) {
        const float a = v[c].x - mean, b = v[c].y - mean, cc = v[c].z - mean, dd = v[c].w - mean;
        sq += a * a + b * b + cc * cc + dd * dd;
      }
    }
    const float rstd = rsqrtf(warp_sum(sq) / p.d + p.eps);
    if (p.y) {
      uint2* yr = reinterpret_cast<uint2*>(p.y + t * p.d);
#pragma unroll
      for (int c = 0; c < MAXC; ++c) {
        const int idx = lane + 32 * c;
        if (idx < nchunk) {
          const float4 g = __ldg(reinterpret_cast<const float4*>(p.gamma) + idx);
          const float4 b = __ldg(reinterpret_cast<const float4*>(p.beta) + idx);
          const float o0 = (v[c].x - mean) * rstd * g.x + b.x;
          const float o1 = (v[c].y - mean) * rstd * g.y + b.y;
          const float o2 = (v[c].z - mean) * rstd * g.z + b.z;
          const float o3 = (v[c].w - mean) * rstd * g.w + b.w;
          yr[idx] = make_uint2(pack_bf16x2(o0, o1), pack_bf16x2(o2, o3));
        }
      }
    }
    if (p.wb) {
      const long long off = (t / p.n_inner) * p.pitch + (t % p.n_inner);
      // 8 heads at a time: per-lane partial dot products, then a recursive-halving butterfly (9 shuffles for 8
      // sums instead of 40): after the xor-16/8/4 steps lane l holds head ((l>>2)&7)'s partial, xor-2/1 finish it.
      for (int h0 = 0; h0 < p.heads; h0 += 8) {
        float acc[8];
#pragma unroll
        for (int hh = 0; hh < 8; ++hh) {
          acc[hh] = 0.f;
          if (h0 + hh < p.heads) {
            const float4* wr = reinterpret_cast<const float4*>(p.wb + static_cast<long long>(h0 + hh) * p.d);
#pragma unroll
            for (int c = 0; c < MAXC; ++c) {
              const int idx = lane + 32 * c;
              if (idx < nchunk) {
                const float4 w = __ldg(wr + idx);
                acc[hh] += v[c].x * w.x + v[c].y * w.y + v[c].z * w.z + v[c].w * w.w;
              }
            }
          }
        }
        const bool b4 = lane & 16, b3 = lane & 8, b2 = lane & 4;
        float w4[4], w2[2];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const float mine = b4 ? acc[4 + i] : acc[i];
          const float other = b4 ? acc[i] : acc[4 + i];
          w4[i] = mine + __shfl_xor_sync(0xffffffffu, other, 16);
        }
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          const float mine = b3 ? w4[2 + i] : w4[i];
          const float other = b3 ? w4[i] : w4[2 + i];
          w2[i] = mine + __shfl_xor_sync(0xffffffffu, other, 8);
        }
        float w1 = (b2 ? w2[1] : w2[0]) + __shfl_xor_sync(0xffffffffu, b2 ? w2[0] : w2[1], 4);
        w1 += __shfl_xor_sync(0xffffffffu, w1, 2);
        w1 += __shfl_xor_sync(0xffffffffu, w1, 1);
        const int hsel = h0 + ((lane >> 2) & 7);
        if ((lane & 3) == 0 && hsel < p.heads) p.bias_out[hsel * p.bias_hs + off] = __float2bfloat16(w1);
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------
// Channel-major fp32 contraction output  ->  token-major bf16 operand of the following Linear.
//   src[c][row * pitch + j]   (c < d channels, row < rows, j < n)    token = row * n + j
//   mode 0 (triangle multiply tail, alphafold2.py:315-316):  y = LayerNorm_c(src) * gamma + beta, * gate[token, c]
//   mode 1 (outer mean tail,      alphafold2.py:347-349):    y = src * scale[token]
// Block = 256 threads handles 32 consecutive j of one row: coalesced reads along j, smem transpose,
// coalesced bf16 writes along c.
// ------------------------------------------------------------------------------------------------
struct ChanLnParams {
  const float* src;
  long long chan_stride;
  int pitch, rows, n, d;
  int mode;
  const float* gamma;
  const float* beta;
  const __nv_bfloat16* gate;   // [tokens, d]
  const float* scale;          // [tokens]
  float scale_const;           // used when scale == nullptr (mode 1)
  float eps;
  __nv_bfloat16* y;            // [tokens, d]
};

__global__ void __launch_bounds__(256) chan_to_token_kernel(const ChanLnParams p) {
  extern __shared__ float tile[];   // [d][33]
  const int jt = blockIdx.x, row = blockIdx.y;
  const int j0 = jt * 32;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const bool j_ok = (j0 + lane) < p.n;
  const float* src = p.src + static_cast<long long>(row) * p.pitch + j0 + lane;
  for (int c = warp; c < p.d; c += 8)
    tile[c * 33 + lane] = j_ok ? __ldg(src + c * p.chan_stride) : 0.f;
  __syncthreads();
  for (int tk = warp; tk < 32; tk += 8) {
    if (j0 + tk >= p.n) break;
    const long long token = static_cast<long long>(row) * p.n + j0 + tk;
    if (p.mode == 0) {
      float sum = 0.f;
      for (int c = lane; c < p.d; c += 32) sum += tile[c * 33 + tk];
      const float mean = warp_sum(sum) / p.d;
      float sq = 0.f;
      for (int c = lane; c < p.d; c += 32) {
        const float a = tile[c * 33 + tk] - mean;
        sq += a * a;
      }
      const float rstd = rsqrtf(warp_sum(sq) / p.d + p.eps);
      for (int c = lane; c < p.d; c += 32) {
        const float g = __bfloat162float(p.gate[token * p.d + c]);
        const float o = ((tile[c * 33 + tk] - mean) * rstd * __ldg(p.gamma + c) + __ldg(p.beta + c)) * g;
        p.y[token * p.d + c] = __float2bfloat16(o);
      }
    } else {
      const float sc = p.scale ? __ldg(p.scale + token) : p.scale_const;
      for (int c = lane; c < p.d; c += 32) p.y[token * p.d + c] = __float2bfloat16(tile[c * 33 + tk] * sc);
    }
  }
}

// ------------------------------------------------------------------------------------------------
// Pair bias of axial / triangle attention (alphafold2.py:214-217, 245-247):
//   bias[h][(t / n_inner) * pitch + t % n_inner] = <x_raw[t, :], Wb[h, :]>      bf16, H <= 8 heads per pass, d <= 256
// Eight lanes share a token (4 tokens per warp instruction): 128-byte coalesced row segments, w_edge staged in shared
// memory, 3-level shuffle reductions.  Streams x once (HBM bound).
// ------------------------------------------------------------------------------------------------
struct PairBiasParams {
  const float* x;
  long long T;
  int d;
  const float* wb;          // [H, d]
  __nv_bfloat16* bias_out;  // [H][bias_hs]
  int heads;
  long long bias_hs;
  int n_inner, pitch;
  int x_evict_last;         // 1: loads of x carry an L2 evict_last hint (AF2_X_EVICT_LAST)
  int transpose;            // 1: token t = (i, j) is stored at [j][i] instead of [i][j] (the attention kernel's K-major bias operand)
};

__device__ __forceinline__ float4 ldg_stream4(const float4* p) {
  float4 v;
  asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p));
  return v;
}

template <int NJ>
__global__ void __launch_bounds__(256, 3) pair_bias_kernel(const PairBiasParams p) {
  // No shared-memory prologue: w_edge (<= 8 KB) is read through L1 (every lane group reads the same 128 bytes), the
  // activations stream past L1 (no_allocate), so a block starts loading tokens immediately.
  const int lane = threadIdx.x & 31, sub = lane & 7, rg = lane >> 3;
  const int warp_global = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int nwarps = gridDim.x * (blockDim.x >> 5);
  const int groups = static_cast<int>((p.T + 3) / 4);
  for (int gidx = warp_global; gidx < groups; gidx += nwarps) {
    const long long t = static_cast<long long>(gidx) * 4 + rg;
    const bool live = t < p.T;
    float4 v[NJ];
    const float4* xr = reinterpret_cast<const float4*>(p.x + (live ? t : 0) * p.d) + sub;
#pragma unroll
    for (int j = 0; j < NJ; ++j) v[j] = live ? ldg_stream4(xr + j * 8) : make_float4(0.f, 0.f, 0.f, 0.f);
    float acc[8];
#pragma unroll
    for (int h = 0; h < 8; ++h) {
      acc[h] = 0.f;
      if (h < p.heads) {
        const float4* wr = reinterpret_cast<const float4*>(p.wb + h * p.d) + sub;
#pragma unroll
        for (int j = 0; j < NJ; ++j) {
          const float4 w = __ldg(wr + j * 8);
          acc[h] += v[j].x * w.x + v[j].y * w.y + v[j].z * w.z + v[j].w * w.w;
        }
      }
    }
    // reduce over the 8 lanes of the token: after xor-4 / 2 / 1 halving, lane `sub` holds head `sub`
    float r4[4], r2[2];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const bool hi = sub & 4;
      const float mine = hi ? acc[4 + k] : acc[k], other = hi ? acc[k] : acc[4 + k];
      r4[k] = mine + __shfl_xor_sync(0xffffffffu, other, 4);
    }
#pragma unroll
    for (int k = 0; k < 2; ++k) {
      const bool hi = sub & 2;
      const float mine = hi ? r4[2 + k] : r4[k], other = hi ? r4[k] : r4[2 + k];
      r2[k] = mine + __shfl_xor_sync(0xffffffffu, other, 2);
    }
    const bool hi1 = sub & 1;
    const float res = (hi1 ? r2[1] : r2[0]) + __shfl_xor_sync(0xffffffffu, hi1 ? r2[0] : r2[1], 1);
    if (live && sub < p.heads) {
      const int ti = static_cast<int>(t);                        // T < 2^31 (checked by the host)
      const int ti_i = ti / p.n_inner, ti_j = ti - ti_i * p.n_inner;
      const long long off = p.transpose ? static_cast<long long>(ti_j) * p.pitch + ti_i : static_cast<long long>(ti_i) * p.pitch + ti_j;
      p.bias_out[sub * p.bias_hs + off] = __float2bfloat16(res);
    }
  }
}

// Tensor-core variant (legacy mma.sync m16n8k16, N = 8 heads is exactly one MMA tile): the SIMT kernel above is bound by
// the load-instruction rate of w_edge (64 loads per 4 tokens); here w_edge lives in B fragments (registers) for the whole
// kernel and x streams through A fragments.  Both operands are split hi + lo into bf16 fragments and three products
// (hi*hi + lo*hi + hi*lo) are accumulated in fp32, i.e. ~16 mantissa bits per operand: the bias matches the fp32 dot
// product of the reference to ~1e-5 relative before its bf16 store.
template <int KSTEPS>   // d / 16
__global__ void __launch_bounds__(256, 2) pair_bias_mma_kernel(const PairBiasParams p) {
  const int lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const int warp_global = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int nwarps = gridDim.x * (blockDim.x >> 5);
  // B fragments: B[k][n] = w_edge[n][k]; thread holds k = 16 ks + {2t, 2t+1} and {2t+8, 2t+9} of head n = g
  uint32_t bfrag[KSTEPS][2], blo[KSTEPS][2];
#pragma unroll
  for (int ks = 0; ks < KSTEPS; ++ks) {
    float2 w0 = make_float2(0.f, 0.f), w1 = make_float2(0.f, 0.f);
    if (g < p.heads) {
      w0 = __ldg(reinterpret_cast<const float2*>(p.wb + g * p.d + ks * 16 + 2 * t));
      w1 = __ldg(reinterpret_cast<const float2*>(p.wb + g * p.d + ks * 16 + 2 * t + 8));
    }
    bfrag[ks][0] = pack_bf16x2(w0.x, w0.y);
    bfrag[ks][1] = pack_bf16x2(w1.x, w1.y);
    blo[ks][0] = pack_bf16x2(w0.x - bf16lo_to_f32(bfrag[ks][0]), w0.y - bf16hi_to_f32(bfrag[ks][0]));
    blo[ks][1] = pack_bf16x2(w1.x - bf16lo_to_f32(bfrag[ks][1]), w1.y - bf16hi_to_f32(bfrag[ks][1]));
  }
  const int groups = static_cast<int>((p.T + 15) / 16);
  const uint64_t pol = l2_policy(p.x_evict_last != 0);
  pdl_wait();            // (the w_edge fragments above are weights: safe to load before the predecessor has finished)
  for (int gi = warp_global; gi < groups; gi += nwarps) {
    const long long r0 = static_cast<long long>(gi) * 16 + g, r1 = r0 + 8;
    const bool l0 = r0 < p.T, l1 = r1 < p.T;
    const float* x0 = p.x + (l0 ? r0 : 0) * p.d + 2 * t;
    const float* x1 = p.x + (l1 ? r1 : 0) * p.d + 2 * t;
    float c[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
    for (int ks = 0; ks < KSTEPS; ++ks) {
      float2 a[4];
      a[0] = l0 ? ldg_f2_hint(reinterpret_cast<const float2*>(x0 + ks * 16), pol) : make_float2(0.f, 0.f);
      a[1] = l1 ? ldg_f2_hint(reinterpret_cast<const float2*>(x1 + ks * 16), pol) : make_float2(0.f, 0.f);
      a[2] = l0 ? ldg_f2_hint(reinterpret_cast<const float2*>(x0 + ks * 16 + 8), pol) : make_float2(0.f, 0.f);
      a[3] = l1 ? ldg_f2_hint(reinterpret_cast<const float2*>(x1 + ks * 16 + 8), pol) : make_float2(0.f, 0.f);
      uint32_t hi[4], lo[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        hi[i] = pack_bf16x2(a[i].x, a[i].y);
        lo[i] = pack_bf16x2(a[i].x - bf16lo_to_f32(hi[i]), a[i].y - bf16hi_to_f32(hi[i]));
      }
      asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
                   : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
                   : "r"(hi[0]), "r"(hi[1]), "r"(hi[2]), "r"(hi[3]), "r"(bfrag[ks][0]), "r"(bfrag[ks][1]));
      asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
                   : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
                   : "r"(lo[0]), "r"(lo[1]), "r"(lo[2]), "r"(lo[3]), "r"(bfrag[ks][0]), "r"(bfrag[ks][1]));
      asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
                   : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
                   : "r"(hi[0]), "r"(hi[1]), "r"(hi[2]), "r"(hi[3]), "r"(blo[ks][0]), "r"(blo[ks][1]));
    }
    // c0, c1: token r0, heads 2t, 2t+1;  c2, c3: token r1
    const int h0 = 2 * t;
    if (l0) {
      const int ti = static_cast<int>(r0);
      const int ti_i = ti / p.n_inner, ti_j = ti - ti_i * p.n_inner;
      const long long off = p.transpose ? static_cast<long long>(ti_j) * p.pitch + ti_i : static_cast<long long>(ti_i) * p.pitch + ti_j;
      if (h0 < p.heads) p.bias_out[h0 * p.bias_hs + off] = __float2bfloat16(c[0]);
      if (h0 + 1 < p.heads) p.bias_out[(h0 + 1) * p.bias_hs + off] = __float2bfloat16(c[1]);
    }
    if (l1) {
      const int ti = static_cast<int>(r1);
      const int ti_i = ti / p.n_inner, ti_j = ti - ti_i * p.n_inner;
      const long long off = p.transpose ? static_cast<long long>(ti_j) * p.pitch + ti_i : static_cast<long long>(ti_i) * p.pitch + ti_j;
      if (h0 < p.heads) p.bias_out[h0 * p.bias_hs + off] = __float2bfloat16(c[2]);
      if (h0 + 1 < p.heads) p.bias_out[(h0 + 1) * p.bias_hs + off] = __float2bfloat16(c[3]);
    }
  }
}

// ------------------------------------------------------------------------------------------------
// Channel-major fp32 contraction output -> token-major bf16 operand, tile version (replaces chan_to_token_kernel when the
// token grid is dense, pitch == n):  a CTA (512 threads) owns 64 consecutive tokens x all d channels:
//   phase 1: 256-byte coalesced row segments src[c][t0 .. t0+63] -> shared tile [d][64] (16 independent 16-byte loads per thread)
//   phase 2: thread = (token, 32-channel slice): LayerNorm over channels (mode 0) or scale (mode 1), gate, 64-byte bf16 stores
// ------------------------------------------------------------------------------------------------
template <int CPT>   // channels per thread = d / 8
__global__ void __launch_bounds__(512) chan_to_token_tile_kernel(const ChanLnParams p, long long T) {
  extern __shared__ float tile[];                      // [d][64] followed by [8][64][2] partial moments
  constexpr int D = CPT * 8;
  const long long t0 = static_cast<long long>(blockIdx.x) * 64;
  const int tid = threadIdx.x;
  // ---- phase 1: D / 32 independent 16-byte loads per thread ----
  {
    const int q = tid & 15;                            // float4 index inside the 64-token segment
    const bool ok = (t0 + q * 4) < T;                  // T % 4 == 0 (pitch multiple of 4)
    const float4* src = reinterpret_cast<const float4*>(p.src + t0) + q;
    float4 v[D / 32];
#pragma unroll
    for (int k = 0; k < D / 32; ++k) {
      const int c = (tid >> 4) + k * 32;
      v[k] = ok ? ldg_stream4(reinterpret_cast<const float4*>(reinterpret_cast<const float*>(src) + static_cast<long long>(c) * p.chan_stride))
                : make_float4(0.f, 0.f, 0.f, 0.f);
    }
#pragma unroll
    for (int k = 0; k < D / 32; ++k) reinterpret_cast<float4*>(tile + ((tid >> 4) + k * 32) * 64)[q] = v[k];
  }
  __syncthreads();
  // ---- phase 2: thread = (token, slice of CPT channels); the slice lives in registers ----
  const int tok = tid & 63, slice = tid >> 6;
  const int c0 = slice * CPT;
  const long long token = t0 + tok;
  float* part = tile + D * 64;
  float x[CPT];
#pragma unroll
  for (int i = 0; i < CPT; ++i) x[i] = tile[(c0 + i) * 64 + tok];
  float mean = 0.f, rstd = 1.f;
  if (p.mode == 0) {
    float s1 = 0.f;
#pragma unroll
    for (int i = 0; i < CPT; ++i) s1 += x[i];
    part[(slice * 64 + tok) * 2] = s1;
    __syncthreads();
    float tot = 0.f;
#pragma unroll
    for (int k = 0; k < 8; ++k) tot += part[(k * 64 + tok) * 2];
    mean = tot * (1.0f / D);
    float s2 = 0.f;
#pragma unroll
    for (int i = 0; i < CPT; ++i) {
      const float a = x[i] - mean;
      s2 += a * a;
    }
    part[(slice * 64 + tok) * 2 + 1] = s2;
    __syncthreads();
    float var = 0.f;
#pragma unroll
    for (int k = 0; k < 8; ++k) var += part[(k * 64 + tok) * 2 + 1];
    rstd = rsqrtf(var * (1.0f / D) + p.eps);
  }
  if (token < T) {
    const float sc = (p.mode == 1) ? (p.scale ? __ldg(p.scale + token) : p.scale_const) : 1.f;
#pragma unroll
    for (int i = 0; i < CPT; i += 8) {
      float o[8];
      if (p.mode == 0) {
        const uint4 gq = __ldg(reinterpret_cast<const uint4*>(p.gate + token * D + c0 + i));
        const uint32_t gw[4] = {gq.x, gq.y, gq.z, gq.w};
        const float4 ga = __ldg(reinterpret_cast<const float4*>(p.gamma + c0 + i)), gb = __ldg(reinterpret_cast<const float4*>(p.gamma + c0 + i + 4));
        const float4 ba = __ldg(reinterpret_cast<const float4*>(p.beta + c0 + i)), bb = __ldg(reinterpret_cast<const float4*>(p.beta + c0 + i + 4));
        const float gm[8] = {ga.x, ga.y, ga.z, ga.w, gb.x, gb.y, gb.z, gb.w};
        const float bt[8] = {ba.x, ba.y, ba.z, ba.w, bb.x, bb.y, bb.z, bb.w};
#pragma unroll
        for (int k = 0; k < 8; ++k) {
          const float g = (k & 1) ? bf16hi_to_f32(gw[k >> 1]) : bf16lo_to_f32(gw[k >> 1]);
          o[k] = ((x[i + k] - mean) * rstd * gm[k] + bt[k]) * g;
        }
      } else {
#pragma unroll
        for (int k = 0; k < 8; ++k) o[k] = x[i + k] * sc;
      }
      *reinterpret_cast<uint4*>(p.y + token * D + c0 + i) =
          make_uint4(pack_bf16x2(o[0], o[1]), pack_bf16x2(o[2], o[3]), pack_bf16x2(o[4], o[5]), pack_bf16x2(o[6], o[7]));
    }
  }
}

// ------------------------------------------------------------------------------------------------
// OuterMean normaliser (quirk Q3, alphafold2.py:345-347):
//   scale[b][i][j] = 1 / (S * (sum_s mask[b,s,i] * mask[b,s,j] + eps))      (fp32, like the reference)
// ------------------------------------------------------------------------------------------------
__global__ void outer_scale_kernel(const uint8_t* __restrict__ mask, float* __restrict__ scale, int B, int S, int N,
                                   float eps) {
  const long long total = static_cast<long long>(B) * N * N;
  for (long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; idx < total;
       idx += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int j = idx % N;
    const int i = (idx / N) % N;
    const int b = idx / (static_cast<long long>(N) * N);
    const uint8_t* mb = mask + static_cast<long long>(b) * S * N;
    int cnt = 0;
    for (int s = 0; s < S; ++s) cnt += (mb[s * N + i] != 0) & (mb[s * N + j] != 0);
    scale[idx] = 1.0f / (static_cast<float>(S) * (static_cast<float>(cnt) + eps));
  }
}

// same for a band of pair rows [row0, row0 + rows) (sharded outer mean): scale[(i - row0) * N + j]
__global__ void outer_scale_rows_kernel(const uint8_t* __restrict__ mask, float* __restrict__ scale, int row0, int rows,
                                        int S, int N, float eps) {
  const long long total = static_cast<long long>(rows) * N;
  for (long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; idx < total;
       idx += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int j = idx % N;
    const int i = row0 + static_cast<int>(idx / N);
    int cnt = 0;
    for (int s = 0; s < S; ++s) cnt += (mask[s * N + i] != 0) & (mask[s * N + j] != 0);
    scale[idx] = 1.0f / (static_cast<float>(S) * (static_cast<float>(cnt) + eps));
  }
}

// Bit-packed version of both kernels above: count[i][j] = popc(bits_i & bits_j) with bits_i = the S mask bits of residue i.
//   mask_pack_bits_kernel: words[w][i] (w = s / 32) <- the [S][N] byte mask, once per call (coalesced byte reads over i);
//   outer_scale_bits_kernel: every block copies the packed words (S/32 * N * 4 bytes, L2 resident) into shared memory and
//   walks its (i, j) pairs: the i-word is a broadcast, the j-words are consecutive -> conflict-free.  S / 32 AND+POPC steps
//   per pair instead of S byte-pair loads (C2: 17.6 us -> ~4 us; the first version packed inside every block: 150 us at C4).
__global__ void __launch_bounds__(256) mask_pack_bits_kernel(const uint8_t* __restrict__ mask, uint32_t* __restrict__ words, int S, int N) {
  const int nw = (S + 31) >> 5;
  for (int idx = blockIdx.x * blockDim.x + threadIdx.x; idx < nw * N; idx += gridDim.x * blockDim.x) {
    const int w = idx / N, i = idx - w * N;
    uint32_t v = 0;
    const int s1 = min(S, (w + 1) * 32);
    for (int s = w * 32; s < s1; ++s) v |= (mask[static_cast<long long>(s) * N + i] != 0 ? 1u : 0u) << (s & 31);
    words[idx] = v;
  }
}
__global__ void __launch_bounds__(256) outer_scale_bits_kernel(const uint32_t* __restrict__ words, float* __restrict__ scale,
                                                               int row0, int rows, int S, int N, float eps) {
  extern __shared__ uint32_t bits[];                 // [words][N]
  const int nw = (S + 31) >> 5;
  for (int idx = threadIdx.x; idx < nw * N; idx += blockDim.x) bits[idx] = words[idx];
  __syncthreads();
  const long long total = static_cast<long long>(rows) * N;
  const float fS = static_cast<float>(S);
  for (long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; idx < total;
       idx += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int j = static_cast<int>(idx % N);
    const int i = row0 + static_cast<int>(idx / N);
    int cnt = 0;
    for (int w = 0; w < nw; ++w) cnt += __popc(bits[w * N + i] & bits[w * N + j]);
    scale[idx] = 1.0f / (fS * (static_cast<float>(cnt) + eps));
  }
}

// ------------------------------------------------------------------------------------------------
// Tied ("global") queries of the extra-MSA stack (alphafold2.py:142-151): q[b'][i][:] <- mean over the folded batch b' of
// q[b'][i][:] (plain mean, the mask plays no role), written back over every b'.  buf row of token(b', i) = b'*tok_sb + i*tok_si
// has ld elements; the first `cols` of them are the (already scaled) queries.  T = float (strict mode) or bf16.
// ------------------------------------------------------------------------------------------------
template <class T> __device__ __forceinline__ float tie_ld(const T* p);
template <> __device__ __forceinline__ float tie_ld<float>(const float* p) { return *p; }
template <> __device__ __forceinline__ float tie_ld<__nv_bfloat16>(const __nv_bfloat16* p) { return __bfloat162float(*p); }
template <class T> __device__ __forceinline__ void tie_st(T* p, float v);
template <> __device__ __forceinline__ void tie_st<float>(float* p, float v) { *p = v; }
template <> __device__ __forceinline__ void tie_st<__nv_bfloat16>(__nv_bfloat16* p, float v) { *p = __float2bfloat16(v); }

template <class T>
__global__ void __launch_bounds__(256) tie_queries_kernel(T* __restrict__ buf, long long ld, int cols, int n, int nbatch,
                                                          long long tok_sb, long long tok_si) {
  const long long total = static_cast<long long>(n) * cols;
  for (long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; idx < total;
       idx += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int c = static_cast<int>(idx % cols);
    const long long i = idx / cols;
    T* base = buf + i * tok_si * ld + c;
    float acc = 0.f;
    for (int b = 0; b < nbatch; ++b) acc += tie_ld<T>(base + b * tok_sb * ld);
    const float mean = acc / static_cast<float>(nbatch);
    for (int b = 0; b < nbatch; ++b) tie_st<T>(base + b * tok_sb * ld, mean);
  }
}

// EXPERIMENT (AF2_ATTN_HEADMAJOR=1): token-major q|k|v [T][3I] -> head-major [3H][T][dh], so that the 128-row K / V / Q boxes
// of the attention kernel are 16 KB of contiguous memory instead of 128 pieces of 128 B at a 3 KB stride
__global__ void __launch_bounds__(256) qkv_to_headmajor_kernel(const uint4* __restrict__ in, uint4* __restrict__ out, long long T, int I3, int dh) {
  const int c8n = I3 >> 3, d8 = dh >> 3;
  const long long total = T * c8n;
  for (long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; idx < total;
       idx += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long t = idx / c8n;
    const int c8 = static_cast<int>(idx - t * c8n);
    const int hc = c8 / d8, e8 = c8 - hc * d8;
    out[(static_cast<long long>(hc) * T + t) * d8 + e8] = in[idx];
  }
}

// bool mask -> float 0/1 row scale
__global__ void mask_to_float_kernel(const uint8_t* __restrict__ mask, float* __restrict__ out, long long n) {
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x)
    out[i] = mask[i] ? 1.0f : 0.0f;
}

// ------------------------------------------------------------------------------------------------
// apply_rotary_pos_emb (rotary.py:9-20): x [b, h, n, dh] fp32; sin/cos [bs, n, rot] (bs = 1 or b).
// Interleaved pairs (x0, x1) -> (x0 c0 - x1 s0, x1 c1 + x0 s1); channels >= rot pass through.
// ------------------------------------------------------------------------------------------------
__global__ void rotary_kernel(const float* __restrict__ x, const float* __restrict__ sn, const float* __restrict__ cs,
                              float* __restrict__ y, int b, int h, int n, int dh, int rot, int sincos_batch) {
  const long long pairs = static_cast<long long>(b) * h * n * (dh / 2);
  for (long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; idx < pairs;
       idx += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int pr = idx % (dh / 2);
    const long long row = idx / (dh / 2);      // (b, h, n) flattened
    const int ni = row % n;
    const int bi = row / (static_cast<long long>(n) * h);
    const float2 v = reinterpret_cast<const float2*>(x)[idx];
    float2 o = v;
    if (2 * pr + 1 < rot) {
      const long long so = (static_cast<long long>(sincos_batch > 1 ? bi : 0) * n + ni) * rot + 2 * pr;
      const float s0 = sn[so], s1 = sn[so + 1], c0 = cs[so], c1 = cs[so + 1];
      // separate roundings (no FMA contraction) so the result is bit-identical to x*cos + rot(x)*sin
      o.x = __fadd_rn(__fmul_rn(v.x, c0), __fmul_rn(-v.y, s0));
      o.y = __fadd_rn(__fmul_rn(v.y, c1), __fmul_rn(v.x, s1));
    }
    reinterpret_cast<float2*>(y)[idx] = o;
  }
}

}  // namespace af2
