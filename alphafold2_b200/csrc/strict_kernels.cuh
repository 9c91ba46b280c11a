// SIMT kernels of the STRICT precision mode (alphafold2_b200.set_precision(model, "strict")).
//
// Strict mode keeps every activation in fp32 between kernels and feeds the wgmma GEMM (gemm_tc.cuh, GemmParams::nseg = 6)
// with SPLIT-bf16 operands: v = p0 + p1 + p2 with p0 = bf16(v), p1 = bf16(v - p0), p2 = bf16(v - p0 - p1) (24 mantissa bits),
// and the six products p0*p2 + p2*p0 + p1*p1 + p0*p1 + p1*p0 + p0*p0 accumulated in fp32 (everything below 2^-24 relative is
// dropped), so the trunk output matches the reference's fp32 path inside the north star's rtol 1e-3 / atol 1e-4 band even
// after 12 blocks (two planes / three products leave 2^-17 per operand: 99.994 % of the C2 depth-12 elements in band,
// measured; the default mode's bf16 operands cannot come close: SURVEY.md Appendix B).  The kernels here do the
// fp32 element-wise work around those GEMMs (LayerNorm, GEGLU, gates, masks, softmax, layout changes) with exact-grade
// math (erff / expf, fp32 statistics) and write the split planes.  Throughput is secondary in this mode.
//
// Split layouts (SPL = 3 planes, P = align8(K) so that every plane row is 16-byte aligned for TMA):
//   token-major   [rows][SPL][P]               row stride SPL * P, plane stride P
//   channel-major, k contiguous (K-major)      [c][rows][SPL][P]
//   channel-major, mn contiguous (MN-major)    [c][SPL][k][P]
#pragma once
#include "common.cuh"
#include "simt_kernels.cuh"

namespace af2 {

constexpr int SPL = 3;        // bf16 planes per split operand
constexpr int SPL_NSEG = 6;   // tensor-core passes over K (GemmParams::nseg)

// p[0], p[ps], p[2 ps] <- the three bf16 planes of v (the subtractions are exact in fp32)
__device__ __forceinline__ void split_store(__nv_bfloat16* p, long long ps, float v) {
  const __nv_bfloat16 h0 = __float2bfloat16(v);
  const float r1 = v - __bfloat162float(h0);
  const __nv_bfloat16 h1 = __float2bfloat16(r1);
  const float r2 = r1 - __bfloat162float(h1);
  p[0] = h0;
  p[ps] = h1;
  p[2 * ps] = __float2bfloat16(r2);
}
__device__ __forceinline__ float sigmoid_acc(float x) { return 1.0f / (1.0f + expf(-x)); }
__device__ __forceinline__ float gelu_acc(float x) { return 0.5f * x * (1.0f + erff(x * 0.70710678118654752f)); }

// ------------------------------------------------------------------------------------------------
// y = LayerNorm(x) * gamma + beta (or y = x when gamma == nullptr) -> split token-major [T][SPL][P]; one warp per row.
// Two-pass statistics in fp32 exactly like nn.LayerNorm (biased variance, eps inside the sqrt).  Pad columns [d, P) zeroed.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) strict_ln_split_kernel(const float* __restrict__ x, const float* __restrict__ gamma,
                                                              const float* __restrict__ beta, __nv_bfloat16* __restrict__ y,
                                                              long long T, int d, int P, float eps) {
  const int lane = threadIdx.x & 31;
  const long long warp_global = static_cast<long long>(blockIdx.x) * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const long long nwarps = static_cast<long long>(gridDim.x) * (blockDim.x >> 5);
  for (long long t = warp_global; t < T; t += nwarps) {
    const float* xr = x + t * d;
    float mean = 0.f, rstd = 1.f;
    if (gamma) {
      float s = 0.f;
      for (int c = lane; c < d; c += 32) s += xr[c];
      mean = warp_sum(s) / d;
      float q = 0.f;
      for (int c = lane; c < d; c += 32) {
        const float a = xr[c] - mean;
        q += a * a;
      }
      rstd = rsqrtf(warp_sum(q) / d + eps);
    }
    __nv_bfloat16* yr = y + t * SPL * P;
    for (int c = lane; c < P; c += 32) {
      float v = 0.f;
      if (c < d) v = gamma ? (xr[c] - mean) * rstd * gamma[c] + beta[c] : xr[c];
      split_store(yr + c, P, v);
    }
  }
}

// ------------------------------------------------------------------------------------------------
// GEGLU (alphafold2.py:69-72): h [T][2*hid] = (a | g) fp32 -> a * gelu_erf(g) -> split [T][SPL][P]
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) strict_geglu_split_kernel(const float* __restrict__ h, __nv_bfloat16* __restrict__ y,
                                                                 long long T, int hid, int P) {
  const long long total = T * P;
  for (long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; idx < total;
       idx += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long t = idx / P;
    const int c = static_cast<int>(idx - t * P);
    float v = 0.f;
    if (c < hid) v = h[t * 2 * hid + c] * gelu_acc(h[t * 2 * hid + hid + c]);
    split_store(y + t * SPL * P + c, P, v);
  }
}

// ------------------------------------------------------------------------------------------------
// attention operands from the fused projection P1 [T][4I] = (q | k | v | gate logits), fp32:
//   Q, K : split [bh][n][SPL][Pd]     (q already carries dim_head^-0.5 through the packed weight)
//   Vt   : split [bh][dh][SPL][Pn]    (V transposed: row = feature e, column = key j) so that P V is a K-major GEMM
// bh = b' * H + h;  token(b', i) = b' * tok_sb + i * tok_si  (row / column fold of AxialAttention, alphafold2.py:228-240)
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) strict_qkv_split_kernel(const float* __restrict__ p1, __nv_bfloat16* __restrict__ Q,
                                                               __nv_bfloat16* __restrict__ K, __nv_bfloat16* __restrict__ Vt,
                                                               int b0, int nb, int H, int n, int dh, int Pd, int Pn,
                                                               long long tok_sb, long long tok_si) {
  const int I = H * dh;
  const long long ld = 4LL * I;
  // q / k: thread per (bh, i, e in [0, Pd))
  const long long tot_qk = static_cast<long long>(nb) * H * n * Pd;
  for (long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; idx < tot_qk;
       idx += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int e = static_cast<int>(idx % Pd);
    const long long r = idx / Pd;
    const int i = static_cast<int>(r % n);
    const long long bh = r / n;
    const int h = static_cast<int>(bh % H);
    const long long bl = bh / H;
    const long long tok = (b0 + bl) * tok_sb + i * tok_si;
    float qv = 0.f, kv = 0.f;
    if (e < dh) {
      qv = p1[tok * ld + h * dh + e];
      kv = p1[tok * ld + I + h * dh + e];
    }
    const long long o = (bh * n + i) * SPL * Pd + e;
    split_store(Q + o, Pd, qv);
    split_store(K + o, Pd, kv);
  }
  // v transposed: thread per (bh, e, j in [0, Pn))
  const long long tot_v = static_cast<long long>(nb) * H * dh * Pn;
  for (long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; idx < tot_v;
       idx += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int j = static_cast<int>(idx % Pn);
    const long long r = idx / Pn;
    const int e = static_cast<int>(r % dh);
    const long long bh = r / dh;
    const int h = static_cast<int>(bh % H);
    const long long bl = bh / H;
    float v = 0.f;
    if (j < n) v = p1[((b0 + bl) * tok_sb + j * tok_si) * ld + 2 * I + h * dh + e];
    const long long o = (bh * dh + e) * SPL * Pn + j;
    split_store(Vt + o, Pn, v);
  }
}

// ------------------------------------------------------------------------------------------------
// pair bias in fp32 (alphafold2.py:214-217, 245-247): bias[h][t] = <x_raw[t, :], w_edge[h, :]>; one warp per token
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) strict_pair_bias_kernel(const float* __restrict__ x, const float* __restrict__ wb,
                                                               float* __restrict__ bias, long long T, int d, int H) {
  const int lane = threadIdx.x & 31;
  const long long warp_global = static_cast<long long>(blockIdx.x) * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const long long nwarps = static_cast<long long>(gridDim.x) * (blockDim.x >> 5);
  for (long long t = warp_global; t < T; t += nwarps) {
    const float* xr = x + t * d;
    for (int h = 0; h < H; ++h) {
      float acc = 0.f;
      for (int c = lane; c < d; c += 32) acc = fmaf(xr[c], wb[h * d + c], acc);
      acc = warp_sum(acc);
      if (lane == 0) bias[static_cast<long long>(h) * T + t] = acc;
    }
  }
}

// ------------------------------------------------------------------------------------------------
// softmax rows of the logits S [bh][n][lds] (fp32, = q k^T) -> P split [bh][n][SPL][Pn]; one warp per (bh, i).
//   logits += bias[h][i][j] (fp32 [H][n][n]);  mask semantics of alphafold2.py:162-167 (quirk Q1): where
//   !(mask[q] & mask[k]) the logit is REPLACED by -FLT_MAX, so a masked query row is uniform over all n keys.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) strict_softmax_split_kernel(const float* __restrict__ S, long long lds,
                                                                   const float* __restrict__ bias, const uint8_t* __restrict__ mask,
                                                                   __nv_bfloat16* __restrict__ P, int b0, int nb, int H, int n, int Pn,
                                                                   long long mask_sb, long long mask_si) {
  const int lane = threadIdx.x & 31;
  const long long warp_global = static_cast<long long>(blockIdx.x) * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const long long nwarps = static_cast<long long>(gridDim.x) * (blockDim.x >> 5);
  const long long rows = static_cast<long long>(nb) * H * n;
  const float NEG = -3.402823466e+38f;
  for (long long r = warp_global; r < rows; r += nwarps) {
    const int i = static_cast<int>(r % n);
    const long long bh = r / n;
    const int h = static_cast<int>(bh % H);
    const long long bl = bh / H;
    const float* sr = S + r * lds;
    const float* br = bias ? bias + (static_cast<long long>(h) * n + i) * n : nullptr;
    const uint8_t* mb = mask ? mask + (b0 + bl) * mask_sb : nullptr;
    const bool qok = mb ? mb[i * mask_si] != 0 : true;
    auto logit = [&](int j) {
      float v = sr[j];
      if (br) v += br[j];
      if (mb && !(qok && mb[j * mask_si] != 0)) v = NEG;
      return v;
    };
    float mx = NEG;
    for (int j = lane; j < n; j += 32) mx = fmaxf(mx, logit(j));
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    float sum = 0.f;
    for (int j = lane; j < n; j += 32) sum += expf(logit(j) - mx);
    sum = warp_sum(sum);
    const float inv = 1.0f / sum;
    __nv_bfloat16* pr = P + r * SPL * Pn;
    for (int j = lane; j < Pn; j += 32) {
      const float v = j < n ? expf(logit(j) - mx) * inv : 0.f;
      split_store(pr + j, Pn, v);
    }
  }
}

// ------------------------------------------------------------------------------------------------
// attention output * sigmoid(gating) (alphafold2.py:184-185): O [bh][n][dh] fp32, gate logits = P1[:, 3I:4I]
//   -> split token-major [T][SPL][Pi] rows of the tokens of batch elements [b0, b0 + nb)
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) strict_gate_split_kernel(const float* __restrict__ O, long long ldo, const float* __restrict__ p1,
                                                                __nv_bfloat16* __restrict__ og, int b0, int nb, int H, int n, int dh, int Pi,
                                                                long long tok_sb, long long tok_si) {
  const int I = H * dh;
  const long long total = static_cast<long long>(nb) * n * Pi;
  for (long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; idx < total;
       idx += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int c = static_cast<int>(idx % Pi);
    const long long r = idx / Pi;
    const int i = static_cast<int>(r % n);
    const long long bl = r / n;
    const long long tok = (b0 + bl) * tok_sb + i * tok_si;
    float v = 0.f;
    if (c < I) {
      const int h = c / dh, e = c - h * dh;
      v = O[((bl * H + h) * n + i) * ldo + e] * sigmoid_acc(p1[tok * 4LL * I + 3 * I + c]);
    }
    split_store(og + tok * SPL * Pi + c, Pi, v);
  }
}

// ------------------------------------------------------------------------------------------------
// token-major fp32 [T][ld] -> channel-major split operand of a per-channel contraction (32 x 32 smem transpose):
//   value v(t, c) = src[t][val_off + c] * (gate_off >= 0 ? sigmoid(src[t][gate_off + c]) : 1) * (mask ? mask[t] : 1)
//   token t = r * inner + k  (r = row of the channel matrix, k = its column);   element (c, r, k, plane) goes to
//   out[c * cs + plane * hs + r * rs + k]       K-major split:  rs = SPL * P, hs = P;   MN-major split: rs = P, hs = rows * P
// grid = (rows * ceil(inner / 32), ceil(C / 32)), block = 32 x 8
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) strict_tok2chan_split_kernel(const float* __restrict__ src, long long ld, int val_off, int gate_off,
                                                                    const uint8_t* __restrict__ mask, __nv_bfloat16* __restrict__ out,
                                                                    int C, int inner, long long cs, long long hs, long long rs) {
  __shared__ float tile[32][33];
  const int ktiles = (inner + 31) / 32;
  const int r = blockIdx.x / ktiles, k0 = (blockIdx.x % ktiles) * 32, c0 = blockIdx.y * 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  for (int kk = ty; kk < 32; kk += 8) {
    const int k = k0 + kk, c = c0 + tx;
    float v = 0.f;
    if (k < inner && c < C) {
      const long long t = static_cast<long long>(r) * inner + k;
      v = src[t * ld + val_off + c];
      if (gate_off >= 0) v *= sigmoid_acc(src[t * ld + gate_off + c]);
      if (mask && !mask[t]) v = 0.f;
    }
    tile[kk][tx] = v;
  }
  __syncthreads();
  for (int cc = ty; cc < 32; cc += 8) {
    const int c = c0 + cc, k = k0 + tx;
    if (c < C && k < inner) {
      __nv_bfloat16* o = out + static_cast<long long>(c) * cs + static_cast<long long>(r) * rs + k;
      split_store(o, hs, tile[tx][cc]);
    }
  }
}

// ------------------------------------------------------------------------------------------------
// channel-major fp32 contraction output -> split token-major operand of the output projection (strict twin of
// chan_to_token_kernel):   src[c][row * pitch + j],  token = row * n + j
//   mode 0 (alphafold2.py:315-316): LayerNorm_c(src) * gamma + beta, * sigmoid(gate_src[token][gate_off + c])
//   mode 1 (alphafold2.py:345-349): src * (scale ? scale[token] : scale_const)
// grid = (ceil(n / 32), rows), block 256, dyn smem d * 33 floats
// ------------------------------------------------------------------------------------------------
struct StrictC2TParams {
  const float* src; long long chan_stride; int pitch, rows, n, d, P, mode;
  const float* gamma; const float* beta;
  const float* gate_src; long long gate_ld; int gate_off;
  const float* scale; float scale_const, eps;
  __nv_bfloat16* y;
};
__global__ void __launch_bounds__(256) strict_chan_to_token_kernel(const StrictC2TParams p) {
  extern __shared__ float tile[];   // [d][33]
  const int j0 = blockIdx.x * 32, row = blockIdx.y;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const bool j_ok = (j0 + lane) < p.n;
  const float* src = p.src + static_cast<long long>(row) * p.pitch + j0 + lane;
  for (int c = warp; c < p.d; c += 8) tile[c * 33 + lane] = j_ok ? src[c * p.chan_stride] : 0.f;
  __syncthreads();
  for (int tk = warp; tk < 32; tk += 8) {
    if (j0 + tk >= p.n) break;
    const long long token = static_cast<long long>(row) * p.n + j0 + tk;
    __nv_bfloat16* yr = p.y + token * SPL * p.P;
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
      for (int c = lane; c < p.P; c += 32) {
        float o = 0.f;
        if (c < p.d) {
          const float g = sigmoid_acc(p.gate_src[token * p.gate_ld + p.gate_off + c]);
          o = ((tile[c * 33 + tk] - mean) * rstd * p.gamma[c] + p.beta[c]) * g;
        }
        split_store(yr + c, p.P, o);
      }
    } else {
      const float sc = p.scale ? p.scale[token] : p.scale_const;
      for (int c = lane; c < p.P; c += 32) split_store(yr + c, p.P, c < p.d ? tile[c * 33 + tk] * sc : 0.f);
    }
  }
}

}  // namespace af2
