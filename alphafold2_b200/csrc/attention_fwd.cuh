// Element-wise kernels of Attention.forward (alphafold2.py:125-190) called on its own: queries from x [B][i][d], keys and
// values from a context [B][j][d] (or x), a query mask [B][i] and a key mask [B][j], and an additive bias given as an fp32
// tensor with arbitrary strides (any shape that broadcasts to [B][heads][i][j]).  The attention itself runs in
// attention_tc_kernel<DH, true> (bf16 mode) or as split-bf16 GEMMs around the strict kernels below.
#pragma once
#include "common.cuh"
#include "strict_kernels.cuh"

namespace af2 {

// fp32 bias of attention_tc_kernel<DH, true>: out [Bb][H][nq][npad] = log2(e) * bias[b sb + h sh + i si + j sj] (the kernel's
// softmax is exp2 based), pad columns j >= nk zero
__global__ void __launch_bounds__(256) attn_bias_log2_kernel(const float* __restrict__ bias, long long sb, long long sh, long long si,
                                                             long long sj, float* __restrict__ out, int Bb, int H, int nq, int nk,
                                                             int npad) {
  const long long total = static_cast<long long>(Bb) * H * nq * npad;
  for (long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; idx < total;
       idx += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int j = static_cast<int>(idx % npad);
    const long long r = idx / npad;
    const int i = static_cast<int>(r % nq);
    const long long bh = r / nq;
    const int h = static_cast<int>(bh % H);
    const long long b = bh / H;
    out[idx] = j < nk ? bias[b * sb + h * sh + i * si + j * sj] * 1.4426950408889634f : 0.f;
  }
}

// ------------------------------------------------------------------------------------------------
// strict mode, batch elements [b0, b0 + nb):
//   Q  split [bh][nq][SPL][Pd] from qg [B nq][2I] (columns [0, I): q * dim_head^-0.5)
//   K  split [bh][nk][SPL][Pd] and Vt split [bh][dh][SPL][Pn] from kv [B nk][2I] (k | v)
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) strict_xqkv_split_kernel(const float* __restrict__ qg, const float* __restrict__ kv,
                                                                __nv_bfloat16* __restrict__ Q, __nv_bfloat16* __restrict__ K,
                                                                __nv_bfloat16* __restrict__ Vt, int b0, int nb, int H, int nq, int nk,
                                                                int dh, int Pd, int Pn) {
  const int I = H * dh;
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  const long long start = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  // q: thread per (bh, i, e in [0, Pd))
  for (long long idx = start; idx < static_cast<long long>(nb) * H * nq * Pd; idx += stride) {
    const int e = static_cast<int>(idx % Pd);
    const long long r = idx / Pd;
    const int i = static_cast<int>(r % nq);
    const long long bh = r / nq;
    const int h = static_cast<int>(bh % H);
    const long long b = b0 + bh / H;
    split_store(Q + r * SPL * Pd + e, Pd, e < dh ? qg[(b * nq + i) * 2LL * I + h * dh + e] : 0.f);
  }
  // k: thread per (bh, j, e in [0, Pd))
  for (long long idx = start; idx < static_cast<long long>(nb) * H * nk * Pd; idx += stride) {
    const int e = static_cast<int>(idx % Pd);
    const long long r = idx / Pd;
    const int j = static_cast<int>(r % nk);
    const long long bh = r / nk;
    const int h = static_cast<int>(bh % H);
    const long long b = b0 + bh / H;
    split_store(K + r * SPL * Pd + e, Pd, e < dh ? kv[(b * nk + j) * 2LL * I + h * dh + e] : 0.f);
  }
  // v transposed: thread per (bh, e, j in [0, Pn))
  for (long long idx = start; idx < static_cast<long long>(nb) * H * dh * Pn; idx += stride) {
    const int j = static_cast<int>(idx % Pn);
    const long long r = idx / Pn;
    const int e = static_cast<int>(r % dh);
    const long long bh = r / dh;
    const int h = static_cast<int>(bh % H);
    const long long b = b0 + bh / H;
    split_store(Vt + r * SPL * Pn + j, Pn, j < nk ? kv[(b * nk + j) * 2LL * I + I + h * dh + e] : 0.f);
  }
}

// softmax rows of the logits S [bh][nq][lds] -> P split [bh][nq][SPL][Pn]; one warp per (bh, i).  logits += bias (fp32,
// natural-log domain, element (b, h, i, j) at bias[b sb + h sh + i si + j sj]); then, when qmask is given, logits where
// !(qmask[b][i] & (kmask ? kmask[b][j] : 1)) are REPLACED by -FLT_MAX (alphafold2.py:162-167, quirk Q1)
__global__ void __launch_bounds__(256) strict_xsoftmax_split_kernel(const float* __restrict__ S, long long lds,
                                                                    const float* __restrict__ bias, long long sb, long long sh, long long si,
                                                                    long long sj, const uint8_t* __restrict__ qmask,
                                                                    const uint8_t* __restrict__ kmask, __nv_bfloat16* __restrict__ P,
                                                                    int b0, int nb, int H, int nq, int nk, int Pn) {
  const int lane = threadIdx.x & 31;
  const long long warp_global = static_cast<long long>(blockIdx.x) * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const long long nwarps = static_cast<long long>(gridDim.x) * (blockDim.x >> 5);
  const long long rows = static_cast<long long>(nb) * H * nq;
  const float NEG = -3.402823466e+38f;
  for (long long r = warp_global; r < rows; r += nwarps) {
    const int i = static_cast<int>(r % nq);
    const long long bh = r / nq;
    const int h = static_cast<int>(bh % H);
    const long long b = b0 + bh / H;
    const float* sr = S + r * lds;
    const float* br = bias ? bias + b * sb + h * sh + i * si : nullptr;
    const bool qok = qmask ? qmask[b * nq + i] != 0 : true;
    const uint8_t* kr = kmask ? kmask + b * nk : nullptr;
    auto logit = [&](int j) {
      float v = sr[j];
      if (br) v += br[j * sj];
      if (qmask && !(qok && (!kr || kr[j] != 0))) v = NEG;
      return v;
    };
    float mx = NEG;
    for (int j = lane; j < nk; j += 32) mx = fmaxf(mx, logit(j));
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    float sum = 0.f;
    for (int j = lane; j < nk; j += 32) sum += expf(logit(j) - mx);
    sum = warp_sum(sum);
    const float inv = 1.0f / sum;
    __nv_bfloat16* pr = P + r * SPL * Pn;
    for (int j = lane; j < Pn; j += 32) split_store(pr + j, Pn, j < nk ? expf(logit(j) - mx) * inv : 0.f);
  }
}

// og split rows [B nq][SPL][Pi] of batch elements [b0, b0 + nb) = O [bh][nq][dh] * sigmoid(gate logits qg[:, I:2I])
__global__ void __launch_bounds__(256) strict_xgate_split_kernel(const float* __restrict__ O, const float* __restrict__ qg,
                                                                 __nv_bfloat16* __restrict__ og, int b0, int nb, int H, int nq, int dh,
                                                                 int Pi) {
  const int I = H * dh;
  const long long total = static_cast<long long>(nb) * nq * Pi;
  for (long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; idx < total;
       idx += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int c = static_cast<int>(idx % Pi);
    const long long r = idx / Pi;
    const int i = static_cast<int>(r % nq);
    const long long bl = r / nq;
    const long long tok = (b0 + bl) * nq + i;
    float v = 0.f;
    if (c < I) {
      const int h = c / dh, e = c - h * dh;
      v = O[((bl * H + h) * nq + i) * dh + e] * sigmoid_acc(qg[tok * 2LL * I + I + c]);
    }
    split_store(og + tok * SPL * Pi + c, Pi, v);
  }
}

}  // namespace af2
