// Pre- / post-trunk glue of Alphafold2.forward as fused kernels (SURVEY.md 8f row n1):
//   alphafold2.py:676-726  token embedding gather, MSA = emb[msa] (+ msa_embed) + emb[seq], pair init
//                          x[i][j] = left[i] + right[j] + pos_emb[clamp(idx_i - idx_j)]            (all fp32, HBM-write bound)
//   alphafold2.py:821-823  trunk_embeds = (x + x^T) / 2 -> LayerNorm -> Linear(d -> 37 buckets)   (HBM-read bound)
// Everything here is fp32 with the reference's operation order (sums are not re-associated), so the results differ from
// the eager PyTorch glue only by the summation order inside the two small dot products.
#pragma once
#include "common.cuh"
#include "simt_kernels.cuh"

namespace af2 {

// e[b][i][:] = token_emb[seq[b][i]] (+ seq_embed);   lr[b][i][0:2d] = to_pairwise_repr(e)  (W [2d][d], bias [2d])
// one block (256 threads) per token; d <= 1024
__global__ void __launch_bounds__(256) glue_seq_kernel(const long long* __restrict__ seq, const float* __restrict__ emb,
                                                       const float* __restrict__ seq_embed, const float* __restrict__ W,
                                                       const float* __restrict__ bias, float* __restrict__ e, float* __restrict__ lr,
                                                       int d, int vocab) {
  extern __shared__ float ev[];        // [d]
  const long long t = blockIdx.x;
  long long tok = seq[t];
  tok = tok < 0 ? 0 : (tok >= vocab ? vocab - 1 : tok);      // (torch would raise on an out-of-range id; never happens for valid inputs)
  for (int c = threadIdx.x; c < d; c += blockDim.x) {
    float v = emb[tok * d + c];
    if (seq_embed) v += seq_embed[t * d + c];
    ev[c] = v;
    e[t * d + c] = v;
  }
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int o = warp; o < 2 * d; o += 8) {                     // one warp per output: coalesced reads of W[o][:]
    const float* wr = W + static_cast<long long>(o) * d;
    float acc = 0.f;
    for (int c = lane; c < d; c += 32) acc = fmaf(ev[c], wr[c], acc);
    acc = warp_sum(acc);
    if (lane == 0) lr[t * 2 * d + o] = acc + bias[o];
  }
}

// m[b][s][j][:] = (token_emb[msa[b][s][j]] (+ msa_embed)) + e[b][j][:]        float4 per thread
__global__ void __launch_bounds__(256) glue_msa_init_kernel(const long long* __restrict__ msa, const float* __restrict__ emb,
                                                            const float* __restrict__ msa_embed, const float* __restrict__ e,
                                                            float* __restrict__ m, long long tokens, int S, int n, int d, int vocab) {
  const int d4 = d >> 2;
  const long long total = tokens * d4;
  for (long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; idx < total;
       idx += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long t = idx / d4;
    const int c4 = static_cast<int>(idx - t * d4);
    const int j = static_cast<int>(t % n);
    const long long b = t / (static_cast<long long>(S) * n);
    long long tok = msa[t];
    tok = tok < 0 ? 0 : (tok >= vocab ? vocab - 1 : tok);
    float4 v = reinterpret_cast<const float4*>(emb + tok * d)[c4];
    if (msa_embed) {
      const float4 a = reinterpret_cast<const float4*>(msa_embed + t * d)[c4];
      v.x += a.x; v.y += a.y; v.z += a.z; v.w += a.w;
    }
    const float4 ee = reinterpret_cast<const float4*>(e + (b * n + j) * d)[c4];
    v.x += ee.x; v.y += ee.y; v.z += ee.z; v.w += ee.w;
    reinterpret_cast<float4*>(m + t * d)[c4] = v;
  }
}

// x[b][i - row0][j][:] = (left[b][i] + right[b][j]) + pos_emb[clamp(idx[i] - idx[j], -R, R) + R]   for i in [row0, row0 + rows)
// (x [B][rows][n][d]; the whole tensor is row0 = 0, rows = n)
__global__ void __launch_bounds__(256) glue_pair_init_kernel(const float* __restrict__ lr, const float* __restrict__ pos,
                                                             const long long* __restrict__ seq_index, float* __restrict__ x,
                                                             int B, int n, int d, int R, int row0, int rows) {
  const int d4 = d >> 2;
  const long long total = static_cast<long long>(B) * rows * n * d4;
  for (long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; idx < total;
       idx += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int c4 = static_cast<int>(idx % d4);
    const long long t = idx / d4;
    const int j = static_cast<int>(t % n);
    const int i = row0 + static_cast<int>((t / n) % rows);
    const long long b = t / (static_cast<long long>(rows) * n);
    const float4 l = reinterpret_cast<const float4*>(lr + (b * n + i) * 2 * d)[c4];
    const float4 r = reinterpret_cast<const float4*>(lr + (b * n + j) * 2 * d + d)[c4];
    long long rel = seq_index ? (seq_index[i] - seq_index[j]) : static_cast<long long>(i - j);
    rel = rel < -R ? -R : (rel > R ? R : rel);
    const float4 p = reinterpret_cast<const float4*>(pos + (rel + R) * d)[c4];
    float4 o;
    o.x = (l.x + r.x) + p.x; o.y = (l.y + r.y) + p.y; o.z = (l.z + r.z) + p.z; o.w = (l.w + r.w) + p.w;
    reinterpret_cast<float4*>(x + t * d)[c4] = o;
  }
}

// distogram head: out[b][i][j][0:nb] = Linear_{d -> nb}( LayerNorm( (x[b][i][j] + xt[b][j][i]) * 0.5 ) )
// x [B][rows][n][D], xt [B][n][ldt][D]: the whole tensor is xt = x, rows = ldt = n; a row shard i in [row0, row0 + rows) reads
// x = its rows and xt = its column shard [n][rows][D] (xt[j][i - row0] = x_whole[j][i]), ldt = rows.
// one warp per token, d = 32 * VPL channels; lane owns the float4 chunks lane, lane + 32, ... of the row (coalesced global
// loads, conflict-free shared-memory reads of W); W staged in smem
template <int VPL>
__global__ void __launch_bounds__(256) glue_distogram_kernel(const float* __restrict__ x, const float* __restrict__ xt, long long ldt,
                                                             const float* __restrict__ gamma,
                                                             const float* __restrict__ beta, const float* __restrict__ W,
                                                             const float* __restrict__ bias, float* __restrict__ out,
                                                             int B, int rows, int n, int nb, float eps) {
  constexpr int D = 32 * VPL;
  extern __shared__ float ws[];                 // [nb][D] + [nb] bias
  for (int i = threadIdx.x; i < nb * D; i += blockDim.x) ws[i] = W[i];
  for (int i = threadIdx.x; i < nb; i += blockDim.x) ws[nb * D + i] = bias[i];
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const long long warp_global = static_cast<long long>(blockIdx.x) * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const long long nwarps = static_cast<long long>(gridDim.x) * (blockDim.x >> 5);
  const long long T = static_cast<long long>(B) * rows * n;
  float g[VPL], be[VPL];
#pragma unroll
  for (int k = 0; k < VPL; ++k) { g[k] = gamma[(lane + 32 * (k >> 2)) * 4 + (k & 3)]; be[k] = beta[(lane + 32 * (k >> 2)) * 4 + (k & 3)]; }
  for (long long t = warp_global; t < T; t += nwarps) {
    const int j = static_cast<int>(t % n);
    const int i = static_cast<int>((t / n) % rows);
    const long long b = t / (static_cast<long long>(rows) * n);
    const float* xa = x + t * D + lane * 4;
    const float* xb = xt + ((b * n + j) * ldt + i) * D + lane * 4;
    float v[VPL];
    float s = 0.f;
#pragma unroll
    for (int k = 0; k < VPL; k += 4) {
      const float4 a = *reinterpret_cast<const float4*>(xa + k * 32), c = *reinterpret_cast<const float4*>(xb + k * 32);
      v[k] = (a.x + c.x) * 0.5f; v[k + 1] = (a.y + c.y) * 0.5f; v[k + 2] = (a.z + c.z) * 0.5f; v[k + 3] = (a.w + c.w) * 0.5f;
      s += v[k] + v[k + 1] + v[k + 2] + v[k + 3];
    }
    const float mean = warp_sum(s) * (1.0f / D);
    float q = 0.f;
#pragma unroll
    for (int k = 0; k < VPL; ++k) { const float a = v[k] - mean; q += a * a; }
    const float rstd = rsqrtf(warp_sum(q) * (1.0f / D) + eps);
#pragma unroll
    for (int k = 0; k < VPL; ++k) v[k] = (v[k] - mean) * rstd * g[k] + be[k];
    float res = 0.f;                            // lane o (and o + 32) ends up holding output o
    for (int o0 = 0; o0 < nb; o0 += 32) {
      float mine = 0.f;
      const int no = min(32, nb - o0);
      for (int o = 0; o < no; ++o) {
        const float* wr = ws + (o0 + o) * D + lane * 4;
        float acc = 0.f;
#pragma unroll
        for (int k = 0; k < VPL; k += 4) {
          const float4 w4 = *reinterpret_cast<const float4*>(wr + k * 32);
          acc = fmaf(v[k], w4.x, acc); acc = fmaf(v[k + 1], w4.y, acc); acc = fmaf(v[k + 2], w4.z, acc); acc = fmaf(v[k + 3], w4.w, acc);
        }
        acc = warp_sum(acc);
        if (lane == o) mine = acc;
      }
      res = mine;
      if (lane < no) out[t * nb + o0 + lane] = res + ws[nb * D + o0 + lane];
    }
  }
}

// recycling embedder (alphafold2.py:730-739), in place, one warp per token of one grid:
//   pair tokens t < B rows n, t = (b, i - row0, j), i in [row0, row0 + rows) (x and p [B][rows][n][d]; the whole tensor is
//   row0 = 0, rows = n):                   x[t] = (x[t] + LN_pair(p[t])) + table[bucket(|coords[b][i] - coords[b][j]|)]
//   MSA-row tokens (b, j) after them:      m[b][0][j] = m[b][0][j] + LN_msa(s[b][j])   (m's batch stride m_bstride elements)
// LayerNorm is fp32 and two-pass (mean, then the centred biased variance), 1 / sqrtf (IEEE).  The distance is the direct one:
// coordinate differences in fp32, squares summed by fmaf over the c coordinates in order, IEEE sqrtf.  bucket = lower bound of
// the distance in bnd[0 .. nb-2] under !(bnd >= v) (torch.bucketize, right=False): NaN -> nb - 1, nb == 1 -> 0.
// Lane owns the float4 chunks lane, lane + 32, ... (NCH of them, d4 = d / 4 <= 32 NCH); every row 16-byte aligned.

// The bucket of the distance between points ci and cj [c] (fp32, global memory) under the edges bnd[0 .. nb-2], as the
// recycling embedder decides it; also the label of the distogram loss (distogram_loss.cuh), which must agree with it bit for bit.
__device__ __forceinline__ int distance_bucket(const float* __restrict__ ci, const float* __restrict__ cj, int c,
                                               const float* __restrict__ bnd, int nb) {
  float s2 = 0.f;
  for (int e = 0; e < c; ++e) { const float dl = __ldg(ci + e) - __ldg(cj + e); s2 = fmaf(dl, dl, s2); }
  const float dist = sqrtf(s2);
  int lo = 0, hi = nb - 1;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (!(__ldg(bnd + mid) >= dist)) lo = mid + 1; else hi = mid;
  }
  return lo;
}

template <int NCH>
__device__ __forceinline__ void recycle_ln_row(const float* __restrict__ src, const float* __restrict__ g, const float* __restrict__ be,
                                               int d, int lane, float eps, float (&y)[4 * NCH]) {
  const int d4 = d >> 2;
  float s = 0.f;
#pragma unroll
  for (int k = 0; k < NCH; ++k) {
    const int c4 = lane + 32 * k;
    float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
    if (c4 < d4) a = __ldcs(reinterpret_cast<const float4*>(src) + c4);
    y[4 * k] = a.x; y[4 * k + 1] = a.y; y[4 * k + 2] = a.z; y[4 * k + 3] = a.w;
    s += (a.x + a.y) + (a.z + a.w);
  }
  const float mean = warp_sum(s) / static_cast<float>(d);
  float q = 0.f;
#pragma unroll
  for (int k = 0; k < NCH; ++k) {
    if (lane + 32 * k < d4) {
#pragma unroll
      for (int e = 0; e < 4; ++e) { const float a = y[4 * k + e] - mean; q = fmaf(a, a, q); }
    }
  }
  const float rstd = 1.0f / sqrtf(warp_sum(q) / static_cast<float>(d) + eps);
#pragma unroll
  for (int k = 0; k < NCH; ++k) {
    const int c4 = lane + 32 * k;
    if (c4 < d4) {
      const float4 g4 = __ldg(reinterpret_cast<const float4*>(g) + c4), b4 = __ldg(reinterpret_cast<const float4*>(be) + c4);
      y[4 * k] = fmaf((y[4 * k] - mean) * rstd, g4.x, b4.x);
      y[4 * k + 1] = fmaf((y[4 * k + 1] - mean) * rstd, g4.y, b4.y);
      y[4 * k + 2] = fmaf((y[4 * k + 2] - mean) * rstd, g4.z, b4.z);
      y[4 * k + 3] = fmaf((y[4 * k + 3] - mean) * rstd, g4.w, b4.w);
    }
  }
}

template <int NCH>
__global__ void __launch_bounds__(256) glue_recycle_kernel(const float* __restrict__ coords, int c, const float* __restrict__ srow,
                                                           const float* __restrict__ pprev, const float* __restrict__ msa_g,
                                                           const float* __restrict__ msa_b, const float* __restrict__ pair_g,
                                                           const float* __restrict__ pair_b, const float* __restrict__ table,
                                                           const float* __restrict__ bnd, int nb, float* __restrict__ x,
                                                           float* __restrict__ m, long long m_bstride, int B, int n, int d, float eps,
                                                           int row0, int rows) {
  const int lane = threadIdx.x & 31;
  const int d4 = d >> 2;
  const long long warp_global = static_cast<long long>(blockIdx.x) * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const long long nwarps = static_cast<long long>(gridDim.x) * (blockDim.x >> 5);
  const long long T1 = static_cast<long long>(B) * rows * n;
  const long long T = T1 + static_cast<long long>(B) * n;
  float y[4 * NCH];
  for (long long t = warp_global; t < T; t += nwarps) {
    if (t < T1) {
      const int j = static_cast<int>(t % n);
      const int i = row0 + static_cast<int>((t / n) % rows);
      const long long b = t / (static_cast<long long>(rows) * n);
      float4 xv[NCH];
#pragma unroll
      for (int k = 0; k < NCH; ++k)
        if (lane + 32 * k < d4) xv[k] = reinterpret_cast<const float4*>(x + t * d)[lane + 32 * k];
      recycle_ln_row<NCH>(pprev + t * d, pair_g, pair_b, d, lane, eps, y);
      const int lo = distance_bucket(coords + (b * n + i) * c, coords + (b * n + j) * c, c, bnd, nb);
      const float4* er = reinterpret_cast<const float4*>(table + static_cast<long long>(lo) * d);
#pragma unroll
      for (int k = 0; k < NCH; ++k) {
        const int c4 = lane + 32 * k;
        if (c4 < d4) {
          const float4 e4 = __ldg(er + c4);
          float4 o;
          o.x = (xv[k].x + y[4 * k]) + e4.x; o.y = (xv[k].y + y[4 * k + 1]) + e4.y;
          o.z = (xv[k].z + y[4 * k + 2]) + e4.z; o.w = (xv[k].w + y[4 * k + 3]) + e4.w;
          reinterpret_cast<float4*>(x + t * d)[c4] = o;
        }
      }
    } else {
      const long long r = t - T1;                  // (b, j)
      const long long b = r / n;
      const int j = static_cast<int>(r - b * n);
      recycle_ln_row<NCH>(srow + r * d, msa_g, msa_b, d, lane, eps, y);
      float4* mr = reinterpret_cast<float4*>(m + b * m_bstride + static_cast<long long>(j) * d);
#pragma unroll
      for (int k = 0; k < NCH; ++k) {
        const int c4 = lane + 32 * k;
        if (c4 < d4) {
          float4 o = mr[c4];
          o.x += y[4 * k]; o.y += y[4 * k + 1]; o.z += y[4 * k + 2]; o.w += y[4 * k + 3];
          mr[c4] = o;
        }
      }
    }
  }
}

}  // namespace af2
