// Structure module (alphafold2.py:841-891): invariant point attention (the IPABlock of invariant-point-attention 0.2.x) and the
// per-residue frame arithmetic around it.  Everything here is fp32 in both precision modes, as the reference runs it
// (alphafold2.py:854-859 converts to fp32 under torch_default_dtype(float32)).  Points are row vectors: global = local R + t.
//
// Per-residue projection layout (one row of `proj`, width 84 H; the rows of the packed weight in this order):
//   [ q_scalar 16H | k_scalar 16H | v_scalar 16H | q_point 12H | k_point 12H | v_point 12H ],  points (h, p, c)
// to_out input layout (one row of `feat`, width H (32 + d)), the package's concatenation order:
//   [ o_scalar (h 16) | o_point (h p c) | |o_point| (h p) | o_pair (h d) ]
#pragma once
#include "simt_kernels.cuh"      // warp_sum

namespace af2 {

constexpr int IPA_THREADS = 256;
constexpr int IPA_MAX_HEADS = 16;
constexpr int IPA_MAX_BATCH = 65535;     // one CTA row of the grid per batch element: gridDim.y
constexpr int IPA_SD = 16;                 // scalar key / value width per head
constexpr int IPA_PT = 4;                  // point keys / values per head
constexpr int IPA_PROJ = 84;               // projection width per head: 3 * 16 + 3 * 12
constexpr int IPA_VW = IPA_SD + 3 * IPA_PT;  // aggregated values per head: 16 scalars + 12 point coordinates

__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ float softplus_torch(float x) { return x > 20.f ? x : log1pf(expf(x)); }  // F.softplus, threshold 20

// 1-D bulk copy global -> shared (the TMA engine, no tensor map), completion counted on `bar`
__device__ __forceinline__ void bulk_load(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}

// pytorch3d quaternion_to_matrix: scale invariant (q need not be a unit quaternion)
__device__ __forceinline__ void quat_to_matrix(const float q[4], float R[9]) {
  const float r = q[0], i = q[1], j = q[2], k = q[3];
  const float s = 2.f / (r * r + i * i + j * j + k * k);
  R[0] = 1.f - s * (j * j + k * k); R[1] = s * (i * j - k * r);       R[2] = s * (i * k + j * r);
  R[3] = s * (i * j + k * r);       R[4] = 1.f - s * (i * i + k * k); R[5] = s * (j * k - i * r);
  R[6] = s * (i * k - j * r);       R[7] = s * (j * k + i * r);       R[8] = 1.f - s * (i * i + j * j);
}

// ------------------------------------------------------------------------------------------------ fp32 linear
// y[M, N] = act(x[M, K] W^T + b), W [N, K] row-major (nn.Linear).  32 x 32 output tile per CTA, 2 x 2 per thread, K in slices of 16.
// Row tiles on gridDim.x (so up to 2^31 - 1 rows), the few column tiles on gridDim.y.
// The per-residue projections of the structure module: M = b * n rows, small N and K, so small tiles for enough CTAs (64 x 64
// tiles gave 16 CTAs at C2 and measured 39 us per call).
constexpr int SL_BM = 32, SL_BN = 32, SL_BK = 16, SL_R = 2;
constexpr int SL_MAX_N = 65535 * SL_BN;   // column tiles on gridDim.y

__global__ void __launch_bounds__(256) structure_linear_kernel(const float* __restrict__ x, const float* __restrict__ w,
                                                               const float* __restrict__ bias, float* __restrict__ y, int M,
                                                               int N, int K, int relu) {
  __shared__ float xs[SL_BK][SL_BM + 4];
  __shared__ float ws[SL_BK][SL_BN + 4];
  const int tid = threadIdx.x, tx = tid % 16, ty = tid / 16;
  const long long m0 = (long long)blockIdx.x * SL_BM;
  const int n0 = blockIdx.y * SL_BN;
  float acc[SL_R][SL_R] = {};
  for (int k0 = 0; k0 < K; k0 += SL_BK) {
    for (int e = tid; e < SL_BM * SL_BK; e += 256) {
      const int r = e / SL_BK, k = e % SL_BK;
      xs[k][r] = (m0 + r < M && k0 + k < K) ? x[(m0 + r) * K + k0 + k] : 0.f;
      ws[k][r] = (n0 + r < N && k0 + k < K) ? w[(long long)(n0 + r) * K + k0 + k] : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < SL_BK; ++k) {
      float a[SL_R], b[SL_R];
#pragma unroll
      for (int u = 0; u < SL_R; ++u) {
        a[u] = xs[k][ty + 16 * u];
        b[u] = ws[k][tx + 16 * u];
      }
#pragma unroll
      for (int u = 0; u < SL_R; ++u)
#pragma unroll
        for (int v = 0; v < SL_R; ++v) acc[u][v] = fmaf(a[u], b[v], acc[u][v]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int u = 0; u < SL_R; ++u) {
    const long long r = m0 + ty + 16 * u;
    if (r >= M) continue;
#pragma unroll
    for (int v = 0; v < SL_R; ++v) {
      const int c = n0 + tx + 16 * v;
      if (c >= N) continue;
      float o = acc[u][v] + (bias ? bias[c] : 0.f);
      y[r * N + c] = relu ? fmaxf(o, 0.f) : o;
    }
  }
}

// ------------------------------------------------------------------------------------------------ frames
// The q / k / v point projections of every residue taken to the global frame in place: X <- X R_r + t_r.
__global__ void ipa_frames_kernel(float* __restrict__ proj, const float* __restrict__ rot, const float* __restrict__ trans,
                                  long long rows, int heads) {
  const int pts = 3 * IPA_PT * heads;                     // q, k and v points of one residue
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= rows * pts) return;
  const long long r = e / pts;
  float* p = proj + r * (IPA_PROJ * heads) + 3 * IPA_SD * heads + (e % pts) * 3;
  const float* R = rot + r * 9;
  const float* t = trans + r * 3;
  const float x = p[0], y = p[1], z = p[2];
#pragma unroll
  for (int c = 0; c < 3; ++c) p[c] = fmaf(x, R[c], fmaf(y, R[3 + c], fmaf(z, R[6 + c], t[c])));
}

// ------------------------------------------------------------------------------------------------ invariant point attention
// One CTA per query row (b, row0 + i), every head.  The keys stream in tiles of TJ pair rows pair[b, i, j0 : j0 + TJ, :], which are
// contiguous, with the keys' projection rows proj[b, j0 : j0 + TJ, :] beside them: two bulk copies per tile on one mbarrier,
// double buffered.  Per tile, from the one copy of the tile in shared memory:
//   pair bias   (pair_ij . W_h + b_h) / sqrt 3              warp per key row, all heads at once
//   logit       + q_i . k_j / sqrt 48 - softplus(w_h) / (2 sqrt 54) sum_p |Q_ip - K_jp|^2, masked to -FLT_MAX
//   softmax     online, fp32, per head
//   aggregates  o_pair (h d) from the tile, o_scalar and the global o_point from the values of keys j
// The epilogue divides by the softmax sum, takes o_point back to the local frame ((o - t_i) R_i^T), adds its norms and writes
// the row of the to_out input.  Nothing of size n^2 is written.
struct IpaSmem {
  // float offsets into dynamic shared memory; the two mbarriers sit in front
  int tile[2], kv[2], wb, acc, accv, q, logit, stat;
  int floats;
  __host__ __device__ IpaSmem(int H, int d, int TJ) {
    int o = 4;                                           // 16 bytes: two mbarriers
    tile[0] = o; o += TJ * d;
    tile[1] = o; o += TJ * d;
    kv[0] = o; o += TJ * IPA_PROJ * H;
    kv[1] = o; o += TJ * IPA_PROJ * H;
    wb = o; o += H * d;
    acc = o; o += H * d;
    accv = o; o += H * IPA_VW;
    q = o; o += H * (IPA_SD + 3 * IPA_PT);
    logit = o; o += H * TJ;
    stat = o; o += 4 * H;                                 // running max, running sum, rescale, point coefficient
    floats = o;
  }
};

struct IpaParams {
  const float* proj;        // [B n, 84 H], points global
  const float* pair;        // [B, rows, n, d]
  const float* w_bias;      // [H, d]  to_pairwise_attn_bias.0
  const float* b_bias;      // [H]
  const float* point_weights;  // [H] (before the softplus)
  const unsigned char* mask;   // [B, n] or null
  const float* rot;         // [B n, 9]
  const float* trans;       // [B n, 3]
  float* out;               // [B rows, H (32 + d)]
  int n, d, H, TJ;
  int row0, rows;           // the query rows [row0, row0 + rows) of each batch; pair and out hold only these rows
};

__global__ void __launch_bounds__(IPA_THREADS) ipa_attention_kernel(const IpaParams p) {
  extern __shared__ __align__(16) float sm[];
  const IpaSmem L(p.H, p.d, p.TJ);
  uint64_t* bar = reinterpret_cast<uint64_t*>(sm);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int H = p.H, d = p.d, n = p.n, TJ = p.TJ;
  const int i = blockIdx.x, b = blockIdx.y;
  const long long row = (long long)b * n + p.row0 + i;  // the query residue: its projection, mask and frame
  const long long lrow = (long long)b * p.rows + i;     // its pair row and output row
  const int PW = IPA_PROJ * H;
  const float* pair_row = p.pair + lrow * n * d;
  const int ntiles = (n + TJ - 1) / TJ;

  if (tid == 0) {
    mbar_init(&bar[0], 1);
    mbar_init(&bar[1], 1);
    fence_barrier_init();
  }
  __syncthreads();
  auto issue = [&](int t) {
    const int j0 = t * TJ, rows = min(TJ, n - j0);
    const uint32_t bytes = (uint32_t)rows * d * 4, kv_bytes = (uint32_t)rows * PW * 4;
    mbar_arrive_expect_tx(&bar[t & 1], bytes + kv_bytes);
    bulk_load(sm + L.tile[t & 1], pair_row + (long long)j0 * d, bytes, &bar[t & 1]);
    bulk_load(sm + L.kv[t & 1], p.proj + ((long long)b * n + j0) * PW, kv_bytes, &bar[t & 1]);
  };
  if (tid == 0) issue(0);

  // per-row constants: bias weights, this query's scalar and global point queries, zeroed accumulators
  const float* prow = p.proj + row * PW;
  for (int e = tid; e < H * d; e += IPA_THREADS) {
    sm[L.wb + e] = p.w_bias[e];
    sm[L.acc + e] = 0.f;
  }
  for (int e = tid; e < H * IPA_VW; e += IPA_THREADS) sm[L.accv + e] = 0.f;
  for (int e = tid; e < H * IPA_SD; e += IPA_THREADS) sm[L.q + e] = prow[e];
  for (int e = tid; e < H * 3 * IPA_PT; e += IPA_THREADS) sm[L.q + H * IPA_SD + e] = prow[3 * IPA_SD * H + e];
  if (tid < H) {
    sm[L.stat + tid] = -INFINITY;
    sm[L.stat + H + tid] = 0.f;
    sm[L.stat + 3 * H + tid] = -0.5f * softplus_torch(p.point_weights[tid]) * rsqrtf(54.f);
  }
  const bool mask_i = p.mask ? p.mask[row] != 0 : true;
  const float* qs = sm + L.q;
  const float* qp = sm + L.q + H * IPA_SD;
  __syncthreads();

  for (int t = 0; t < ntiles; ++t) {
    const int j0 = t * TJ, rows = min(TJ, n - j0);
    if (tid == 0 && t + 1 < ntiles) {
      fence_proxy_async_smem();                          // the buffer's last generic reads (tile t - 1) precede this write
      issue(t + 1);
    }
    mbar_wait(&bar[t & 1], (t >> 1) & 1);
    const float* tile = sm + L.tile[t & 1];
    const float* kvt = sm + L.kv[t & 1];

    // logits: warp per key row
    for (int jj = warp; jj < TJ; jj += IPA_THREADS / 32) {
      float part[IPA_MAX_HEADS];
#pragma unroll
      for (int h = 0; h < IPA_MAX_HEADS; ++h) part[h] = 0.f;
      if (jj < rows) {
        for (int c = lane; c < d; c += 32) {
          const float xv = tile[jj * d + c];
#pragma unroll
          for (int h = 0; h < IPA_MAX_HEADS; ++h)
            if (h < H) part[h] = fmaf(xv, sm[L.wb + h * d + c], part[h]);
        }
      }
      float bias = 0.f;
#pragma unroll
      for (int h = 0; h < IPA_MAX_HEADS; ++h) {
        if (h < H) {
          const float v = warp_sum(part[h]);
          if (lane == h) bias = v;
        }
      }
      if (lane < H) {
        const int h = lane, j = j0 + jj;
        float logit = -INFINITY;                          // beyond n: no weight
        if (jj < rows) {
          const float* kr = kvt + jj * PW;
          const float* ks = kr + IPA_SD * H + h * IPA_SD;
          const float* kp = kr + 3 * IPA_SD * H + 3 * IPA_PT * H + h * 3 * IPA_PT;
          float sdot = 0.f, dist = 0.f;
#pragma unroll
          for (int e = 0; e < IPA_SD; ++e) sdot = fmaf(qs[h * IPA_SD + e], ks[e], sdot);
#pragma unroll
          for (int e = 0; e < 3 * IPA_PT; ++e) {
            const float df = qp[h * 3 * IPA_PT + e] - kp[e];
            dist = fmaf(df, df, dist);
          }
          logit = (bias + p.b_bias[h]) * rsqrtf(3.f) + sdot * rsqrtf(48.f) + sm[L.stat + 3 * H + h] * dist;
          if (p.mask && !(mask_i && p.mask[(long long)b * n + j])) logit = -FLT_MAX;
        }
        sm[L.logit + h * TJ + jj] = logit;
      }
    }
    __syncthreads();

    // online softmax: warp per head, lanes over the tile's keys
    for (int h = warp; h < H; h += IPA_THREADS / 32) {
      float mt = -INFINITY;
      for (int jj = lane; jj < TJ; jj += 32) mt = fmaxf(mt, sm[L.logit + h * TJ + jj]);
      mt = warp_max(mt);
      const float m_old = sm[L.stat + h];
      const float m_new = fmaxf(m_old, mt);
      float ps = 0.f;
      for (int jj = lane; jj < TJ; jj += 32) {
        const float pv = expf(sm[L.logit + h * TJ + jj] - m_new);
        sm[L.logit + h * TJ + jj] = pv;
        ps += pv;
      }
      ps = warp_sum(ps);
      __syncwarp();
      if (lane == 0) {
        const float alpha = expf(m_old - m_new);         // 0 on the first tile (m_old = -inf)
        sm[L.stat + h] = m_new;
        sm[L.stat + H + h] = sm[L.stat + H + h] * alpha + ps;
        sm[L.stat + 2 * H + h] = alpha;
      }
    }
    __syncthreads();

    // aggregates: o_pair from the tile, o_scalar and global o_point from the keys' values
    for (int e = tid; e < H * d; e += IPA_THREADS) {
      const int h = e / d, c = e - h * d;
      const float* pr = sm + L.logit + h * TJ;
      float a = sm[L.acc + e] * sm[L.stat + 2 * H + h];
      for (int jj = 0; jj < rows; ++jj) a = fmaf(pr[jj], tile[jj * d + c], a);
      sm[L.acc + e] = a;
    }
    for (int e = tid; e < H * IPA_VW; e += IPA_THREADS) {
      const int h = e / IPA_VW, f = e - h * IPA_VW;
      const int col = f < IPA_SD ? 2 * IPA_SD * H + h * IPA_SD + f : 3 * IPA_SD * H + 6 * IPA_PT * H + h * 3 * IPA_PT + (f - IPA_SD);
      const float* pr = sm + L.logit + h * TJ;
      const float* vr = kvt + col;
      float a = sm[L.accv + e] * sm[L.stat + 2 * H + h];
      for (int jj = 0; jj < rows; ++jj) a = fmaf(pr[jj], vr[jj * PW], a);
      sm[L.accv + e] = a;
    }
    __syncthreads();
  }

  // epilogue
  const int OW = H * (2 * IPA_SD + d);
  float* orow = p.out + lrow * OW;
  for (int e = tid; e < H * d; e += IPA_THREADS) {
    const int h = e / d;
    orow[H * 2 * IPA_SD + e] = sm[L.acc + e] / sm[L.stat + H + h];
  }
  for (int e = tid; e < H * IPA_SD; e += IPA_THREADS) {
    const int h = e / IPA_SD;
    orow[e] = sm[L.accv + h * IPA_VW + (e - h * IPA_SD)] / sm[L.stat + H + h];
  }
  if (tid < H * IPA_PT) {
    const int h = tid / IPA_PT, pt = tid - h * IPA_PT;
    const float inv = 1.f / sm[L.stat + H + h];
    const float* g = sm + L.accv + h * IPA_VW + IPA_SD + pt * 3;
    const float* R = p.rot + row * 9;
    const float* tr = p.trans + row * 3;
    const float gx = g[0] * inv - tr[0], gy = g[1] * inv - tr[1], gz = g[2] * inv - tr[2];
    float sq = 0.f;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const float l = fmaf(gx, R[3 * c], fmaf(gy, R[3 * c + 1], gz * R[3 * c + 2]));   // (g - t) R^T
      orow[H * IPA_SD + h * 3 * IPA_PT + pt * 3 + c] = l;
      sq = fmaf(l, l, sq);
    }
    orow[H * IPA_SD + H * 3 * IPA_PT + h * IPA_PT + pt] = sqrtf(sq + 1e-8f);
  }
}

// ------------------------------------------------------------------------------------------------ layer tail
// Warp per residue.  s <- LayerNorm(s + o) (the post-norm residual of IPABlock).  With w_qu (after ff_norm): the quaternion /
// translation update of alphafold2.py:879-885 -- (u, v) = to_quaternion_update(s), q <- standardise(q (x) (1, u)),
// t <- t + v R (R of this layer) -- then the next layer's R = quat_to_matrix(q).  With coords (the last layer): coords =
// to_points(s) quat_to_matrix(q) + t and confidence = lddt_linear(s) (alphafold2.py:889-891, 903).
struct TailParams {
  float* s;                  // [rows, d]
  const float* o;            // [rows, d]
  const float *gamma, *beta;
  const float *w_qu, *b_qu;  // [6, d], [6] or null
  float *quat, *trans, *rot; // [rows, 4], [rows, 3], [rows, 9]
  const float *w_points, *b_points, *w_lddt, *b_lddt;
  float *coords, *confidence;  // [rows, 3], [rows] or null
  long long rows;
  int d;
  float eps;
};

__global__ void structure_tail_kernel(const TailParams p) {
  const int lane = threadIdx.x & 31;
  const long long r = (long long)blockIdx.x * (blockDim.x / 32) + threadIdx.x / 32;
  if (r >= p.rows) return;
  const int d = p.d;
  float* s = p.s + r * d;
  const float* o = p.o + r * d;
  float sum = 0.f;
  for (int c = lane; c < d; c += 32) sum += s[c] + o[c];
  const float mean = warp_sum(sum) / d;
  float var = 0.f;
  for (int c = lane; c < d; c += 32) {
    const float v = s[c] + o[c] - mean;
    var = fmaf(v, v, var);
  }
  const float rstd = rsqrtf(warp_sum(var) / d + p.eps);
  float dots[10] = {};                                   // 6 quaternion / translation updates, 3 points, 1 confidence
  for (int c = lane; c < d; c += 32) {
    const float y = fmaf((s[c] + o[c] - mean) * rstd, p.gamma[c], p.beta[c]);
    s[c] = y;
    if (p.w_qu) {
#pragma unroll
      for (int k = 0; k < 6; ++k) dots[k] = fmaf(y, p.w_qu[k * d + c], dots[k]);
    }
    if (p.coords) {
#pragma unroll
      for (int k = 0; k < 3; ++k) dots[6 + k] = fmaf(y, p.w_points[k * d + c], dots[6 + k]);
      dots[9] = fmaf(y, p.w_lddt[c], dots[9]);
    }
  }
  if (!p.w_qu) return;
#pragma unroll
  for (int k = 0; k < 10; ++k) dots[k] = warp_sum(dots[k]);
  if (lane != 0) return;
  float u[6];
#pragma unroll
  for (int k = 0; k < 6; ++k) u[k] = dots[k] + p.b_qu[k];
  float* qg = p.quat + r * 4;
  float* tg = p.trans + r * 3;
  float* Rg = p.rot + r * 9;
  const float a0 = qg[0], a1 = qg[1], a2 = qg[2], a3 = qg[3];
  const float b0 = 1.f, b1 = u[0], b2 = u[1], b3 = u[2];
  float q[4] = {a0 * b0 - a1 * b1 - a2 * b2 - a3 * b3, a0 * b1 + a1 * b0 + a2 * b3 - a3 * b2,
                a0 * b2 - a1 * b3 + a2 * b0 + a3 * b1, a0 * b3 + a1 * b2 - a2 * b1 + a3 * b0};
  if (q[0] < 0.f) {
#pragma unroll
    for (int k = 0; k < 4; ++k) q[k] = -q[k];
  }
  float t[3];
#pragma unroll
  for (int c = 0; c < 3; ++c) t[c] = tg[c] + fmaf(u[3], Rg[c], fmaf(u[4], Rg[3 + c], u[5] * Rg[6 + c]));
  float R[9];
  quat_to_matrix(q, R);
#pragma unroll
  for (int k = 0; k < 4; ++k) qg[k] = q[k];
#pragma unroll
  for (int c = 0; c < 3; ++c) tg[c] = t[c];
#pragma unroll
  for (int k = 0; k < 9; ++k) Rg[k] = R[k];
  if (p.coords) {
    float x[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) x[k] = dots[6 + k] + p.b_points[k];
#pragma unroll
    for (int c = 0; c < 3; ++c) p.coords[r * 3 + c] = fmaf(x[0], R[c], fmaf(x[1], R[3 + c], fmaf(x[2], R[6 + c], t[c])));
    p.confidence[r] = dots[9] + p.b_lddt[0];
  }
}

}  // namespace af2
