// Distogram to coordinates (alphafold2_pytorch/utils.py:718-833): the centring of a distogram into a distance estimate and
// a weight per pair, and the SMACOF loop of the reference's weighted MDS.
//
//  center_distogram_kernel   one pass over [P = B*N*N pairs][nb] fp32.  Each warp stages a run of 32 consecutive pairs
//                            (32 * nb * 4 B, contiguous) in shared memory with coalesced 16-byte loads; lane l then reduces
//                            pair l of the run from shared memory.  Writes central and weights [P] fp32.
//  mds_smacof_kernel         the whole SMACOF loop in one cooperative launch, one grid sync per iteration.  Work item =
//                            MDS_ROWS rows of one batch element; X of that element lives in shared memory.  Each item
//                            writes its fp64 stress and |X'|^2 partial; after the grid sync every CTA reduces the partials
//                            of the iteration in the same fixed order, so all CTAs take the same stop decision without a
//                            second sync, and the result does not depend on the grid size.
#pragma once
#include <cooperative_groups.h>
#include "common.cuh"

namespace af2 {

constexpr int CD_WARPS = 8;            // warps per CTA of the centring kernel
constexpr int CD_MAX_BINS = 128;       // largest bin count: 16 KB of shared memory per warp
constexpr int MDS_THREADS = 256;
constexpr int MDS_WARPS = MDS_THREADS / 32;
constexpr int MDS_ROWS = 2 * MDS_WARPS;  // rows per work item: two per warp
constexpr int MDS_MAX_N = 12288;       // X as float4 in shared memory: 192 KB

enum CenterMode { CD_MEAN = 0, CD_MEDIAN = 1 };
enum WideMode { CD_STD = 0, CD_VAR = 1, CD_NONE = 2 };

struct CenterParams {
  const float* dist;       // [P][nb] probabilities, or logits when softmax
  const float* centres;    // [nb] bin centres (the reference's n_bins)
  const unsigned char* mask;  // [B][N] residue mask or nullptr: a pair with a masked residue gets weight 0
  float* central;          // [P]
  float* weights;          // [P]
  long long pairs;         // B * N * N
  int n, nb, center, wide, softmax;
  float thr;               // a pair's weight is kept only where central <= thr (bins[-2])
};

__global__ void __launch_bounds__(CD_WARPS * 32) center_distogram_kernel(CenterParams p) {
  extern __shared__ float cd_smem[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int nb = p.nb;
  float* run = cd_smem + (size_t)warp * 32 * nb;
  const long long runs = (p.pairs + 31) / 32;
  const long long nn = (long long)p.n * p.n;
  for (long long r = (long long)blockIdx.x * CD_WARPS + warp; r < runs; r += (long long)gridDim.x * CD_WARPS) {
    const long long p0 = r * 32;
    const int count = p.pairs - p0 < 32 ? (int)(p.pairs - p0) : 32;
    const float* src = p.dist + p0 * nb;  // 64-bit element offset: B*N*N*nb passes 2^31 at B 3, N 4800
    __syncwarp();
    if (count == 32) {  // 32 * nb floats = 8 * nb float4, 16-byte aligned because the run starts at a multiple of 128 * nb B
      const float4* s4 = reinterpret_cast<const float4*>(src);
      float4* d4 = reinterpret_cast<float4*>(run);
#pragma unroll 4
      for (int k = lane; k < 8 * nb; k += 32) d4[k] = __ldcs(s4 + k);
    } else {
      for (int k = lane; k < count * nb; k += 32) run[k] = __ldcs(src + k);
    }
    __syncwarp();
    if (lane >= count) continue;
    float* v = run + lane * nb;  // nb odd (37): lanes hit distinct banks
    if (p.softmax) {
      float m = v[0];
      for (int k = 1; k < nb; ++k) m = fmaxf(m, v[k]);
      float s = 0.f;
      for (int k = 0; k < nb; ++k) { const float e = expf(v[k] - m); v[k] = e; s += e; }
      const float inv = 1.f / s;
      for (int k = 0; k < nb; ++k) v[k] = v[k] * inv;
    }
    float mag = 0.f;
    for (int k = 0; k < nb; ++k) mag += v[k];
    float c;
    if (p.center == CD_MEDIAN) {  // searchsorted(cumsum, 0.5 * total, side left), clamped to the last bin
      const float half = 0.5f * mag;
      float cum = 0.f;
      int idx = nb;
      for (int k = 0; k < nb; ++k) {
        cum += v[k];
        if (cum >= half) { idx = k; break; }
      }
      c = __ldg(p.centres + (idx < nb - 1 ? idx : nb - 1));
    } else {
      float s = 0.f;
      for (int k = 0; k < nb; ++k) s += v[k] * __ldg(p.centres + k);
      c = s / mag;
    }
    const float keep = c <= p.thr ? 1.f : 0.f;
    const long long pair = p0 + lane;
    const long long ij = pair % nn;
    const int i = (int)(ij / p.n), j = (int)(ij % p.n);
    if (i == j) c *= 0.f;  // the reference's `*= 0.`: NaN stays NaN
    float disp = 0.f;
    if (p.wide != CD_NONE) {
      float s = 0.f;
      for (int k = 0; k < nb; ++k) {
        const float d = __ldg(p.centres + k) - c;
        s += v[k] * (d * d);
      }
      disp = s / mag;
      if (p.wide == CD_STD) disp = sqrtf(disp);
    }
    float w = keep / (1.f + disp);  // a NaN weight stays NaN: the reference's `weights[w != w] *= 0.`
    if (i == j) w *= 0.f;
    if (p.mask) {
      const long long e = pair / nn;
      if (!p.mask[e * p.n + i] || !p.mask[e * p.n + j]) w = 0.f;
    }
    p.central[pair] = c;
    p.weights[pair] = w;
  }
}

struct MdsParams {
  const float* delta;    // [B][N][N] target distances
  const float* w;        // [B][N][N] weights, or nullptr for all ones
  float* x;              // [B][N][3] in: the init; out: the coords the loop returns
  float* xalt;           // [B][N][3] workspace: the other buffer of the double-buffered X
  double* part;          // workspace [2][B][tiles][2]: (stress, |X'|^2) per item, by iteration parity
  double* his;           // [iters + 1][B]: his[0] = inf, his[k + 1] = stress / |X'| of iteration k (every evaluated one)
  double* stress;        // [iters][B]: the stress of every evaluated iteration
  int* steps;            // [2]: accepted iterations, and 1 if the loop stopped on tol
  int B, n, tiles, iters;
  float invn;            // 1 / n
  double tol;
};

__device__ __forceinline__ double block_sum_f64(double v, double* red) {
  // fixed-order block reduction: warp shuffle tree, then warp 0 over the per-warp sums; every CTA gets the same bits
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  __syncthreads();
  if (lane == 0) red[warp] = v;
  __syncthreads();
  double t = 0.0;
  if (warp == 0) {
    t = lane < MDS_WARPS ? red[lane] : 0.0;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
    if (lane == 0) red[MDS_WARPS] = t;
  }
  __syncthreads();
  return red[MDS_WARPS];
}

__global__ void __launch_bounds__(MDS_THREADS) mds_smacof_kernel(MdsParams p) {
  namespace cg = cooperative_groups;
  cg::grid_group grid = cg::this_grid();
  extern __shared__ float4 sx[];  // [N] (x, y, z, 0) of the current batch element
  __shared__ double red[MDS_WARPS + 1];
  __shared__ double wpart[MDS_WARPS][2];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int N = p.n;
  const long long nn = (long long)N * N;
  const int items = p.B * p.tiles;
  const float invn = p.invn;
  if (blockIdx.x == 0)
    for (int e = threadIdx.x; e < p.B; e += blockDim.x) p.his[e] = __longlong_as_double(0x7ff0000000000000LL);
  float* cur = p.x;
  float* nxt = p.xalt;
  int steps = 0, stopped = 0;
  for (int it = 0; it < p.iters; ++it) {
    double* part = p.part + (size_t)(it & 1) * items * 2;
    int loaded = -1;
    for (int item = blockIdx.x; item < items; item += gridDim.x) {
      const int e = item / p.tiles, tile = item % p.tiles;
      if (e != loaded) {
        __syncthreads();
        const float* xe = cur + (size_t)e * N * 3;
        for (int k = threadIdx.x; k < N; k += blockDim.x) sx[k] = make_float4(xe[3 * k], xe[3 * k + 1], xe[3 * k + 2], 0.f);
        __syncthreads();
        loaded = e;
      }
      double st_w = 0.0, nrm_w = 0.0;
#pragma unroll 1
      for (int rr = 0; rr < MDS_ROWS / MDS_WARPS; ++rr) {
        const int i = tile * MDS_ROWS + rr * MDS_WARPS + warp;
        if (i >= N) break;
        const float4 xi = sx[i];
        const float* drow = p.delta + e * nn + (long long)i * N;
        const float* wrow = p.w ? p.w + e * nn + (long long)i * N : nullptr;
        float ax = 0.f, ay = 0.f, az = 0.f;
        double st = 0.0;
#pragma unroll 4
        for (int j = lane; j < N; j += 32) {
          const float4 xj = sx[j];
          const float dx = xi.x - xj.x, dy = xi.y - xj.y, dz = xi.z - xj.z;
          // direct differences, not the matmul form of cdist; sqrt and 1 / dist on the SFU (~2 ulp), so the loop has no
          // IEEE slow-path calls
          const float dsq = dx * dx + dy * dy + dz * dz;
          const float rs = rsqrtf(dsq);
          const float d = dsq > 0.f ? dsq * rs : 0.f;
          const float del = __ldg(drow + j);
          const float wt = wrow ? __ldg(wrow + j) : 1.f;
          const float diff = d - del;
          st += (double)(wt * (diff * diff));                  // stress before the 1e-7 perturbation, diagonal included
          const float r = wt * (d <= 0.f ? del * 1e7f : del * rs);  // delta / dist, dist <= 0 perturbed to 1e-7
          ax += r * dx; ay += r * dy; az += r * dz;            // sum_j r_ij (x_i - x_j) = (B X)_i
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
          ax += __shfl_xor_sync(0xffffffffu, ax, o);
          ay += __shfl_xor_sync(0xffffffffu, ay, o);
          az += __shfl_xor_sync(0xffffffffu, az, o);
          st += __shfl_xor_sync(0xffffffffu, st, o);
        }
        const float nx = invn * ax, ny = invn * ay, nz = invn * az;
        if (lane == 0) {
          float* o = nxt + ((size_t)e * N + i) * 3;
          o[0] = nx; o[1] = ny; o[2] = nz;
        }
        st_w += st;
        nrm_w += (double)nx * nx + (double)ny * ny + (double)nz * nz;
      }
      if (lane == 0) { wpart[warp][0] = st_w; wpart[warp][1] = nrm_w; }
      __syncthreads();
      if (threadIdx.x == 0) {
        double s = 0.0, q = 0.0;
        for (int k = 0; k < MDS_WARPS; ++k) { s += wpart[k][0]; q += wpart[k][1]; }
        part[2 * (size_t)item] = s;
        part[2 * (size_t)item + 1] = q;
      }
      __syncthreads();
    }
    grid.sync();
    // every CTA: stress_e = 0.5 sum of item partials, |X'_e| = sqrt(sum), and the reference's stop rule on the batch mean
    double gap = 0.0;
    for (int e = 0; e < p.B; ++e) {
      double s = 0.0, q = 0.0;
      for (int t = threadIdx.x; t < p.tiles; t += blockDim.x) {
        s += part[2 * ((size_t)e * p.tiles + t)];
        q += part[2 * ((size_t)e * p.tiles + t) + 1];
      }
      s = 0.5 * block_sum_f64(s, red);
      q = block_sum_f64(q, red);
      const double val = __ddiv_rn(s, __dsqrt_rn(q));
      gap += p.his[(size_t)it * p.B + e] - val;
      __syncthreads();
      if (blockIdx.x == 0 && threadIdx.x == 0) {
        p.his[(size_t)(it + 1) * p.B + e] = val;
        p.stress[(size_t)it * p.B + e] = s;
      }
    }
    if (gap / p.B <= p.tol) { stopped = 1; break; }
    ++steps;
    float* t = cur; cur = nxt; nxt = t;
    // his[it + 1] is read by every CTA in the next iteration's decision, after that iteration's grid sync
  }
  if (cur != p.x) {  // the accepted coords sit in the workspace buffer: copy them out (no CTA reads p.x any more)
    const long long total = (long long)p.B * N * 3;
    for (long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x; k < total; k += (long long)gridDim.x * blockDim.x)
      p.x[k] = cur[k];
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) { p.steps[0] = steps; p.steps[1] = stopped; }
}

}  // namespace af2
