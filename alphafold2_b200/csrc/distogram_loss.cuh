// The distogram loss of the reference's training script (train_pre.py:76-90): the cross-entropy of the distogram logits
// against the bucketed true distances of get_bucketed_distance_matrix (utils.py:45-50), and those labels on their own.
//
//  xent_rows_kernel<L>       one CTA per (element, pair row) of the logits rows [row0, row0 + rows) of the L::H heads of a
//                            label policy L (DistanceLabels here: the distogram, one head; AngleLabels in angle_loss.cuh).
//                            Each warp walks the row's tiles of P = min(32, DX_TILE / sum nb) consecutive pairs (P * nb[h]
//                            contiguous floats of each head) with a stride of DX_WARPS tiles, copying them into a
//                            DX_STAGES-deep ring of its own with 4-byte cp.async: coalesced at any alignment of the row
//                            start (N * nb need not be a multiple of 4) and with two tiles in flight while the third is
//                            reduced.  Lane l reduces pair l of a tile from shared memory (its labels from L), and the CTA
//                            writes the row's fp64 sum and int64 count per head.  A row whose residue is masked reads no
//                            logits.
//  xent_finish_kernel        one CTA per loss: its per-row partials summed in a fixed order, divided by the count.
//  bucketed_distance_kernel  the int64 labels [B][n][n] (grid-stride, one pair per thread, store-bound).
//
// Numerics: term = (max + logf(sum_c expf(l_c - max))) - l[label] in fp32 with the IEEE-accurate expf / logf (the library is
// built without --use_fast_math), the sum over c in a fixed per-lane order.  Each lane adds its terms to an fp64 sum in tile
// order; the CTA adds the lanes by a fixed shuffle tree and the warps in order.  The order depends only on (n, nb), never on
// row0 or rows, so partials of any split of the rows are bitwise those of the whole, and the finish kernel, which sees only
// the concatenated partials, returns the same bits however the rows were split over calls or ranks.
#pragma once
#include "common.cuh"
#include "glue_kernels.cuh"

namespace af2 {

constexpr int DX_WARPS = 4;
constexpr int DX_THREADS = DX_WARPS * 32;
constexpr int DX_STAGES = 3;
constexpr int DX_TILE = 4096;           // floats per ring slot at most: 16 KB
constexpr int DX_MAX_BINS = DX_TILE;    // one pair per tile at the largest bucket count
constexpr int DX_FIN_THREADS = 256;

struct XentPart {                        // one per (element, row)
  double sum;
  long long count;
};

// The rows kernel's side of a label policy L (DistanceLabels below, AngleLabels in angle_loss.cuh): L::H heads, each with its
// own logits and bucket count, scored against the labels L computes per pair.  L::Row row(e, i) holds what the CTA needs of
// residue i; labels(row, e, j, lab) writes the H labels of pair (i, j) (an unmasked j; the kernel applies the mask and
// ignore_index).
template <int H>
struct XentParams {
  const float* logits[H];                // head h: [B][rows][n][nb[h]], the rows [row0, row0 + rows)
  int nb[H];
  const unsigned char* mask;             // [B][n] or null
  long long ignore_index;
  int n, row0, rows;
  int pairs_per_tile, slot;              // P and the ring slot size in floats (P * (nb[0] + ... + nb[H-1]))
  XentPart* part;                        // [B][rows][H]
};

// P = pairs per tile for the bucket counts nb[0 .. H-1] summing to nbs: 32, fewer above nbs 128 (one at DX_TILE)
inline int xent_pairs_per_tile(int nbs) { return nbs <= DX_TILE / 32 ? 32 : DX_TILE / nbs; }

__device__ __forceinline__ void cp_async4(float* dst, const float* src) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(smem_u32(dst)), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// (max + logf(sum_c expf(v_c - max))) - v[label] over v[0 .. nb-1], channels visited from rot on (cyclically)
__device__ __forceinline__ float xent_term(const float* v, int nb, int rot, int label) {
  float m = v[rot];
  for (int k = 1, cc = rot + 1; k < nb; ++k, ++cc) {
    if (cc == nb) cc = 0;
    m = fmaxf(m, v[cc]);
  }
  float s = 0.f;
  for (int k = 0, cc = rot; k < nb; ++k, ++cc) {
    if (cc == nb) cc = 0;
    s += expf(v[cc] - m);
  }
  return (m + logf(s)) - v[label];
}

// The distogram's labels: distance_bucket of the coordinates of i and j under the edges bnd
struct DistanceLabels {
  static constexpr int H = 1;
  const float* coords;                   // [B][n][c]
  const float* bnd;                      // [nb]: the bucket edges, the first nb - 1 searched
  int c, nb;
  struct Row { const float* ci; };
  __device__ __forceinline__ Row row(int e, int i, int n) const { return {coords + ((long long)e * n + i) * c}; }
  __device__ __forceinline__ void labels(const Row& r, int e, int j, int n, int (&lab)[1]) const {
    lab[0] = distance_bucket(r.ci, coords + ((long long)e * n + j) * c, c, bnd, nb);
  }
};

template <class L>
__global__ void __launch_bounds__(DX_THREADS) xent_rows_kernel(XentParams<L::H> p, L lp) {
  constexpr int H = L::H;
  extern __shared__ float dx_smem[];
  __shared__ double red_s[H][DX_WARPS];
  __shared__ long long red_c[H][DX_WARPS];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int r = blockIdx.x, e = blockIdx.y, i = p.row0 + r;
  const int n = p.n, P = p.pairs_per_tile;
  const long long prow = (long long)e * p.rows + r;
  double acc[H];
  long long cnt[H];
#pragma unroll
  for (int h = 0; h < H; ++h) { acc[h] = 0.0; cnt[h] = 0; }
  if (!p.mask || p.mask[(long long)e * n + i]) {
    float* ring = dx_smem + (size_t)warp * DX_STAGES * p.slot;
    const float* Lg[H];
    int off[H], rot[H];
    int o = 0;
#pragma unroll
    for (int h = 0; h < H; ++h) {
      Lg[h] = p.logits[h] + prow * n * p.nb[h];         // 64-bit: B * rows * n * nb passes 2^31
      off[h] = o;                                        // head h's P * nb[h] floats within a slot
      o += P * p.nb[h];
      // even nb: lane l reads its channels from (l mod nb) on, so that the stride-nb pair layout stays conflict-free
      rot[h] = (p.nb[h] & 1) ? 0 : lane % p.nb[h];
    }
    const typename L::Row ri = lp.row(e, i, n);
    const int tiles = (n + P - 1) / P;
    const int mine = warp < tiles ? (tiles - warp + DX_WARPS - 1) / DX_WARPS : 0;
    auto issue = [&](int q) {                            // this warp's q-th tile into slot q % DX_STAGES
      const int t = warp + q * DX_WARPS;
      const int np = min(n - t * P, P);
      float* dst = ring + (q % DX_STAGES) * p.slot;
#pragma unroll
      for (int h = 0; h < H; ++h) {
        const float* src = Lg[h] + (long long)t * P * p.nb[h];
        for (int k = lane; k < np * p.nb[h]; k += 32) cp_async4(dst + off[h] + k, src + k);
      }
    };
#pragma unroll
    for (int q = 0; q < DX_STAGES - 1; ++q) {
      if (q < mine) issue(q);
      cp_async_commit();
    }
    for (int q = 0; q < mine; ++q) {
      if (q + DX_STAGES - 1 < mine) issue(q + DX_STAGES - 1);
      cp_async_commit();
      cp_async_wait<DX_STAGES - 1>();
      __syncwarp();
      const int j = (warp + q * DX_WARPS) * P + lane;
      if (lane < P && j < n && (!p.mask || p.mask[(long long)e * n + j])) {
        int lab[H];
        lp.labels(ri, e, j, n, lab);
        const float* slot = ring + (q % DX_STAGES) * p.slot;
#pragma unroll
        for (int h = 0; h < H; ++h) {
          if ((long long)lab[h] != p.ignore_index) {
            acc[h] += (double)xent_term(slot + off[h] + lane * p.nb[h], p.nb[h], rot[h], lab[h]);
            cnt[h] += 1;
          }
        }
      }
      __syncwarp();                                      // the slot is refilled at iteration q + 1
    }
    cp_async_wait<0>();
  }
#pragma unroll
  for (int h = 0; h < H; ++h) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      acc[h] += __shfl_xor_sync(0xffffffffu, acc[h], o);
      cnt[h] += __shfl_xor_sync(0xffffffffu, cnt[h], o);
    }
    if (lane == 0) { red_s[h][warp] = acc[h]; red_c[h][warp] = cnt[h]; }
  }
  __syncthreads();
  if (threadIdx.x < H) {
    const int h = threadIdx.x;
    double s = 0.0;
    long long c = 0;
    for (int w = 0; w < DX_WARPS; ++w) { s += red_s[h][w]; c += red_c[h][w]; }
    p.part[prow * H + h].sum = s;
    p.part[prow * H + h].count = c;
  }
}

// Loss h = blockIdx.x of `losses` from parts partials each, interleaved ([parts][losses], row order): thread t sums the
// contiguous run [t * per, (t + 1) * per), thread 0 the runs in thread order; the order depends only on the number of parts.
// 0 / 0 = NaN when no pair counts.
__global__ void __launch_bounds__(DX_FIN_THREADS) xent_finish_kernel(const XentPart* part, long long parts, int losses, float* out) {
  __shared__ double red_s[DX_FIN_THREADS];
  __shared__ long long red_c[DX_FIN_THREADS];
  const int h = blockIdx.x;
  const long long per = (parts + DX_FIN_THREADS - 1) / DX_FIN_THREADS;
  const long long k0 = threadIdx.x * per, k1 = min(parts, k0 + per);
  double s = 0.0;
  long long c = 0;
  for (long long k = k0; k < k1; ++k) { s += part[k * losses + h].sum; c += part[k * losses + h].count; }
  red_s[threadIdx.x] = s;
  red_c[threadIdx.x] = c;
  __syncthreads();
  if (threadIdx.x == 0) {
    double ts = 0.0;
    long long tc = 0;
    for (int t = 0; t < DX_FIN_THREADS; ++t) { ts += red_s[t]; tc += red_c[t]; }
    out[h] = (float)(ts / (double)tc);
  }
}

// labels[b][i][j] = distance_bucket(coords[b][i], coords[b][j]), or ignore_index where mask[b][i] & mask[b][j] is false
__global__ void __launch_bounds__(256) bucketed_distance_kernel(const float* __restrict__ coords, int c, const unsigned char* __restrict__ mask,
                                                                const float* __restrict__ bnd, int nb, long long ignore_index, int B, int n,
                                                                long long* __restrict__ labels) {
  const long long nn = (long long)n * n, T = (long long)B * nn;
  for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < T; t += (long long)gridDim.x * blockDim.x) {
    const long long b = t / nn;
    const int i = (int)((t - b * nn) / n), j = (int)(t - b * nn - (long long)i * n);
    long long v = ignore_index;
    if (!mask || (mask[b * n + i] && mask[b * n + j])) v = distance_bucket(coords + (b * n + i) * c, coords + (b * n + j) * c, c, bnd, nb);
    labels[t] = v;
  }
}

}  // namespace af2
