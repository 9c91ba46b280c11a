// Structure scores (alphafold2_pytorch/utils.py:999-1247): Kabsch superposition, RMSD, GDT, TM-score, lDDT-CA and the
// distance-matrix loss.
//
//  pair_distance_kernel<MODE, AMAT, BMAT>   one pass over the b * N^2 pairs of two structures, never writing an N x N
//                            matrix.  Grid (row tile, column split, element); each CTA stages PD_TJ points of both
//                            structures' j coordinates in shared memory; each warp owns PD_ROWS / PD_WARPS rows and its
//                            lanes stride over j.  MODE PD_LDDT: per row, the in-radius count and the score sum as int32,
//                            one slot per column split (integer sums: exact, summed by superpose_scores_kernel).  MODE
//                            PD_LOSS: fp64 (sum, count) per CTA, summed in a fixed order by loss_reduce_kernel.  AMAT /
//                            BMAT: that operand is a stored [*, N, N] fp32 distance matrix instead of coordinates.
//  superpose_scores_kernel   one CTA per element: the selected points in order, their fp64 centroids and covariance
//                            (fixed-order block sums), a 3 x 3 one-sided Jacobi SVD with the reference's determinant fix,
//                            then one pass that writes the aligned coordinates and reduces sum d^2, the GDT counts and the
//                            TM sum; and the lDDT ratios from the pair kernel's counters.
//
// Every threshold decision uses dist64: sqrt((dx * dx + dy * dy) + dz * dz) with dx = double(a) - double(b), each operation
// an explicitly rounded intrinsic so that nvcc cannot contract it into FMAs; the oracle evaluates the same expression.
#pragma once
#include "common.cuh"

namespace af2 {

constexpr int PD_THREADS = 256;
constexpr int PD_WARPS = PD_THREADS / 32;
constexpr int PD_ROWS = 32;              // rows per CTA: 4 per warp
constexpr int PD_RPW = PD_ROWS / PD_WARPS;
constexpr int PD_TJ = 512;               // j points staged per tile
constexpr int PD_MAX_SPLITS = 16;        // column splits: the lDDT counters are [splits][b][N][2]
constexpr int SS_THREADS = 256;
constexpr int SS_WARPS = SS_THREADS / 32;
constexpr int SS_MAX_CUT = 8;

enum PairMode { PD_LDDT = 0, PD_LOSS = 1 };

__device__ __forceinline__ double dist64(float ax, float ay, float az, float bx, float by, float bz) {
  const double dx = __dsub_rn((double)ax, (double)bx);
  const double dy = __dsub_rn((double)ay, (double)by);
  const double dz = __dsub_rn((double)az, (double)bz);
  return __dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz)));
}

struct PairOperand {
  const float* p;
  long long sb;      // elements between batch elements (0: one structure shared by the batch)
  long long sn;      // coordinates: elements between points; matrix: row stride
  long long sk;      // coordinates: elements between x, y and z
};

struct PairParams {
  PairOperand a, b;              // lDDT: a = true, b = predicted; loss: a = X, b = Y
  const unsigned char* mask;     // lDDT: residue mask [b][N] (stride mask_sn, mask_sb); loss: pair mask [b][N][N]; or null
  long long mask_sb, mask_sn;
  int n, split_cols;
  float lo, hi;                  // loss: coordinates clamped to [lo, hi]
  double r0;                     // lDDT inclusion radius (strict)
  double qh;                     // loss: ((da - db)^2)^qh
  int qmode;                     // 2: squared difference, 1: absolute difference, 0: pow(d^2, qh)
  int* counts;                   // lDDT: [splits][B][N][2] (count, score sum)
  double* part;                  // loss: [B][splits][tiles][2] (sum, count)
};

__device__ __forceinline__ float clampf_nan(float v, float lo, float hi) { return v < lo ? lo : (v > hi ? hi : v); }

template <int MODE, bool AMAT, bool BMAT>
__global__ void __launch_bounds__(PD_THREADS) pair_distance_kernel(PairParams p) {
  __shared__ float sa[3][PD_TJ];
  __shared__ float sb[3][PD_TJ];
  __shared__ unsigned char sm[PD_TJ];
  __shared__ double red[PD_WARPS][2];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int n = p.n, e = blockIdx.z;
  const int j0 = blockIdx.y * p.split_cols;
  const int j1 = min(n, j0 + p.split_cols);
  const int ibase = blockIdx.x * PD_ROWS + warp * PD_RPW;
  const float* A = p.a.p + (long long)e * p.a.sb;
  const float* Bp = p.b.p + (long long)e * p.b.sb;
  float ai[PD_RPW][3], bi[PD_RPW][3];
  bool rowok[PD_RPW];
#pragma unroll
  for (int r = 0; r < PD_RPW; ++r) {
    const int i = ibase + r;
    rowok[r] = i < n;
    if (MODE == PD_LDDT && rowok[r] && p.mask) rowok[r] = p.mask[(long long)e * p.mask_sb + (long long)i * p.mask_sn] != 0;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      ai[r][k] = (!AMAT && i < n) ? clampf_nan(__ldg(A + (long long)i * p.a.sn + k * p.a.sk), p.lo, p.hi) : 0.f;
      bi[r][k] = (!BMAT && i < n) ? clampf_nan(__ldg(Bp + (long long)i * p.b.sn + k * p.b.sk), p.lo, p.hi) : 0.f;
    }
  }
  int cnt[PD_RPW], scr[PD_RPW];
#pragma unroll
  for (int r = 0; r < PD_RPW; ++r) cnt[r] = scr[r] = 0;
  double lsum = 0.0, lcnt = 0.0;
  for (int t0 = j0; t0 < j1; t0 += PD_TJ) {
    const int tn = min(PD_TJ, j1 - t0);
    if (!AMAT || !BMAT || MODE == PD_LDDT) {
      __syncthreads();
      for (int k = threadIdx.x; k < tn; k += blockDim.x) {
        const long long j = t0 + k;
#pragma unroll
        for (int c = 0; c < 3; ++c) {
          if (!AMAT) sa[c][k] = clampf_nan(__ldg(A + j * p.a.sn + c * p.a.sk), p.lo, p.hi);
          if (!BMAT) sb[c][k] = clampf_nan(__ldg(Bp + j * p.b.sn + c * p.b.sk), p.lo, p.hi);
        }
        if (MODE == PD_LDDT) sm[k] = p.mask ? p.mask[(long long)e * p.mask_sb + j * p.mask_sn] : 1;
      }
      __syncthreads();
    }
#pragma unroll
    for (int r = 0; r < PD_RPW; ++r) {
      if (!rowok[r]) continue;
      const long long i = ibase + r;
      if (MODE == PD_LDDT) {
        for (int k = lane; k < tn; k += 32) {
          if (!sm[k]) continue;
          const double dt = dist64(ai[r][0], ai[r][1], ai[r][2], sa[0][k], sa[1][k], sa[2][k]);
          if (dt < p.r0) {
            const double dp = dist64(bi[r][0], bi[r][1], bi[r][2], sb[0][k], sb[1][k], sb[2][k]);
            const double diff = fabs(__dsub_rn(dp, dt));
            cnt[r] += 1;
            scr[r] += (diff <= 0.5) + (diff <= 1.0) + (diff <= 2.0) + (diff <= 4.0);
          }
        }
      } else {
        const unsigned char* mrow = p.mask ? p.mask + (long long)e * p.mask_sb + i * p.mask_sn : nullptr;
        const float* arow = A + i * p.a.sn;
        const float* brow = Bp + i * p.b.sn;
        for (int k = lane; k < tn; k += 32) {
          const long long j = t0 + k;
          if (mrow && !mrow[j]) continue;
          const double da = AMAT ? (double)__ldcs(arow + j) : dist64(ai[r][0], ai[r][1], ai[r][2], sa[0][k], sa[1][k], sa[2][k]);
          const double db = BMAT ? (double)__ldcs(brow + j) : dist64(bi[r][0], bi[r][1], bi[r][2], sb[0][k], sb[1][k], sb[2][k]);
          const double d = __dsub_rn(da, db);
          const double sq = __dmul_rn(d, d);
          lsum += p.qmode == 2 ? sq : (p.qmode == 1 ? fabs(d) : pow(sq, p.qh));
          lcnt += 1.0;
        }
      }
    }
  }
  if (MODE == PD_LDDT) {
#pragma unroll
    for (int r = 0; r < PD_RPW; ++r) {
      int c = cnt[r], s = scr[r];
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        c += __shfl_xor_sync(0xffffffffu, c, o);
        s += __shfl_xor_sync(0xffffffffu, s, o);
      }
      const int i = ibase + r;
      if (lane == 0 && i < n) {
        int* out = p.counts + (((long long)blockIdx.y * gridDim.z + e) * n + i) * 2;
        out[0] = c;
        out[1] = s;
      }
    }
  } else {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      lsum += __shfl_xor_sync(0xffffffffu, lsum, o);
      lcnt += __shfl_xor_sync(0xffffffffu, lcnt, o);
    }
    if (lane == 0) { red[warp][0] = lsum; red[warp][1] = lcnt; }
    __syncthreads();
    if (threadIdx.x == 0) {
      double s = 0.0, c = 0.0;
      for (int w = 0; w < PD_WARPS; ++w) { s += red[w][0]; c += red[w][1]; }
      const long long cta = ((long long)e * gridDim.y + blockIdx.y) * gridDim.x + blockIdx.x;
      p.part[2 * cta] = s;
      p.part[2 * cta + 1] = c;
    }
  }
}

// the loss: sum over the pair kernel's partials in a fixed order, mean over the counted pairs (0 / 0 = NaN for an empty mask)
__global__ void __launch_bounds__(SS_THREADS) loss_reduce_kernel(const double* part, long long parts, float* out) {
  __shared__ double red[SS_WARPS][2];
  double s = 0.0, c = 0.0;
  for (long long k = threadIdx.x; k < parts; k += blockDim.x) { s += part[2 * k]; c += part[2 * k + 1]; }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    s += __shfl_xor_sync(0xffffffffu, s, o);
    c += __shfl_xor_sync(0xffffffffu, c, o);
  }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (lane == 0) { red[warp][0] = s; red[warp][1] = c; }
  __syncthreads();
  if (threadIdx.x == 0) {
    double ts = 0.0, tc = 0.0;
    for (int w = 0; w < SS_WARPS; ++w) { ts += red[w][0]; tc += red[w][1]; }
    out[0] = (float)(ts / tc);
  }
}

struct Coords3 {
  float* p;              // const for inputs
  long long sb, sn, sk;  // element, point and coordinate strides (elements)
};

struct SuperposeParams {
  Coords3 x, y;                  // x: predicted (moved), y: true; x.p null: lDDT finalisation only
  const unsigned char* mask;     // [B][N] (strides mask_sb, mask_sn), or null: every point selected
  long long mask_sb, mask_sn;
  int* idx;                      // workspace [B][N]: the selected points in order (mask only)
  int n, align, shift;           // align: Kabsch; shift: the aligned x is placed in y's frame
  Coords3 xo, yo;                // aligned x and centred y, or p null
  double* rot;                   // [B][9] the reference's U (row-major), or null
  float *rmsd, *tm;              // [B] or null
  int ncut;
  float cut[SS_MAX_CUT];         // a point counts at cutoff c when d <= c
  float* gdt[2];                 // [B] or null: sum_k w_k (count_k / n) / K over the cutoffs gidx[g][0..gk[g])
  int gk[2], gidx[2][SS_MAX_CUT];
  float gw[2][SS_MAX_CUT];
  const int* counts;             // the pair kernel's lDDT counters [splits][B][N][2], or null
  int splits;
  float* lddt;                   // [B][N]
  float* lddt_mean;              // [B] or null
};

// fixed-order block sum of NV doubles: warp shuffle tree, then thread 0 over the warps in order; every thread gets the sums
template <int NV>
__device__ __forceinline__ void block_sums(double (&v)[NV], double (*red)[NV]) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int q = 0; q < NV; ++q)
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v[q] += __shfl_xor_sync(0xffffffffu, v[q], o);
  __syncthreads();
  if (lane == 0)
#pragma unroll
    for (int q = 0; q < NV; ++q) red[warp][q] = v[q];
  __syncthreads();
  if (threadIdx.x == 0)
#pragma unroll
    for (int q = 0; q < NV; ++q) {
      double t = 0.0;
      for (int w = 0; w < SS_WARPS; ++w) t += red[w][q];
      red[SS_WARPS][q] = t;
    }
  __syncthreads();
#pragma unroll
  for (int q = 0; q < NV; ++q) v[q] = red[SS_WARPS][q];
}

__device__ __forceinline__ double det3(const double m[3][3]) {
  return m[0][0] * (m[1][1] * m[2][2] - m[1][2] * m[2][1]) - m[0][1] * (m[1][0] * m[2][2] - m[1][2] * m[2][0]) +
         m[0][2] * (m[1][0] * m[2][1] - m[1][1] * m[2][0]);
}

// The reference's rotation for C = V S W (torch.linalg.svd): U = V W, with the last column of V negated when
// det V det W < 0.  One-sided Jacobi on the columns of C gives C J = [s_0 b_0, s_1 b_1, s_2 b_2]; sorted by s descending,
// V's columns are the b_k and W's rows the matching columns v_k of J.  Since V is orthonormal, the fixed last column is
// det(J_sorted) (b_0 x b_1), so U = b_0 v_0' + b_1 v_1' + det(J_sorted) (b_0 x b_1) v_2', which needs no b_2 and stays a
// proper rotation when C has rank 2 or less.
__device__ void kabsch_rotation(const double C[3][3], double U[3][3]) {
  double a[3][3], j[3][3];
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) { a[r][c] = C[r][c]; j[r][c] = r == c ? 1.0 : 0.0; }
  for (int sweep = 0; sweep < 30; ++sweep) {
    double off = 0.0;
    for (int pq = 0; pq < 3; ++pq) {
      const int P = pq == 2 ? 1 : 0, Q = pq == 0 ? 1 : 2;
      double al = 0.0, be = 0.0, ga = 0.0;
      for (int r = 0; r < 3; ++r) { al += a[r][P] * a[r][P]; be += a[r][Q] * a[r][Q]; ga += a[r][P] * a[r][Q]; }
      if (ga == 0.0 || al == 0.0 || be == 0.0) continue;
      const double rel = fabs(ga) / sqrt(al * be);
      if (rel <= 1e-17) continue;
      off = fmax(off, rel);
      const double zeta = (be - al) / (2.0 * ga);
      const double t = copysign(1.0, zeta) / (fabs(zeta) + sqrt(1.0 + zeta * zeta));
      const double cs = 1.0 / sqrt(1.0 + t * t), sn = cs * t;
      for (int r = 0; r < 3; ++r) {
        const double ap = a[r][P], aq = a[r][Q];
        a[r][P] = cs * ap - sn * aq; a[r][Q] = sn * ap + cs * aq;
        const double jp = j[r][P], jq = j[r][Q];
        j[r][P] = cs * jp - sn * jq; j[r][Q] = sn * jp + cs * jq;
      }
    }
    if (off <= 1e-15) break;
  }
  double s[3];
  for (int c = 0; c < 3; ++c) s[c] = sqrt(a[0][c] * a[0][c] + a[1][c] * a[1][c] + a[2][c] * a[2][c]);
  int o[3] = {0, 1, 2};
  for (int u = 0; u < 2; ++u)
    for (int w = 0; w < 2 - u; ++w)
      if (s[o[w]] < s[o[w + 1]]) { const int t = o[w]; o[w] = o[w + 1]; o[w + 1] = t; }
  double b0[3], b1[3], b2[3], v[3][3];
  for (int r = 0; r < 3; ++r)
    for (int k = 0; k < 3; ++k) v[r][k] = j[r][o[k]];
  if (s[o[0]] > 0.0) {
    for (int r = 0; r < 3; ++r) b0[r] = a[r][o[0]] / s[o[0]];
  } else {
    b0[0] = 1.0; b0[1] = 0.0; b0[2] = 0.0;
  }
  double pr = 0.0;
  for (int r = 0; r < 3; ++r) pr += b0[r] * a[r][o[1]];
  for (int r = 0; r < 3; ++r) b1[r] = a[r][o[1]] - pr * b0[r];
  double nb = sqrt(b1[0] * b1[0] + b1[1] * b1[1] + b1[2] * b1[2]);
  if (!(nb > 1e-12 * s[o[0]]) || nb == 0.0) {  // rank 1 or 0: any unit vector orthogonal to b0
    const int m = fabs(b0[0]) <= fabs(b0[1]) ? (fabs(b0[0]) <= fabs(b0[2]) ? 0 : 2) : (fabs(b0[1]) <= fabs(b0[2]) ? 1 : 2);
    double e[3] = {0.0, 0.0, 0.0};
    e[m] = 1.0;
    pr = b0[m];
    for (int r = 0; r < 3; ++r) b1[r] = e[r] - pr * b0[r];
    nb = sqrt(b1[0] * b1[0] + b1[1] * b1[1] + b1[2] * b1[2]);
  }
  for (int r = 0; r < 3; ++r) b1[r] /= nb;
  const double dv = det3(v) < 0.0 ? -1.0 : 1.0;
  b2[0] = dv * (b0[1] * b1[2] - b0[2] * b1[1]);
  b2[1] = dv * (b0[2] * b1[0] - b0[0] * b1[2]);
  b2[2] = dv * (b0[0] * b1[1] - b0[1] * b1[0]);
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) U[r][c] = b0[r] * v[c][0] + b1[r] * v[c][1] + b2[r] * v[c][2];
}

__global__ void __launch_bounds__(SS_THREADS) superpose_scores_kernel(SuperposeParams p) {
  __shared__ int scan[SS_THREADS + 1];
  __shared__ double redbuf[(SS_WARPS + 1) * (2 + SS_MAX_CUT)];
  __shared__ double rot[3][3];
  const int tid = threadIdx.x, T = blockDim.x;
  const int e = blockIdx.x, n = p.n;
  const unsigned char* mask = p.mask ? p.mask + (long long)e * p.mask_sb : nullptr;
  const long long msn = p.mask_sn;
  // 1. the selected points in order: chunk counts, an exclusive scan over the threads, then the indices
  int nsel = n;
  int* idx = p.idx ? p.idx + (long long)e * n : nullptr;
  if (mask) {
    const int per = (n + T - 1) / T, c0 = min(n, tid * per), c1 = min(n, c0 + per);
    int c = 0;
    for (int i = c0; i < c1; ++i) c += mask[i * msn] != 0;
    scan[tid + 1] = c;
    __syncthreads();
    if (tid == 0) {
      scan[0] = 0;
      for (int t = 1; t <= T; ++t) scan[t] += scan[t - 1];
    }
    __syncthreads();
    int r = scan[tid];
    for (int i = c0; i < c1; ++i)
      if (mask[i * msn]) idx[r++] = i;
    nsel = scan[T];
    __syncthreads();
  }
  const float nanf_ = __int_as_float(0x7fffffff);
  if (p.x.p) {
    const float* X = p.x.p + (long long)e * p.x.sb;
    const float* Y = p.y.p + (long long)e * p.y.sb;
    double cx[3] = {0.0, 0.0, 0.0}, cy[3] = {0.0, 0.0, 0.0};
    if (p.align && nsel > 0) {
      // 2. centroids and covariance, fp64, fixed order
      double v[9];
      for (int q = 0; q < 6; ++q) v[q] = 0.0;
      for (int r = tid; r < nsel; r += T) {
        const long long i = mask ? idx[r] : r;
        for (int k = 0; k < 3; ++k) {
          v[k] += (double)X[i * p.x.sn + k * p.x.sk];
          v[3 + k] += (double)Y[i * p.y.sn + k * p.y.sk];
        }
      }
      double c6[6];
      for (int q = 0; q < 6; ++q) c6[q] = v[q];
      block_sums<6>(c6, reinterpret_cast<double (*)[6]>(redbuf));
      for (int k = 0; k < 3; ++k) { cx[k] = c6[k] / nsel; cy[k] = c6[3 + k] / nsel; }
      for (int q = 0; q < 9; ++q) v[q] = 0.0;
      for (int r = tid; r < nsel; r += T) {
        const long long i = mask ? idx[r] : r;
        double xc[3], yc[3];
        for (int k = 0; k < 3; ++k) {
          xc[k] = (double)X[i * p.x.sn + k * p.x.sk] - cx[k];
          yc[k] = (double)Y[i * p.y.sn + k * p.y.sk] - cy[k];
        }
        for (int a = 0; a < 3; ++a)
          for (int b = 0; b < 3; ++b) v[3 * a + b] += xc[a] * yc[b];
      }
      block_sums<9>(v, reinterpret_cast<double (*)[9]>(redbuf));
      if (tid == 0) {
        double C[3][3], U[3][3];
        for (int a = 0; a < 3; ++a)
          for (int b = 0; b < 3; ++b) C[a][b] = v[3 * a + b];
        kabsch_rotation(C, U);
        for (int a = 0; a < 3; ++a)
          for (int b = 0; b < 3; ++b) rot[a][b] = U[a][b];
      }
      __syncthreads();
      if (p.rot && tid < 9) p.rot[(long long)e * 9 + tid] = rot[tid / 3][tid % 3];
    } else if (p.align && p.rot && tid < 9) {  // no selected point: no rotation, and none of the caller's memory left stale
      p.rot[(long long)e * 9 + tid] = __longlong_as_double(0x7ff8000000000000LL);
    }
    // 3. d0 of the reference's TM-score on the selected points: L = max(15, n), no lower clamp
    const double d0 = 1.24 * pow((double)((nsel > 15 ? nsel : 15) - 15), 1.0 / 3.0) - 1.8;
    // x moved by the rotation (rounded to fp32, as the reference's Kabsch returns it) and y centred, or both as given
    auto place = [&](long long i, float (&xa)[3], float (&ya)[3], double (&a64)[3]) {
      if (p.align) {
        double xc[3];
        for (int k = 0; k < 3; ++k) xc[k] = (double)X[i * p.x.sn + k * p.x.sk] - cx[k];
        for (int c = 0; c < 3; ++c) {
          a64[c] = nsel > 0 ? rot[0][c] * xc[0] + rot[1][c] * xc[1] + rot[2][c] * xc[2] : (double)nanf_;
          xa[c] = (float)a64[c];
          ya[c] = (float)((double)Y[i * p.y.sn + c * p.y.sk] - cy[c]);
        }
      } else {
        for (int c = 0; c < 3; ++c) { xa[c] = X[i * p.x.sn + c * p.x.sk]; ya[c] = Y[i * p.y.sn + c * p.y.sk]; a64[c] = xa[c]; }
      }
    };
    if (p.xo.p || p.yo.p) {  // the whole chain, selected or not
      for (int i = tid; i < n; i += T) {
        float xa[3], ya[3];
        double a64[3];
        place(i, xa, ya, a64);
        if (p.xo.p)
          for (int c = 0; c < 3; ++c) p.xo.p[(long long)e * p.xo.sb + i * p.xo.sn + c * p.xo.sk] = p.shift ? (float)(a64[c] + cy[c]) : xa[c];
        if (p.yo.p)
          for (int c = 0; c < 3; ++c) p.yo.p[(long long)e * p.yo.sb + i * p.yo.sn + c * p.yo.sk] = ya[c];
      }
    }
    // the scores: over the selected points in order, so that a masked call sums exactly as the same call on the compacted
    // points does
    double acc[2] = {0.0, 0.0};
    int cnt[SS_MAX_CUT];
    for (int k = 0; k < SS_MAX_CUT; ++k) cnt[k] = 0;
    for (int r = tid; r < nsel; r += T) {
      float xa[3], ya[3];
      double a64[3];
      place(mask ? idx[r] : r, xa, ya, a64);
      const double d = dist64(xa[0], xa[1], xa[2], ya[0], ya[1], ya[2]);
      acc[0] += d * d;
      const double u = d / d0;
      acc[1] += 1.0 / (1.0 + u * u);
      for (int k = 0; k < p.ncut; ++k) cnt[k] += d <= (double)p.cut[k];
    }
    double sums[2 + SS_MAX_CUT];
    sums[0] = acc[0];
    sums[1] = acc[1];
    for (int k = 0; k < SS_MAX_CUT; ++k) sums[2 + k] = (double)cnt[k];
    block_sums<2 + SS_MAX_CUT>(sums, reinterpret_cast<double (*)[2 + SS_MAX_CUT]>(redbuf));
    if (tid == 0) {
      const bool none = nsel == 0;
      if (p.rmsd) p.rmsd[e] = none ? nanf_ : (float)sqrt(sums[0] / (3.0 * nsel));
      if (p.tm) p.tm[e] = none ? nanf_ : (float)(sums[1] / nsel);
      for (int g = 0; g < 2; ++g) {
        if (!p.gdt[g]) continue;
        float s = 0.f;
        for (int k = 0; k < p.gk[g]; ++k) s += __fdiv_rn((float)sums[2 + p.gidx[g][k]], (float)nsel) * p.gw[g][k];
        p.gdt[g][e] = none ? nanf_ : s / (float)p.gk[g];
      }
    }
  }
  // 4. lDDT: (score - 4) / (4 count - 4) in fp32 from the exact integer sums; 0 without a CA
  if (p.counts) {
    double v[2] = {0.0, 0.0};
    for (int i = tid; i < n; i += T) {
      int c = 0, s = 0;
      for (int k = 0; k < p.splits; ++k) {
        const int* q = p.counts + (((long long)k * gridDim.x + e) * n + i) * 2;
        c += q[0];
        s += q[1];
      }
      float l = 0.f;
      if (!mask || mask[i * msn]) {
        l = __fdiv_rn((float)s - 4.f, 4.f * (float)c - 4.f);
        if (isfinite(l)) { v[0] += l; v[1] += 1.0; }
      }
      p.lddt[(long long)e * n + i] = l;
    }
    if (p.lddt_mean) {
      block_sums<2>(v, reinterpret_cast<double (*)[2]>(redbuf));
      if (tid == 0) p.lddt_mean[e] = (float)(v[0] / v[1]);
    }
  }
}

}  // namespace af2
