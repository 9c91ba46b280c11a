// The trRosetta inter-residue orientations (Yang et al., PNAS 2020) as labels for the angle heads (theta_logits, phi_logits,
// omega_logits of af2_angle_heads), and the heads' cross-entropies against them in one pass over the logits (DESIGN.md §4f).
//
//  xent_rows_kernel<AngleLabels>  distogram_loss.cuh's rows kernel over the three heads: per pair the labels of AngleLabels
//                                 and one fp32 log-sum-exp term per head, 48 B of partials per (element, row).
//  bucketed_angles_kernel         the three int64 label matrices [B][n][n] (grid-stride, one pair per thread, store-bound).
//
// Geometry, all in fp64 on the fp32 atoms, every operation an explicitly rounded intrinsic so that nvcc cannot contract it
// into an FMA (the oracle, oracle/angle_loss_oracle.py, evaluates the same expressions in the same order):
//   virtual CB   b = CA - N, c = C - CA, a = b x c, CB = ((-0.58273431 a + 0.56802827 b) - 0.54067466 c) + CA
//   contact      i != j and |CB_i - CB_j| <= 20 (a NaN distance is no contact)
//   theta_ij     dihedral(N_i, CA_i, CB_i, CB_j)      omega_ij  dihedral(CA_i, CB_i, CB_j, CA_j)
//   phi_ij       atan2(|v x w|, v . w), v = CA_i - CB_i, w = CB_j - CB_i
//   dihedral     the reference's get_dihedral_torch: u1 = c2 - c1, u2 = c3 - c2, u3 = c4 - c3,
//                atan2(((|u2| u1) . (u2 x u3)), ((u1 x u2) . (u2 x u3))), dot products summed from +0 x, y, then z
//   bucket       a head of nb buckets has K = nb - 1 bins: the number of edges below the angle (torch.bucketize, right =
//                False), edges -pi + (k + 1) (2 pi / K) (theta, omega) or (k + 1) (pi / K) (phi), k < K - 1, and the last
//                edge pi; no contact is nb - 1.
#pragma once
#include "common.cuh"
#include "distogram_loss.cuh"

namespace af2 {

constexpr double AG_PI = 3.141592653589793;      // fl(pi)
constexpr double AG_CONTACT = 20.0;

struct D3 {
  double x, y, z;
};
__device__ __forceinline__ D3 d3_load(const float* p) { return {(double)__ldg(p), (double)__ldg(p + 1), (double)__ldg(p + 2)}; }
__device__ __forceinline__ D3 d3_sub(D3 a, D3 b) { return {__dsub_rn(a.x, b.x), __dsub_rn(a.y, b.y), __dsub_rn(a.z, b.z)}; }
__device__ __forceinline__ D3 d3_scale(double s, D3 a) { return {__dmul_rn(s, a.x), __dmul_rn(s, a.y), __dmul_rn(s, a.z)}; }
__device__ __forceinline__ D3 d3_cross(D3 a, D3 b) {
  return {__dsub_rn(__dmul_rn(a.y, b.z), __dmul_rn(a.z, b.y)), __dsub_rn(__dmul_rn(a.z, b.x), __dmul_rn(a.x, b.z)),
          __dsub_rn(__dmul_rn(a.x, b.y), __dmul_rn(a.y, b.x))};
}
// summed from +0, as torch's .sum(dim=-1) in get_dihedral_torch is: a dot product of zeros is +0 (a planar dihedral +pi, never -pi)
__device__ __forceinline__ double d3_dot(D3 a, D3 b) {
  return __dadd_rn(__dadd_rn(__dadd_rn(0.0, __dmul_rn(a.x, b.x)), __dmul_rn(a.y, b.y)), __dmul_rn(a.z, b.z));
}
__device__ __forceinline__ double d3_norm(D3 a) { return __dsqrt_rn(d3_dot(a, a)); }

// the virtual CB of a residue from its N, CA and C
__device__ __forceinline__ D3 virtual_cb(D3 n, D3 ca, D3 c) {
  const D3 b = d3_sub(ca, n), cc = d3_sub(c, ca), a = d3_cross(b, cc);
  auto one = [](double ak, double bk, double ck, double cak) {
    return __dadd_rn(__dsub_rn(__dadd_rn(__dmul_rn(-0.58273431, ak), __dmul_rn(0.56802827, bk)), __dmul_rn(0.54067466, ck)), cak);
  };
  return {one(a.x, b.x, cc.x, ca.x), one(a.y, b.y, cc.y, ca.y), one(a.z, b.z, cc.z, ca.z)};
}

__device__ __forceinline__ double dihedral(D3 c1, D3 c2, D3 c3, D3 c4) {
  const D3 u1 = d3_sub(c2, c1), u2 = d3_sub(c3, c2), u3 = d3_sub(c4, c3);
  const D3 c23 = d3_cross(u2, u3);
  return atan2(d3_dot(d3_scale(d3_norm(u2), u1), c23), d3_dot(d3_cross(u1, u2), c23));
}

// the number of edges below v among K bins: edge k = lo + (k + 1) * step (k < K - 1), edge K - 1 = pi
__device__ __forceinline__ int angle_bin(double v, double lo, double step, int K) {
  int a = 0, b = K;
  while (a < b) {
    const int mid = (a + b) >> 1;
    const double edge = mid == K - 1 ? AG_PI : __dadd_rn(lo, __dmul_rn((double)(mid + 1), step));
    if (edge < v) a = mid + 1; else b = mid;
  }
  return a;
}

struct AngleFrame {                      // residue i: N, CA and the virtual CB
  D3 n, ca, cb;
};

__device__ __forceinline__ AngleFrame angle_frame(const float* r) {
  const D3 n = d3_load(r), ca = d3_load(r + 3);
  return {n, ca, virtual_cb(n, ca, d3_load(r + 6))};
}

// labels (theta, phi, omega) of pair (i, j), i != j given by the caller, for heads of nb[0..2] buckets
__device__ __forceinline__ void angle_labels(const AngleFrame& fi, const float* rj, bool same, const int* nb, int (&lab)[3]) {
  const D3 caj = d3_load(rj + 3);
  const D3 cbj = virtual_cb(d3_load(rj), caj, d3_load(rj + 6));
  const D3 w = d3_sub(cbj, fi.cb);
  if (same || !(d3_norm(w) <= AG_CONTACT)) {
    lab[0] = nb[0] - 1; lab[1] = nb[1] - 1; lab[2] = nb[2] - 1;
    return;
  }
  const double theta = dihedral(fi.n, fi.ca, fi.cb, cbj);
  const double omega = dihedral(fi.ca, fi.cb, cbj, caj);
  const D3 v = d3_sub(fi.ca, fi.cb);
  const double phi = atan2(d3_norm(d3_cross(v, w)), d3_dot(v, w));
  const int kt = nb[0] - 1, kp = nb[1] - 1, ko = nb[2] - 1;
  lab[0] = angle_bin(theta, -AG_PI, __ddiv_rn(2.0 * AG_PI, (double)kt), kt);
  lab[1] = angle_bin(phi, 0.0, __ddiv_rn(AG_PI, (double)kp), kp);
  lab[2] = angle_bin(omega, -AG_PI, __ddiv_rn(2.0 * AG_PI, (double)ko), ko);
}

// The rows kernel's label policy for the three angle heads
struct AngleLabels {
  static constexpr int H = 3;
  const float* bb;                       // [B][n][A][3]: atoms 0, 1, 2 are N, CA, C
  int A;
  int nb[3];
  struct Row {
    AngleFrame f;
    int i;
  };
  __device__ __forceinline__ Row row(int e, int i, int n) const { return {angle_frame(bb + ((long long)e * n + i) * A * 3), i}; }
  __device__ __forceinline__ void labels(const Row& r, int e, int j, int n, int (&lab)[3]) const {
    angle_labels(r.f, bb + ((long long)e * n + j) * A * 3, j == r.i, nb, lab);
  }
};

// labels[h][b][i][j]: angle_labels of (i, j), or ignore_index where mask[b][i] & mask[b][j] is false
__global__ void __launch_bounds__(256) bucketed_angles_kernel(const float* __restrict__ bb, int A, const unsigned char* __restrict__ mask,
                                                              int nb0, int nb1, int nb2, long long ignore_index, int B, int n,
                                                              long long* __restrict__ theta, long long* __restrict__ phi,
                                                              long long* __restrict__ omega) {
  const long long nn = (long long)n * n, T = (long long)B * nn;
  const int nb[3] = {nb0, nb1, nb2};
  for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < T; t += (long long)gridDim.x * blockDim.x) {
    const long long b = t / nn;
    const int i = (int)((t - b * nn) / n), j = (int)(t - b * nn - (long long)i * n);
    long long v[3] = {ignore_index, ignore_index, ignore_index};
    if (!mask || (mask[b * n + i] && mask[b * n + j])) {
      int lab[3];
      angle_labels(angle_frame(bb + (b * n + i) * A * 3), bb + (b * n + j) * A * 3, i == j, nb, lab);
      v[0] = lab[0]; v[1] = lab[1]; v[2] = lab[2];
    }
    theta[t] = v[0];
    phi[t] = v[1];
    omega[t] = v[2];
  }
}

}  // namespace af2
