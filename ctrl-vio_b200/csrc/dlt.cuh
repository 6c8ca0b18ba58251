// DLT triangulation pieces shared by the two triangulation kernels of frontend.cu (triangulate_kernel: poses from the
// caller; triangulate_window_kernel: poses from the resident spline at each observation's row time).
//
// The reference runs Eigen::JacobiSVD on the tall 2m x 4 matrix (QR preconditioner + two-sided Jacobi on R).  Here one
// thread per landmark streams the rows through a Givens QR (R stays in registers, any number of frames) and then runs a
// one-sided Jacobi SVD on the 4x4 R: same conditioning as the reference (no A'A squaring), no local-memory arrays.
#pragma once
#include "device_math.cuh"

namespace ctvio {

struct R4 {
  double r[4][4];  // upper triangular
};

// fold one row a[4] into R with 4 Givens rotations
__device__ __forceinline__ void qr_push_row(R4& R, double a0, double a1, double a2, double a3) {
  double a[4] = {a0, a1, a2, a3};
#pragma unroll
  for (int c = 0; c < 4; ++c) {
    const double x = R.r[c][c], y = a[c];
    if (y == 0.0) continue;
    const double h = hypot(x, y);
    const double cs = x / h, sn = y / h;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      if (k < c) continue;
      const double rk = R.r[c][k], ak = a[k];
      R.r[c][k] = cs * rk + sn * ak;
      a[k] = -sn * rk + cs * ak;
    }
  }
}

// The two rows of one observation (feature_manager.cpp:252-261): camera pose (R1, t1) relative to the anchor camera
// (R0, t0), P = [R' | -R' t], bearing f normalised.
__device__ __forceinline__ void dlt_push_observation(R4& Rq, const M3& R0, const V3& t0, const M3& R1, const V3& t1, V3 f) {
  const V3 t = m3_tvec(R0, t1 - t0);
  const M3 R = m3_mul(m3_transpose(R0), R1);
  // P = [R' | -R' t]   (:255-257)
  const M3 Rt = m3_transpose(R);
  const V3 pt = neg(m3_vec(Rt, t));
  const double fn = sqrt(f.x * f.x + f.y * f.y + f.z * f.z);
  f = (1.0 / fn) * f;
  const double P0[4] = {Rt.m[0], Rt.m[1], Rt.m[2], pt.x};
  const double P1[4] = {Rt.m[3], Rt.m[4], Rt.m[5], pt.y};
  const double P2[4] = {Rt.m[6], Rt.m[7], Rt.m[8], pt.z};
  qr_push_row(Rq, f.x * P2[0] - f.z * P0[0], f.x * P2[1] - f.z * P0[1], f.x * P2[2] - f.z * P0[2],
              f.x * P2[3] - f.z * P0[3]);
  qr_push_row(Rq, f.y * P2[0] - f.z * P1[0], f.y * P2[1] - f.z * P1[1], f.y * P2[2] - f.z * P1[2],
              f.y * P2[3] - f.z * P1[3]);
}

// right singular vector of the smallest singular value of the upper triangular R (one-sided Jacobi, Hestenes)
__device__ __forceinline__ void smallest_right_singular_vector(const R4& R, double v_out[4]) {
  double G[4][4], V[4][4];  // column-major use: G[row][col]
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      G[i][j] = j >= i ? R.r[i][j] : 0.0;
      V[i][j] = i == j ? 1.0 : 0.0;
    }
  for (int sweep = 0; sweep < 40; ++sweep) {
    bool rotated = false;
#pragma unroll
    for (int p = 0; p < 3; ++p)
#pragma unroll
      for (int q = p + 1; q < 4; ++q) {
        double al = 0, be = 0, ga = 0;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          al = fma(G[i][p], G[i][p], al);
          be = fma(G[i][q], G[i][q], be);
          ga = fma(G[i][p], G[i][q], ga);
        }
        if (ga == 0.0 || fabs(ga) <= 1e-300 || fabs(ga) <= 2.3e-16 * sqrt(al * be)) continue;
        rotated = true;
        const double zeta = (be - al) / (2.0 * ga);
        const double t = (zeta >= 0 ? 1.0 : -1.0) / (fabs(zeta) + sqrt(1.0 + zeta * zeta));
        const double c = 1.0 / sqrt(1.0 + t * t), s = c * t;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const double gp = G[i][p], gq = G[i][q];
          G[i][p] = c * gp - s * gq;
          G[i][q] = s * gp + c * gq;
          const double vp = V[i][p], vq = V[i][q];
          V[i][p] = c * vp - s * vq;
          V[i][q] = s * vp + c * vq;
        }
      }
    if (!rotated) break;
  }
  int best = 0;
  double best_n = 1e300;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    double nj = 0;
#pragma unroll
    for (int i = 0; i < 4; ++i) nj = fma(G[i][j], G[i][j], nj);
    if (nj < best_n) { best_n = nj; best = j; }
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    // select without dynamic register indexing
    v_out[i] = best == 0 ? V[i][0] : best == 1 ? V[i][1] : best == 2 ? V[i][2] : V[i][3];
  }
}

}  // namespace ctvio
