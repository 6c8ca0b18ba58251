// ORACLE (test infrastructure, NOT product code).  Parity pinned for this file: tests/test_frontend_cpu.py checks it
// against numpy.linalg.svd (LAPACK) on the same inputs.
// Restates FeatureManager::triangulate(Rs, Ps, ric, tic) (visual_odometry/feature_manager.cpp:230-275; the
// identity-extrinsic overload :173-223 is ric = I, tic = 0).  The reference's Eigen::JacobiSVD is not part of
// the reference repository (Eigen 3.3 is an external dependency, README.md:15-20); the smallest right singular vector is unique
// up to sign and V(2)/V(3) is sign free, so any backward-stable SVD restates it: here a one-sided Jacobi (Hestenes)
// sweep on the full 2m x 4 matrix.
#pragma once
#include <cmath>
#include <cstdint>
#include <vector>

namespace ctvio_oracle {

inline void mat3_mul(const double* a, const double* b, double* c) {
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) c[3 * i + j] = a[3 * i] * b[j] + a[3 * i + 1] * b[3 + j] + a[3 * i + 2] * b[6 + j];
}

inline void triangulate(int n_frames, const double* Rs, const double* Ps, const double* ric, const double* tic, int nl,
                        const int32_t* start_frame, const int32_t* obs_offset, const double* obs_point, int window_size,
                        double init_depth, double* depth) {
  for (int l = 0; l < nl; ++l) {
    const int o0 = obs_offset[l], used = obs_offset[l + 1] - o0, imu_i = start_frame[l];
    if (!(used >= 2 && imu_i < window_size - 2)) continue;  // :236-238
    if (depth[l] > 0) continue;                              // :239-240
    if (imu_i < 0 || imu_i + used > n_frames) { depth[l] = init_depth; continue; }
    std::vector<double> A(size_t(2 * used) * 4);
    double R0[9], t0[3];
    mat3_mul(Rs + 9 * imu_i, ric, R0);                                                            // :246
    for (int r = 0; r < 3; ++r)
      t0[r] = Ps[3 * imu_i + r] + Rs[9 * imu_i + 3 * r] * tic[0] + Rs[9 * imu_i + 3 * r + 1] * tic[1] +
              Rs[9 * imu_i + 3 * r + 2] * tic[2];                                                 // :245
    for (int k = 0; k < used; ++k) {
      const int j = imu_i + k;
      double R1[9], t1[3];
      mat3_mul(Rs + 9 * j, ric, R1);
      for (int r = 0; r < 3; ++r)
        t1[r] = Ps[3 * j + r] + Rs[9 * j + 3 * r] * tic[0] + Rs[9 * j + 3 * r + 1] * tic[1] + Rs[9 * j + 3 * r + 2] * tic[2];
      double t[3], R[9];  // t = R0' (t1 - t0), R = R0' R1  (:252-253)
      for (int r = 0; r < 3; ++r) {
        t[r] = 0;
        for (int c = 0; c < 3; ++c) t[r] += R0[3 * c + r] * (t1[c] - t0[c]);
        for (int c = 0; c < 3; ++c) {
          double s = 0;
          for (int m = 0; m < 3; ++m) s += R0[3 * m + r] * R1[3 * m + c];
          R[3 * r + c] = s;
        }
      }
      double P[3][4];  // [R' | -R' t]  (:255-257)
      for (int r = 0; r < 3; ++r) {
        double s = 0;
        for (int c = 0; c < 3; ++c) { P[r][c] = R[3 * c + r]; s += R[3 * c + r] * t[c]; }
        P[r][3] = -s;
      }
      const double* pt = obs_point + 3 * size_t(o0 + k);
      const double fn = std::sqrt(pt[0] * pt[0] + pt[1] * pt[1] + pt[2] * pt[2]);
      const double f[3] = {pt[0] / fn, pt[1] / fn, pt[2] / fn};                                  // :258
      for (int c = 0; c < 4; ++c) {
        A[size_t(2 * k) * 4 + c] = f[0] * P[2][c] - f[2] * P[0][c];                               // :260
        A[size_t(2 * k + 1) * 4 + c] = f[1] * P[2][c] - f[2] * P[1][c];                           // :261
      }
    }
    // one-sided Jacobi on the columns of A; V accumulates the right singular vectors
    const int rows = 2 * used;
    double V[4][4] = {{1, 0, 0, 0}, {0, 1, 0, 0}, {0, 0, 1, 0}, {0, 0, 0, 1}};
    for (int sweep = 0; sweep < 60; ++sweep) {
      bool rotated = false;
      for (int p = 0; p < 3; ++p)
        for (int q = p + 1; q < 4; ++q) {
          long double al = 0, be = 0, ga = 0;
          for (int r = 0; r < rows; ++r) {
            al += (long double)A[size_t(r) * 4 + p] * A[size_t(r) * 4 + p];
            be += (long double)A[size_t(r) * 4 + q] * A[size_t(r) * 4 + q];
            ga += (long double)A[size_t(r) * 4 + p] * A[size_t(r) * 4 + q];
          }
          if (ga == 0 || std::fabs((double)ga) <= 1e-17 * std::sqrt((double)(al * be))) continue;
          rotated = true;
          const double zeta = double((be - al) / (2 * ga));
          const double tt = (zeta >= 0 ? 1.0 : -1.0) / (std::fabs(zeta) + std::sqrt(1.0 + zeta * zeta));
          const double c = 1.0 / std::sqrt(1.0 + tt * tt), s = c * tt;
          for (int r = 0; r < rows; ++r) {
            const double gp = A[size_t(r) * 4 + p], gq = A[size_t(r) * 4 + q];
            A[size_t(r) * 4 + p] = c * gp - s * gq;
            A[size_t(r) * 4 + q] = s * gp + c * gq;
          }
          for (int r = 0; r < 4; ++r) {
            const double vp = V[r][p], vq = V[r][q];
            V[r][p] = c * vp - s * vq;
            V[r][q] = s * vp + c * vq;
          }
        }
      if (!rotated) break;
    }
    int best = 0;
    double bn = 1e300;
    for (int c = 0; c < 4; ++c) {
      double s = 0;
      for (int r = 0; r < rows; ++r) s += A[size_t(r) * 4 + c] * A[size_t(r) * 4 + c];
      if (s < bn) { bn = s; best = c; }
    }
    double d = V[2][best] / V[3][best];  // :266-267
    if (!(d >= 0.1) || !std::isfinite(d)) d = init_depth;  // :268-271
    depth[l] = d;
  }
}

}  // namespace ctvio_oracle
