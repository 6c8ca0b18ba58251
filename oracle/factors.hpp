// ORACLE (test infrastructure, NOT product code).  Parity unpinned (see so3.hpp).
// CPU fp64 restatement of the Ctrl-VIO cost functors.
//
// Restates:
//   factor/analytic_diff/image_feature_factor.h:63-269  ImageFeatureDelayFactor::Evaluate
//   factor/analytic_diff/trajectory_value_factor.h:141-248  IMUFactor::Evaluate
//   factor/analytic_diff/trajectory_value_factor.h:45-99    BiasFactor::Evaluate
//   factor/analytic_diff/marginalization_factor.cpp:326-373 MarginalizationFactor::Evaluate
//   marginalization_factor.cpp:39-67 + Ceres 1.14 corrector.cc / loss_function.cc
//        (CauchyLoss + Corrector; Ceres itself is not part of the reference repository)
// Jacobians are returned per GLOBAL knot (start index + 4 blocks per side)
// instead of the reference's padded parameter-block list; the unused padded
// blocks are identically zero there (image_feature_factor.h:165-180).
#pragma once
#include <cmath>
#include <limits>
#include <vector>

#include "spline.hpp"

namespace ctvio_oracle {

struct Calib {
  Quat S_CtoI;       // ImageFeatureDelayFactor::S_CtoI   (image_feature_factor.h:273)
  Vec3 p_CinI;       // ImageFeatureDelayFactor::p_CinI   (:274)
  double sqrt_info;  // image_weight (sqrt_info = w * I2, trajectory_manager.cpp:57)
  Vec3 gravity;
  double imu_info[6];  // opt_weight.h:124-126
};

struct ImageObs {
  int64_t ti, tj;
  int32_t rowi, rowj;
  double pi[2], pj[2];  // undistorted normalised coordinates, z == 1
  int32_t lm;           // landmark (inverse-depth) index
  int32_t marg;         // marg_this_feature flag
};

struct ImuObs {
  int64_t t;
  double gyro[3], accel[3];
  int32_t bias_idx;
  int32_t marg;
};

struct BiasObs {
  int32_t i, j;
  double sqrt_info[6];  // already divided by sqrt(dt) (trajectory_value_factor.h:41-43)
  int32_t marg;
};

struct ImageEval {
  double r[2];
  int64_t s[2];           // global start knot of side i / side j
  double Jrot[2][4][6];   // [side][knot k][2x3 row-major]  d r / d delta_rot(s+k)
  double Jpos[2][4][6];   // [side][knot k][2x3 row-major]  d r / d P(s+k)
  double Jrho[2];
  double Jld[2];
  bool ok;                // false if a time fell outside the spline
};

inline void mul23_33(const double A[6], const Mat3& B, double out[6]) {
  for (int r = 0; r < 2; ++r)
    for (int c = 0; c < 3; ++c) out[3 * r + c] = A[3 * r] * B(0, c) + A[3 * r + 1] * B(1, c) + A[3 * r + 2] * B(2, c);
}

// image_feature_factor.h:63-269.  want_jac == false reproduces the
// `jacobians == nullptr` path (no VelocityBody / velocity evaluation).
inline void EvaluateImage(const SplineGrid& g, const Calib& cal, const double* q, const double* p, double d_inv,
                          double l_delay, const ImageObs& o, bool want_jac, ImageEval& out) {
  const int64_t l_delay_ns = int64_t(l_delay * 1e9);  // truncation, :72
  const int64_t t_i = o.ti + int64_t(o.rowi) * l_delay_ns;
  const int64_t t_j = o.tj + int64_t(o.rowj) * l_delay_ns;
  int64_t si, sj; double u;
  out.ok = g.computeTIndexNs(t_i, si, u) && g.computeTIndexNs(t_j, sj, u);
  if (!out.ok) return;
  out.s[0] = si; out.s[1] = sj;

  const Vec3 p_i(o.pi[0], o.pi[1], 1.0);
  const Vec3 xci(p_i.x / d_inv, p_i.y / d_inv, p_i.z / d_inv);  // x_ci = p_i / d_inv, :104
  const Vec3 p_Ii = so3_rotate(cal.S_CtoI, xci) + cal.p_CinI;

  So3Jacobian J_R[2];
  RdJacobian J_p[2];
  Quat S_IitoG, S_GtoIj;
  Vec3 p_IiinG, p_IjinG, Omega_Ii, Omega_Ij, v_IiinG, v_IjinG;
  if (want_jac) {
    Omega_Ii = VelocityBody(g, q, t_i, nullptr);
    v_IiinG = RdEvaluate<1>(g, p, t_i, nullptr);
    S_IitoG = EvaluateRp(g, q, t_i, &J_R[0]);
    p_IiinG = RdEvaluate<0>(g, p, t_i, &J_p[0]);
  } else {
    S_IitoG = EvaluateRp(g, q, t_i, nullptr);
    p_IiinG = RdEvaluate<0>(g, p, t_i, nullptr);
  }
  const Vec3 p_G = so3_rotate(S_IitoG, p_Ii) + p_IiinG;
  if (want_jac) {
    Omega_Ij = VelocityBody(g, q, t_j, nullptr);
    v_IjinG = RdEvaluate<1>(g, p, t_j, nullptr);
    S_GtoIj = EvaluateRTp(g, q, t_j, &J_R[1]);
    p_IjinG = RdEvaluate<0>(g, p, t_j, &J_p[1]);
  } else {
    S_GtoIj = EvaluateRTp(g, q, t_j, nullptr);
    p_IjinG = RdEvaluate<0>(g, p, t_j, nullptr);
  }
  const Quat S_ItoC = cal.S_CtoI.conj();
  const Quat S_GtoCj = so3_mul(S_ItoC, S_GtoIj);
  const Vec3 dp = p_G - p_IjinG;
  const Vec3 x_j = so3_rotate(S_GtoCj, dp) - so3_rotate(S_ItoC, cal.p_CinI);
  const double depth_j_inv = 1.0 / x_j.z;
  out.r[0] = x_j.x * depth_j_inv - o.pj[0];
  out.r[1] = x_j.y * depth_j_inv - o.pj[1];

  if (want_jac) {
    const double w = cal.sqrt_info;
    double J_v[6] = {depth_j_inv, 0, -depth_j_inv * depth_j_inv * x_j.x,
                     0, depth_j_inv, -depth_j_inv * depth_j_inv * x_j.y};
    const Mat3 R_GtoCj = so3_matrix(S_GtoCj);
    const Mat3 R_CjIi = so3_matrix(so3_mul(S_GtoCj, S_IitoG));
    double JvR[6], JvRi[6], lhsR[2][6], lhsP[2][6];
    mul23_33(J_v, R_GtoCj, JvR);
    mul23_33(J_v, R_CjIi, JvRi);
    mul23_33(JvRi, hat(p_Ii), lhsR[0]);
    for (int k = 0; k < 6; ++k) lhsR[0][k] = -lhsR[0][k];
    for (int k = 0; k < 6; ++k) lhsP[0][k] = JvR[k];
    mul23_33(JvR, hat(dp), lhsR[1]);
    for (int k = 0; k < 6; ++k) lhsP[1][k] = -JvR[k];
    for (int seg = 0; seg < 2; ++seg) {
      for (int k = 0; k < 4; ++k) {
        double tmp[6];
        mul23_33(lhsR[seg], J_R[seg].d_val_d_knot[k], tmp);
        for (int e = 0; e < 6; ++e) out.Jrot[seg][k][e] = w * tmp[e];
        for (int e = 0; e < 6; ++e) out.Jpos[seg][k][e] = w * (J_p[seg].d_val_d_knot[k] * lhsP[seg][e]);
      }
    }
    // inverse depth, :239-248
    {
      const Quat S = so3_mul(so3_mul(S_GtoCj, S_IitoG), cal.S_CtoI);
      const Vec3 t = so3_matrix(S) * xci;
      const Vec3 J_Xm_d(-t.x / d_inv, -t.y / d_inv, -t.z / d_inv);
      out.Jrho[0] = w * (J_v[0] * J_Xm_d.x + J_v[1] * J_Xm_d.y + J_v[2] * J_Xm_d.z);
      out.Jrho[1] = w * (J_v[3] * J_Xm_d.x + J_v[4] * J_Xm_d.y + J_v[5] * J_Xm_d.z);
    }
    // line delay, :251-264
    {
      const Mat3 R_GtoIj = so3_matrix(S_GtoIj);
      const Mat3 R_IitoG = so3_matrix(S_IitoG);
      Vec3 J_x = so3_rotate(S_GtoIj, double(o.rowi) * v_IiinG - double(o.rowj) * v_IjinG);
      J_x = J_x + (double(o.rowj) * transpose(hat(Omega_Ij))) * (R_GtoIj * dp);
      J_x = J_x + (double(o.rowi) * (R_GtoIj * R_IitoG)) * (hat(Omega_Ii) * p_Ii);
      J_x = so3_rotate(S_ItoC, J_x);
      out.Jld[0] = w * (J_v[0] * J_x.x + J_v[1] * J_x.y + J_v[2] * J_x.z);
      out.Jld[1] = w * (J_v[3] * J_x.x + J_v[4] * J_x.y + J_v[5] * J_x.z);
    }
  }
  out.r[0] *= cal.sqrt_info;
  out.r[1] *= cal.sqrt_info;
}

// Ceres 1.14 CauchyLoss::Evaluate (loss_function.cc) with b = a^2.
inline void CauchyLoss(double a, double s, double rho[3]) {
  const double b = a * a, c = 1.0 / b;
  const double sum = 1.0 + s * c;
  const double inv = 1.0 / sum;
  rho[0] = b * std::log(sum);
  rho[1] = std::max(std::numeric_limits<double>::min(), inv);
  rho[2] = -c * (inv * inv);
}

// Ceres 1.14 Corrector (corrector.cc) == marginalization_factor.cpp:39-67.
struct Corrector {
  double sqrt_rho1, residual_scaling, alpha_sq_norm;
  Corrector(double sq_norm, const double rho[3]) {
    sqrt_rho1 = std::sqrt(rho[1]);
    if (sq_norm == 0.0 || rho[2] <= 0.0) {
      residual_scaling = sqrt_rho1;
      alpha_sq_norm = 0.0;
      return;
    }
    const double D = 1.0 + 2.0 * sq_norm * rho[2] / rho[1];
    const double alpha = 1.0 - std::sqrt(D);
    residual_scaling = sqrt_rho1 / (1 - alpha);
    alpha_sq_norm = alpha / sq_norm;
  }
};

// Applies the loss to a 2-residual visual block in place; returns the block's
// cost 0.5*rho(s).  J columns are corrected with the *uncorrected* residual
// (residual_block.cc order).
inline double ApplyLossImage(double cauchy_a, ImageEval& e, bool has_jac) {
  const double s = e.r[0] * e.r[0] + e.r[1] * e.r[1];
  double rho[3];
  CauchyLoss(cauchy_a, s, rho);
  Corrector c(s, rho);
  if (has_jac) {
    auto fix = [&](double& j0, double& j1) {
      const double rtj = e.r[0] * j0 + e.r[1] * j1;
      j0 = c.sqrt_rho1 * (j0 - c.alpha_sq_norm * e.r[0] * rtj);
      j1 = c.sqrt_rho1 * (j1 - c.alpha_sq_norm * e.r[1] * rtj);
    };
    for (int side = 0; side < 2; ++side)
      for (int k = 0; k < 4; ++k)
        for (int col = 0; col < 3; ++col) {
          fix(e.Jrot[side][k][col], e.Jrot[side][k][3 + col]);
          fix(e.Jpos[side][k][col], e.Jpos[side][k][3 + col]);
        }
    fix(e.Jrho[0], e.Jrho[1]);
    fix(e.Jld[0], e.Jld[1]);
  }
  e.r[0] *= c.residual_scaling;
  e.r[1] *= c.residual_scaling;
  return 0.5 * rho[0];
}

struct ImuEval {
  double r[6];
  int64_t s;
  double Jrot[4][18];  // 6x3 row-major per knot
  double Jpos[4][18];  // 6x3 row-major per knot
  double Jbg[6], Jba[6];  // diagonal entries: rows 0-2 -> bg, rows 3-5 -> ba  (:240-244)
  bool ok;
};

// trajectory_value_factor.h:141-248
inline void EvaluateImu(const SplineGrid& g, const Calib& cal, const double* q, const double* p, const double* bg,
                        const double* ba, const ImuObs& o, bool want_jac, ImuEval& out) {
  int64_t s; double u;
  out.ok = g.computeTIndexNs(o.t, s, u);
  if (!out.ok) return;
  out.s = s;
  So3Jacobian J_rot_w, J_rot_a;
  RdJacobian J_pos;
  SplineIMUData sd = want_jac ? SplitEvaluate(g, q, p, o.t, cal.gravity, &J_rot_w, &J_rot_a, &J_pos)
                              : SplitEvaluate(g, q, p, o.t, cal.gravity, nullptr, nullptr, nullptr);
  for (int k = 0; k < 3; ++k) {
    out.r[k] = sd.gyro[k] - (o.gyro[k] - bg[k]);
    out.r[3 + k] = sd.accel[k] - (o.accel[k] - ba[k]);
  }
  for (int k = 0; k < 6; ++k) out.r[k] = cal.imu_info[k] * out.r[k];
  if (!want_jac) return;
  const Mat3 Rinv = so3_matrix(sd.R_inv);
  for (int i = 0; i < 4; ++i) {
    for (int r = 0; r < 3; ++r)
      for (int c = 0; c < 3; ++c) {
        out.Jrot[i][3 * r + c] = cal.imu_info[r] * J_rot_w.d_val_d_knot[i](r, c);
        out.Jrot[i][9 + 3 * r + c] = cal.imu_info[3 + r] * J_rot_a.d_val_d_knot[i](r, c);
        out.Jpos[i][3 * r + c] = 0.0;
        out.Jpos[i][9 + 3 * r + c] = cal.imu_info[3 + r] * (J_pos.d_val_d_knot[i] * Rinv(r, c));
      }
  }
  for (int k = 0; k < 3; ++k) {
    out.Jbg[k] = cal.imu_info[k];
    out.Jbg[3 + k] = 0;
    out.Jba[k] = 0;
    out.Jba[3 + k] = cal.imu_info[3 + k];
  }
}

// trajectory_value_factor.h:45-99.  r = diag(s) [bg_j - bg_i; ba_j - ba_i].
inline void EvaluateBias(const double* bias_i, const double* bias_j, const BiasObs& o, double r[6]) {
  for (int k = 0; k < 6; ++k) r[k] = o.sqrt_info[k] * (bias_j[k] - bias_i[k]);
}

// Block kinds of the prior / marginalization bookkeeping.
enum BlockType { kBlkRot = 0, kBlkPos = 1, kBlkBg = 2, kBlkBa = 3, kBlkLd = 4, kBlkRho = 5 };
inline int blockGlobalSize(int type) { return type == kBlkRot ? 4 : (type == kBlkLd || type == kBlkRho) ? 1 : 3; }
inline int blockLocalSize(int type) { return (type == kBlkLd || type == kBlkRho) ? 1 : 3; }

struct PriorBlock {
  int32_t type;   // BlockType
  int32_t index;  // knot / bias node / landmark index (0 for ld)
  int32_t col;    // first column in J_lin (== keep_block_idx - m)
  double x0[4];   // keep_block_data (linearisation point)
};

struct Prior {
  int n = 0;
  std::vector<double> J;  // n x n row-major, linearized_jacobians
  std::vector<double> r;  // n, linearized_residuals
  std::vector<PriorBlock> blocks;
  bool valid() const { return n > 0; }
};

}  // namespace ctvio_oracle
