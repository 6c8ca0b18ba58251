// Per-thread spline + factor math of the CUDA engine (fp64), host+device inline.
//
// What the reference computes per factor with four separate View calls
// (so3_spline_view.h:136-276,356-426; rd_spline_view.h:63-94;
// split_spline_view.h:67-214) is reorganised here GPU-first:
//   * everything that depends only on the knots — d_k = log(R_k^-1 R_k+1),
//     |d_k|, Jr^-1(d_k) — is computed ONCE per linearisation point into a
//     "knot-pair table" (KnotPair, 128 B per pair) that the residual kernels stage
//     in shared memory, instead of 3x per View call per factor;
//   * one `SideEval` = pose R(t), p(t), the 4 rotation Jacobian blocks, the 4
//     position weights and (optionally) body angular velocity / world velocity
//     at ONE evaluation time.  An image factor needs two (anchor, observation);
//     the visual kernel gives each to one lane of a lane pair;
//   * EvaluateRTp's Jacobian (left/world tangent) equals R(t) * EvaluateRp's
//     Jacobian (right/body tangent) — Jr(-phi) A^T-prefix == prefix Jr(phi) —
//     so both sides run the same code and the observation side folds R(t) into
//     its left factor (image_feature_factor.h:196).
#pragma once
#include "device_math.cuh"

namespace ctvio {

struct KnotPair {   // 16 doubles = 128 B
  double d[3];      // log(R_k^-1 R_{k+1})           (so3_spline_view.h:167)
  double theta;     // |d|
  double jrinv[9];  // rightJacobianInvSO3(d)        (so3_spline_view.h:174)
  double pad[3];
};

struct SplineParams {
  int64_t t0_ns, dt_ns;
  int32_t n_knots;
  double inv_dt;  // pow_inv_dt[1] = 1e9 / dt_ns (spline_segment.h:58)
};

// spline_segment.h:72-88 — int64 div/mod, u in [0,1)
CTVIO_HD bool spline_index(const SplineParams& sp, int64_t t, int32_t& s, double& u) {
  const int64_t st = t - sp.t0_ns;
  if (st < 0 || t >= sp.t0_ns + int64_t(sp.n_knots - 3) * sp.dt_ns) return false;
  const int64_t si = st / sp.dt_ns;
  s = int32_t(si);
  u = double(st - si * sp.dt_ns) / double(sp.dt_ns);
  return true;
}

// blending (spline_common.h:76-153 for N=4): rows of M / M_c against [1,u,u^2,u^3] and derivatives
CTVIO_HD void cum_coeffs(double u, double lam[4]) {  // M_c * U, lam[0] == 1
  const double u2 = u * u, u3 = u2 * u;
  const double k6 = 1.0 / 6.0;
  lam[0] = 1.0;
  lam[1] = (5.0 * k6) + (3.0 * k6) * u + (-3.0 * k6) * u2 + k6 * u3;
  lam[2] = k6 + (3.0 * k6) * u + (3.0 * k6) * u2 + (-2.0 * k6) * u3;
  lam[3] = k6 * u3;
}
CTVIO_HD void cum_dcoeffs(double u, double inv_dt, double dl[4]) {  // inv_dt * M_c * [0,1,2u,3u^2]
  const double u2 = u * u;
  const double k6 = 1.0 / 6.0;
  dl[0] = 0.0;
  dl[1] = inv_dt * ((3.0 * k6) + (-3.0 * k6) * (2.0 * u) + k6 * (3.0 * u2));
  dl[2] = inv_dt * ((3.0 * k6) + (3.0 * k6) * (2.0 * u) + (-2.0 * k6) * (3.0 * u2));
  dl[3] = inv_dt * (k6 * (3.0 * u2));
}
template <int D>
CTVIO_HD void plain_coeffs(double u, double inv_dt, double c[4]) {  // inv_dt^D * M * U^(D)
  const double k6 = 1.0 / 6.0;
  double U0, U1, U2, U3, sc;
  if (D == 0) { U0 = 1; U1 = u; U2 = u * u; U3 = u * u * u; sc = 1.0; }
  else if (D == 1) { U0 = 0; U1 = 1; U2 = 2 * u; U3 = 3 * u * u; sc = inv_dt; }
  else { U0 = 0; U1 = 0; U2 = 2; U3 = 6 * u; sc = inv_dt * inv_dt; }
  c[0] = sc * (k6 * U0 + (-3.0 * k6) * U1 + (3.0 * k6) * U2 + (-k6) * U3);
  c[1] = sc * ((4.0 * k6) * U0 + (-6.0 * k6) * U2 + (3.0 * k6) * U3);
  c[2] = sc * (k6 * U0 + (3.0 * k6) * U1 + (3.0 * k6) * U2 + (-3.0 * k6) * U3);
  c[3] = sc * (k6 * U3);
}

CTVIO_HD Q4 load_q(const double* q, int k) { return Q4{q[4 * k], q[4 * k + 1], q[4 * k + 2], q[4 * k + 3]}; }
template <int PS>
CTVIO_HD V3 load_p(const double* p, int k) { return V3{p[PS * k], p[PS * k + 1], p[PS * k + 2]}; }

// knot-pair table entry k from knots k, k+1
CTVIO_HD void make_knot_pair(const double* q, int k, KnotPair& out) {
  const V3 d = so3_log(so3_mul(q_conj(load_q(q, k)), load_q(q, k + 1)));
  out.d[0] = d.x; out.d[1] = d.y; out.d[2] = d.z;
  out.theta = sqrt(dot(d, d));
  const M3 J = right_jacobian_inv(d);
#pragma unroll
  for (int i = 0; i < 9; ++i) out.jrinv[i] = J.m[i];
  out.pad[0] = out.pad[1] = out.pad[2] = 0.0;
}

struct SideEval {
  int32_t s;       // global start knot
  M3 R;            // R(t)
  V3 p;            // p(t)
  M3 J[4];         // d R(t) / d delta_{s+k}, right tangent, "left factor omitted" (so3_spline_view.h:128-135)
  double c[4];     // d p(t) / d P_{s+k}
  V3 omega, vel;   // body angular velocity, world linear velocity (only when want_jac)
};

// One pose evaluation with Jacobians.  q/p/table may live in shared or global memory.
//   WANT_JAC=false reproduces the `jacobians == nullptr` path of the factors (value only).
//   PS = stride (doubles) of the position array: 3 on the host ABI, 4 in HBM/shared memory.
template <bool WANT_JAC, int PS>
CTVIO_HD void eval_side(const SplineParams& sp, const double* q, const double* p, const KnotPair* tab, int32_t s,
                        double u, SideEval& o) {
  o.s = s;
  double lam[4];
  cum_coeffs(u, lam);
  // E_j = exp(-lam_j d_{j-1}), accumulated exactly like EvaluateRp: A_accum_inv *= exp(-k delta), i = 2,1,0
  Q4 E[3];
  V3 phi[3];
#pragma unroll
  for (int j = 0; j < 3; ++j) {
    const KnotPair& kp = tab[s + j];
    const double l = lam[j + 1];
    phi[j] = V3{l * kp.d[0], l * kp.d[1], l * kp.d[2]};
    const double th = fabs(l) * kp.theta;
    E[j] = so3_exp_theta(neg(phi[j]), th * th, th);
  }
  const Q4 B3 = E[2];
  const Q4 B32 = so3_mul(B3, E[1]);
  const Q4 B321 = so3_mul(B32, E[0]);
  o.R = so3_matrix(so3_mul(load_q(q, s), q_conj(B321)));
  double c[4];
  plain_coeffs<0>(u, sp.inv_dt, c);
  V3 pp = c[0] * load_p<PS>(p, s);
#pragma unroll
  for (int k = 1; k < 4; ++k) pp = pp + c[k] * load_p<PS>(p, s + k);
  o.p = pp;
#pragma unroll
  for (int k = 0; k < 4; ++k) o.c[k] = c[k];
  if (!WANT_JAC) return;

  // J_0 = P0; H_i = lam_{i+1} P_{i+1} Jr(phi_i);  J_i -= H_i JrInv_i^T;  J_{i+1} = H_i JrInv_i   (so3_spline_view.h:183-195)
  const M3 P0 = so3_matrix(B321), P1 = so3_matrix(B32), P2 = so3_matrix(B3);
  M3 Jr[3];
#pragma unroll
  for (int j = 0; j < 3; ++j) Jr[j] = right_jacobian(phi[j]);
  M3 JI[3];
#pragma unroll
  for (int j = 0; j < 3; ++j)
#pragma unroll
    for (int e = 0; e < 9; ++e) JI[j].m[e] = tab[s + j].jrinv[e];
  const M3 H0 = m3_scale(lam[1], m3_mul(P1, Jr[0]));
  const M3 H1 = m3_scale(lam[2], m3_mul(P2, Jr[1]));
  const M3 H2 = m3_scale(lam[3], Jr[2]);
  o.J[0] = m3_sub(P0, m3_mul_bt(H0, JI[0]));
  o.J[1] = m3_sub(m3_mul(H0, JI[0]), m3_mul_bt(H1, JI[1]));
  o.J[2] = m3_sub(m3_mul(H1, JI[1]), m3_mul_bt(H2, JI[2]));
  o.J[3] = m3_mul(H2, JI[2]);

  // body angular velocity (VelocityBody value path, so3_spline_view.h:401-411)
  double dl[4];
  cum_dcoeffs(u, sp.inv_dt, dl);
  V3 w = V3{dl[1] * tab[s].d[0], dl[1] * tab[s].d[1], dl[1] * tab[s].d[2]};
#pragma unroll
  for (int j = 1; j < 3; ++j) {
    const KnotPair& kp = tab[s + j];
    w = so3_rotate(E[j], w) + V3{dl[j + 1] * kp.d[0], dl[j + 1] * kp.d[1], dl[j + 1] * kp.d[2]};
  }
  o.omega = w;
  double c1[4];
  plain_coeffs<1>(u, sp.inv_dt, c1);
  V3 vv = c1[0] * load_p<PS>(p, s);
#pragma unroll
  for (int k = 1; k < 4; ++k) vv = vv + c1[k] * load_p<PS>(p, s + k);
  o.vel = vv;
}

// ---- two-stage form of eval_side for the fused visual kernel -------------------------------------------
// Stage A (pose_stage) produces what the partner lane needs (R, p, omega, vel) and keeps only the three
// incremental quaternions E_j = exp(-lam_j d_j); stage B (jacobian_stage) regenerates the Jacobian blocks one
// knot at a time and hands each to `emit`, so that the 4 x 3x3 blocks never sit in registers together with
// the exchanged pose.  Jr(phi) is rebuilt from the half-angle sine/cosine already inside E_j
// (1 - cos t = 2 sin^2(t/2), sin t = 2 sin(t/2) cos(t/2)): no second sincos.
struct PoseStage {
  int32_t s;
  double lam[4];
  Q4 E[3];
  M3 R;
  V3 p;
  double c[4];
  V3 omega, vel;
};

template <bool WANT_JAC, int PS>
CTVIO_HD void pose_stage(const SplineParams& sp, const double* q, const double* p, const KnotPair* tab, int32_t s,
                         double u, PoseStage& o) {
  o.s = s;
  cum_coeffs(u, o.lam);
#pragma unroll
  for (int j = 0; j < 3; ++j) {
    const KnotPair& kp = tab[s + j];
    const double l = o.lam[j + 1];
    const double th = fabs(l) * kp.theta;
    o.E[j] = so3_exp_theta(V3{-l * kp.d[0], -l * kp.d[1], -l * kp.d[2]}, th * th, th);
  }
  const Q4 B321 = so3_mul(so3_mul(o.E[2], o.E[1]), o.E[0]);
  o.R = so3_matrix(so3_mul(load_q(q, s), q_conj(B321)));
  plain_coeffs<0>(u, sp.inv_dt, o.c);
  V3 pp = o.c[0] * load_p<PS>(p, s);
#pragma unroll
  for (int k = 1; k < 4; ++k) pp = pp + o.c[k] * load_p<PS>(p, s + k);
  o.p = pp;
  if (!WANT_JAC) return;
  double dl[4];
  cum_dcoeffs(u, sp.inv_dt, dl);
  V3 w = V3{dl[1] * tab[s].d[0], dl[1] * tab[s].d[1], dl[1] * tab[s].d[2]};
#pragma unroll
  for (int j = 1; j < 3; ++j) {
    const KnotPair& kp = tab[s + j];
    w = so3_rotate(o.E[j], w) + V3{dl[j + 1] * kp.d[0], dl[j + 1] * kp.d[1], dl[j + 1] * kp.d[2]};
  }
  o.omega = w;
  double c1[4];
  plain_coeffs<1>(u, sp.inv_dt, c1);
  V3 vv = c1[0] * load_p<PS>(p, s);
#pragma unroll
  for (int k = 1; k < 4; ++k) vv = vv + c1[k] * load_p<PS>(p, s + k);
  o.vel = vv;
}

// rightJacobianSO3(phi) with phi = lam * d and the half-angle values held by E = exp(-phi):
// E.w = cos(|phi|/2), |E.xyz| = sin(|phi|/2)  (Taylor branch like utils/sophus_utils.hpp:165-199)
CTVIO_HD M3 right_jacobian_from_half(V3 phi, const Q4& Eneg) {
  const double n2 = dot(phi, phi);
  if (n2 > kSo3Eps) {
    const double n = sqrt(n2);
    const double sh = sqrt(Eneg.x * Eneg.x + Eneg.y * Eneg.y + Eneg.z * Eneg.z), ch = Eneg.w;
    const double one_minus_cos = 2.0 * sh * sh, sn = 2.0 * sh * ch;
    return rodrigues_like(phi, n2, -one_minus_cos / n2, (n - sn) / (n2 * n));
  }
  return rodrigues_like(phi, n2, -0.5, 1.0 / 6.0);
}

template <class Emit>
CTVIO_HD void jacobian_stage(const KnotPair* tab, const PoseStage& ps, Emit&& emit) {
  const int s = ps.s;
  M3 Hprev;  // H_{k-1} * JrInv_{k-1}
  {
    const Q4 B32 = so3_mul(ps.E[2], ps.E[1]);
    const Q4 B321 = so3_mul(B32, ps.E[0]);
    const KnotPair& kp = tab[s];
    const V3 phi = V3{ps.lam[1] * kp.d[0], ps.lam[1] * kp.d[1], ps.lam[1] * kp.d[2]};
    M3 JI;
#pragma unroll
    for (int e = 0; e < 9; ++e) JI.m[e] = kp.jrinv[e];
    const M3 H0 = m3_scale(ps.lam[1], m3_mul(so3_matrix(B32), right_jacobian_from_half(phi, ps.E[0])));
    emit(0, m3_sub(so3_matrix(B321), m3_mul_bt(H0, JI)));
    Hprev = m3_mul(H0, JI);
  }
  {
    const KnotPair& kp = tab[s + 1];
    const V3 phi = V3{ps.lam[2] * kp.d[0], ps.lam[2] * kp.d[1], ps.lam[2] * kp.d[2]};
    M3 JI;
#pragma unroll
    for (int e = 0; e < 9; ++e) JI.m[e] = kp.jrinv[e];
    const M3 H1 = m3_scale(ps.lam[2], m3_mul(so3_matrix(ps.E[2]), right_jacobian_from_half(phi, ps.E[1])));
    emit(1, m3_sub(Hprev, m3_mul_bt(H1, JI)));
    Hprev = m3_mul(H1, JI);
  }
  {
    const KnotPair& kp = tab[s + 2];
    const V3 phi = V3{ps.lam[3] * kp.d[0], ps.lam[3] * kp.d[1], ps.lam[3] * kp.d[2]};
    M3 JI;
#pragma unroll
    for (int e = 0; e < 9; ++e) JI.m[e] = kp.jrinv[e];
    const M3 H2 = m3_scale(ps.lam[3], right_jacobian_from_half(phi, ps.E[2]));
    emit(2, m3_sub(Hprev, m3_mul_bt(H2, JI)));
    emit(3, m3_mul(H2, JI));
  }
}

struct RigParams {
  M3 R_CI;     // S_CtoI.matrix()
  V3 p_CI;     // p_CinI
  double w_img;  // sqrt_info = w * I2
  V3 gravity;
  double imu_info[6];
};

// What one lane of an image-factor lane pair needs from its partner.
struct SideShare {
  M3 R;
  V3 p, omega, vel;
};

struct ImageCommon {   // quantities both lanes compute identically
  double r[2];         // weighted residual (before the loss)
  double JvR[6];       // W * J_v * R_GtoCj, 2x3 row-major
  double Jv[6];        // W * J_v
  V3 p_Ii, dp, xci;
  double sqrt_rho1, cost;
};

// image_feature_factor.h:104-163 given both pose evaluations
CTVIO_HD void image_common(const RigParams& rig, const double pi_xy[2], const double pj_xy[2], double rho,
                           const M3& R_i, V3 p_i, const M3& R_j, V3 p_j, double cauchy_a, ImageCommon& o) {
  o.xci = V3{pi_xy[0] / rho, pi_xy[1] / rho, 1.0 / rho};
  o.p_Ii = m3_vec(rig.R_CI, o.xci) + rig.p_CI;
  const V3 p_G = m3_vec(R_i, o.p_Ii) + p_i;
  o.dp = p_G - p_j;
  // x_j = R_IC (R_j^T dp) - R_IC p_CI
  const V3 x_j = m3_tvec(rig.R_CI, m3_tvec(R_j, o.dp) - rig.p_CI);
  const double dinv = 1.0 / x_j.z;
  const double w = rig.w_img;
  double r0 = w * (x_j.x * dinv - pj_xy[0]);
  double r1 = w * (x_j.y * dinv - pj_xy[1]);
  // loss (Ceres CauchyLoss + Corrector; marginalization_factor.cpp:39-67).  rho'' < 0 always -> sqrt(rho') scaling
  double srho = 1.0;
  const double s = r0 * r0 + r1 * r1;
  if (cauchy_a > 0.0) {
    const double b = cauchy_a * cauchy_a;
    const double sum = 1.0 + s / b;
    o.cost = 0.5 * b * log(sum);
    srho = sqrt(1.0 / sum);
  } else {
    o.cost = 0.5 * s;
  }
  o.sqrt_rho1 = srho;
  o.r[0] = srho * r0;
  o.r[1] = srho * r1;
  const double ws = w * srho;
  o.Jv[0] = ws * dinv; o.Jv[1] = 0.0; o.Jv[2] = -ws * dinv * dinv * x_j.x;
  o.Jv[3] = 0.0; o.Jv[4] = ws * dinv; o.Jv[5] = -ws * dinv * dinv * x_j.y;
  // R_GtoCj = R_CI^T R_j^T ;  JvR = Jv * R_CI^T * R_j^T
  double t[6];
#pragma unroll
  for (int r = 0; r < 2; ++r)
#pragma unroll
    for (int c = 0; c < 3; ++c)  // (Jv R_CI^T)_{rc} = sum_k Jv[r][k] R_CI[c][k]
      t[3 * r + c] = o.Jv[3 * r] * rig.R_CI.m[3 * c] + o.Jv[3 * r + 1] * rig.R_CI.m[3 * c + 1] +
                     o.Jv[3 * r + 2] * rig.R_CI.m[3 * c + 2];
#pragma unroll
  for (int r = 0; r < 2; ++r)
#pragma unroll
    for (int c = 0; c < 3; ++c)
      o.JvR[3 * r + c] = t[3 * r] * R_j.m[3 * c] + t[3 * r + 1] * R_j.m[3 * c + 1] + t[3 * r + 2] * R_j.m[3 * c + 2];
}

CTVIO_HD void mul23_33(const double A[6], const M3& B, double out[6]) {
#pragma unroll
  for (int r = 0; r < 2; ++r)
#pragma unroll
    for (int c = 0; c < 3; ++c) out[3 * r + c] = A[3 * r] * B.m[c] + A[3 * r + 1] * B.m[3 + c] + A[3 * r + 2] * B.m[6 + c];
}

// Knot Jacobian blocks of one side (image_feature_factor.h:188-236).
//   side 0 (anchor):      rot_k = (-JvR R_i hat(p_Ii)) J_k ,  pos_k =  c_k JvR
//   side 1 (observation): rot_k = ( JvR hat(dp) R_j)   J_k ,  pos_k = -c_k JvR
// image_side_lhs returns the 2x3 left factor of the rotation blocks.
CTVIO_HD void image_side_lhs(int side, const ImageCommon& cm, const M3& R_me, double lhs[6]) {
  M3 jv;  // JvR as the top 2 rows of a 3x3 to reuse the m3 helpers
#pragma unroll
  for (int e = 0; e < 6; ++e) jv.m[e] = cm.JvR[e];
  jv.m[6] = jv.m[7] = jv.m[8] = 0.0;
  if (side == 0) {
    const M3 t = m3_mul_hat(m3_mul(jv, R_me), cm.p_Ii);
#pragma unroll
    for (int e = 0; e < 6; ++e) lhs[e] = -t.m[e];
  } else {
    const M3 t = m3_mul(m3_mul_hat(jv, cm.dp), R_me);
#pragma unroll
    for (int e = 0; e < 6; ++e) lhs[e] = t.m[e];
  }
}
// out: rot[4][6], pos[4][6] (2x3 row-major each)
CTVIO_HD void image_side_blocks(int side, const ImageCommon& cm, const SideEval& me, double rot[4][6], double pos[4][6]) {
  double lhs[6];
  image_side_lhs(side, cm, me.R, lhs);
  const double sgn = side == 0 ? 1.0 : -1.0;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    mul23_33(lhs, me.J[k], rot[k]);
#pragma unroll
    for (int e = 0; e < 6; ++e) pos[k][e] = sgn * me.c[k] * cm.JvR[e];
  }
}

// inverse depth (image_feature_factor.h:239-248):  JvR * ( -R_i R_CI x_ci / rho )
CTVIO_HD void image_jrho(const RigParams& rig, const ImageCommon& cm, const M3& R_i, double rho, double out[2]) {
  const V3 t = m3_vec(R_i, m3_vec(rig.R_CI, cm.xci));
  const V3 v = V3{-t.x / rho, -t.y / rho, -t.z / rho};
  out[0] = cm.JvR[0] * v.x + cm.JvR[1] * v.y + cm.JvR[2] * v.z;
  out[1] = cm.JvR[3] * v.x + cm.JvR[4] * v.y + cm.JvR[5] * v.z;
}

// line delay (image_feature_factor.h:251-264)
CTVIO_HD void image_jld(const RigParams& rig, const ImageCommon& cm, int rowi, int rowj, const M3& R_i, V3 om_i, V3 v_i,
                        const M3& R_j, V3 om_j, V3 v_j, double out[2]) {
  const double ri = double(rowi), rj = double(rowj);
  V3 Jx = m3_tvec(R_j, ri * v_i - rj * v_j);
  // rowj * hat(w_j)^T * R_j^T dp = -rowj * w_j x (R_j^T dp)
  const V3 a = m3_tvec(R_j, cm.dp);
  Jx = Jx - rj * cross(om_j, a);
  // rowi * R_j^T R_i (w_i x p_Ii)
  Jx = Jx + ri * m3_tvec(R_j, m3_vec(R_i, cross(om_i, cm.p_Ii)));
  const V3 y = m3_tvec(rig.R_CI, Jx);
  out[0] = cm.Jv[0] * y.x + cm.Jv[1] * y.y + cm.Jv[2] * y.z;
  out[1] = cm.Jv[3] * y.x + cm.Jv[4] * y.y + cm.Jv[5] * y.z;
}

// ------------------------------- IMU ------------------------------------------------------------
struct ImuEvalOut {
  int32_t s;
  double r[6];
  double Jrot[4][18];  // 6x3 row-major: rows 0-2 gyro (d omega / d delta), rows 3-5 accel
  double Jpos[4][18];  // rows 0-2 zero, rows 3-5 = lambda_a[k] R^T
  double cost;
};

// trajectory_value_factor.h:141-248 + split_spline_view.h:67-214
template <bool WANT_JAC, int PS>
CTVIO_HD void eval_imu(const SplineParams& sp, const RigParams& rig, const double* q, const double* p,
                       const KnotPair* tab, int32_t s, double u, const double gyro[3], const double accel[3],
                       const double bias[6], ImuEvalOut& o) {
  o.s = s;
  double lam[4], dl[4], ca[4];
  cum_coeffs(u, lam);
  cum_dcoeffs(u, sp.inv_dt, dl);
  plain_coeffs<2>(u, sp.inv_dt, ca);
  V3 acc = ca[0] * load_p<PS>(p, s);
#pragma unroll
  for (int k = 1; k < 4; ++k) acc = acc + ca[k] * load_p<PS>(p, s + k);
  Q4 E[3];
  V3 phi[3], d[3];
#pragma unroll
  for (int j = 0; j < 3; ++j) {
    const KnotPair& kp = tab[s + j];
    d[j] = V3{kp.d[0], kp.d[1], kp.d[2]};
    phi[j] = lam[j + 1] * d[j];
    const double th = fabs(lam[j + 1]) * kp.theta;
    E[j] = so3_exp_theta(neg(phi[j]), th * th, th);
  }
  const Q4 B3 = E[2];
  const Q4 B32 = so3_mul(B3, E[1]);
  const Q4 B321 = so3_mul(B32, E[0]);
  // omega recursion (split_spline_view.h:141-148)
  V3 om[4];
  om[0] = V3{0, 0, 0};
#pragma unroll
  for (int i = 0; i < 3; ++i) om[i + 1] = so3_rotate(E[i], om[i]) + dl[i + 1] * d[i];
  const Q4 Rinv_q = so3_mul(B321, q_conj(load_q(q, s)));
  const M3 Rinv = so3_matrix(Rinv_q);
  const V3 ag = acc + rig.gravity;
  const V3 a_body = so3_rotate(Rinv_q, ag);
  const V3 g = om[3];
  o.r[0] = rig.imu_info[0] * (g.x - (gyro[0] - bias[0]));
  o.r[1] = rig.imu_info[1] * (g.y - (gyro[1] - bias[1]));
  o.r[2] = rig.imu_info[2] * (g.z - (gyro[2] - bias[2]));
  o.r[3] = rig.imu_info[3] * (a_body.x - (accel[0] - bias[3]));
  o.r[4] = rig.imu_info[4] * (a_body.y - (accel[1] - bias[4]));
  o.r[5] = rig.imu_info[5] * (a_body.z - (accel[2] - bias[5]));
  double cs = 0;
#pragma unroll
  for (int k = 0; k < 6; ++k) cs += o.r[k] * o.r[k];
  o.cost = 0.5 * cs;
  if (!WANT_JAC) return;

  const M3 P[4] = {so3_matrix(B321), so3_matrix(B32), so3_matrix(B3), m3_identity()};  // A_post_inv
  M3 JrN[3], JI[3];  // Jr(-k delta), JrInv(d)
#pragma unroll
  for (int j = 0; j < 3; ++j) {
    JrN[j] = right_jacobian_from_half(neg(phi[j]), E[j]);  // Jr(-k delta) from the half-angle values in E_j
#pragma unroll
    for (int e = 0; e < 9; ++e) JI[j].m[e] = tab[s + j].jrinv[e];
  }
  // d omega / d d_j (split_spline_view.h:166-173)
  M3 dw[3];
  dw[0] = m3_scale(dl[1], P[1]);
#pragma unroll
  for (int i = 1; i < 3; ++i) {
    const M3 t = m3_mul(m3_mul_hat(P[i], om[i]), JrN[i]);
#pragma unroll
    for (int e = 0; e < 9; ++e) dw[i].m[e] = lam[i + 1] * t.m[e] + dl[i + 1] * P[i + 1].m[e];
  }
  M3 Jw[4], Ja[4];
#pragma unroll
  for (int k = 0; k < 4; ++k)
#pragma unroll
    for (int e = 0; e < 9; ++e) Jw[k].m[e] = Ja[k].m[e] = 0.0;
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    const M3 a = m3_mul_bt(dw[i], JI[i]), b = m3_mul(dw[i], JI[i]);
#pragma unroll
    for (int e = 0; e < 9; ++e) { Jw[i].m[e] -= a.m[e]; Jw[i + 1].m[e] += b.m[e]; }
  }
  // accel rows (split_spline_view.h:183-211); R_accum[i] = R_s A_1..A_i = R P_i
  const M3 R = m3_transpose(Rinv);
  const M3 lhs = m3_mul_hat(Rinv, ag);
  const M3 lR = m3_mul(lhs, R);  // lhs * R_accum[i] = lR * P_i
  {
    const M3 t = m3_mul(lR, P[0]);
#pragma unroll
    for (int e = 0; e < 9; ++e) Ja[0].m[e] += t.m[e];
  }
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    const M3 da = m3_scale(lam[i + 1], m3_mul(m3_mul(lR, P[i]), JrN[i]));
    const M3 a = m3_mul_bt(da, JI[i]), b = m3_mul(da, JI[i]);
#pragma unroll
    for (int e = 0; e < 9; ++e) { Ja[i].m[e] -= a.m[e]; Ja[i + 1].m[e] += b.m[e]; }
  }
#pragma unroll
  for (int k = 0; k < 4; ++k)
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        o.Jrot[k][3 * r + c] = rig.imu_info[r] * Jw[k].m[3 * r + c];
        o.Jrot[k][9 + 3 * r + c] = rig.imu_info[3 + r] * Ja[k].m[3 * r + c];
        o.Jpos[k][3 * r + c] = 0.0;
        o.Jpos[k][9 + 3 * r + c] = rig.imu_info[3 + r] * (ca[k] * Rinv.m[3 * r + c]);
      }
}

}  // namespace ctvio
