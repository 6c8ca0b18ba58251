// Host-side mirror of ctrlvio::TrajectoryEstimator (reference: src/estimator/trajectory_estimator.h:61-206,
// .cpp:97-408) on top of the C-ABI of include/ctvio.h.
//
// Same method names, argument order and meaning as the reference class so that
// TrajectoryManager::{UpdateTrajectory, UpdateVIOPrior, InitTrajectory}
// (src/estimator/trajectory_manager.cpp:122-483) keep their call sites; what changes is that Ceres parameter
// blocks (`double*` identity) become indices.  The adapter keeps the pointer -> index maps, so callers keep
// passing the same `double*` they pass today:
//   knot blocks      trajectory_->getKnotSO3(i).data() / getKnotPos(i).data()   -> knot index i
//   bias blocks      all_imu_bias_[t].gyro_bias.data() / accel_bias.data()      -> bias node index
//   para_Feature[k]                                                              -> landmark index k
//   &trajectory_->line_delay                                                     -> the line delay
// Header-only, C++17, no Eigen / Ceres / ROS: vectors and quaternions cross as plain arrays (Eigen maps bind to
// them without a copy: Eigen::Map<Eigen::Vector3d>(ptr)).
// Error behaviour: the reference aborts (assert / BASALT_ASSERT) on out-of-window times and otherwise ignores
// return values; here every failing C-ABI call throws ctvio::Error with ctvio_last_error().
#pragma once
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <functional>
#include <map>
#include <memory>
#include <stdexcept>
#include <algorithm>
#include <string>
#include <vector>

#include "../../include/ctvio.h"

namespace ctvio_host {

struct Error : std::runtime_error {
  int code;
  Error(int c, const std::string& what) : std::runtime_error(what), code(c) {}
};
inline void check(int rc, const char* where) {
  if (rc != CTVIO_OK) throw Error(rc, std::string(where) + ": " + ctvio_last_error());
}

// Minimal stand-in for the parts of ctrlvio::Trajectory (src/spline/trajectory.h:38-117, se3_spline.h) the
// estimator touches: knot storage with stable addresses, time grid, extrinsics, line-delay settings.
struct Trajectory {
  int64_t t0_ns = 0, dt_ns = 50000000;
  std::vector<double> knot_q;  // [n][4] xyzw   (so3_spline.h:410 keeps Sophus::SO3d knots in a deque)
  std::vector<double> knot_p;  // [n][3]
  double q_CtoI[4] = {0, 0, 0, 1}, p_CinI[3] = {0, 0, 0};
  double line_delay = 0, ld_lower = 0, ld_upper = 0;
  bool fix_ld = true;
  size_t numKnots() const { return knot_q.size() / 4; }
  int64_t minTimeNs() const { return t0_ns; }
  int64_t maxTimeNs() const { return t0_ns + int64_t(numKnots() - 3) * dt_ns; }
  size_t knotIndex(int64_t t) const { return size_t((t - t0_ns) / dt_ns); }  // computeTIndexNs(t).second
  double* getKnotSO3(size_t i) { return &knot_q[4 * i]; }
  double* getKnotPos(size_t i) { return &knot_p[3 * i]; }
  void SetLineDelay(double init, bool fix, double lo, double hi) { line_delay = init; fix_ld = fix; ld_lower = lo; ld_upper = hi; }
};

// trajectory_estimator_options.h:34-68 (fields the hot path reads)
struct TrajectoryEstimatorOptions {
  bool lock_traj = false, lock_ab = true, lock_wb = true;
  bool is_marg_state = false;
  int ctrl_to_be_opt_now = 0, ctrl_to_be_opt_later = 0;
};

// MarginalizationInfo payload in index form (marginalization_factor.h:96-131)
struct MarginalizationInfo {
  using Ptr = std::shared_ptr<MarginalizationInfo>;
  int n = 0;
  std::vector<double> linearized_jacobians, linearized_residuals, keep_block_data;  // n x n, n, nb x 4
  std::vector<int32_t> keep_block_type, keep_block_index, keep_block_idx;
};

// ResidualSummary (trajectory_estimator.h:38-58, .cpp:36-95): per residual type the number of blocks and the sum of
// |residual_i| (evaluated WITHOUT the loss, like cost_function->Evaluate in AddResidualInfo); err_ave = sum / num.
enum ResidualType { RType_IMU = 0, RType_Bias = 1, RType_Image = 2, RType_Prior = 3 };
struct ResidualSummary {
  int err_type_number[4] = {0, 0, 0, 0};
  std::vector<double> err_type_sum[4];
  std::string descri_info;
  void PrintSummary(FILE* f = stderr) const {
    static const char* names[4] = {"IMU", "Bias", "Image", "Prior"};
    if (err_type_number[0] + err_type_number[1] + err_type_number[2] + err_type_number[3] == 0) return;
    std::fprintf(f, "ResidualSummary :%s\n", descri_info.c_str());
    for (int t = 0; t < 4; ++t) {
      if (err_type_number[t] <= 0) continue;
      std::fprintf(f, "\t- %s: num = %d; err_ave = ", names[t], err_type_number[t]);
      for (size_t i = 0; i < err_type_sum[t].size(); ++i) std::fprintf(f, "%g, ", err_type_sum[t][i] / err_type_number[t]);
      std::fprintf(f, "\n");
    }
  }
};

struct SolverSummary {  // what callers log from ceres::Solver::Summary::BriefReport()
  int iterations = 0, num_successful_steps = 0, num_unsuccessful_steps = 0, termination = 0;
  double initial_cost = 0, final_cost = 0, device_ms = 0;
};

class TrajectoryEstimator {
 public:
  using Ptr = std::shared_ptr<TrajectoryEstimator>;

  // reference: TrajectoryEstimator(Trajectory::Ptr, TrajectoryEstimatorOptions&)   (trajectory_estimator.cpp:97)
  // image_weight / imu_info / gravity are the statics the reference injects through InitFactorInfo
  // (trajectory_manager.cpp:51-62), OptWeight (opt_weight.h:124-126) and gravity_.
  TrajectoryEstimator(std::shared_ptr<Trajectory> trajectory, const TrajectoryEstimatorOptions& option, double image_weight,
                      const double imu_info[6], const double gravity[3], int device = 0)
      : trajectory_(std::move(trajectory)), options(option) {
    ctvio_config cfg{};
    cfg.t0_ns = trajectory_->t0_ns;
    cfg.dt_ns = trajectory_->dt_ns;
    for (int k = 0; k < 4; ++k) cfg.q_CtoI[k] = trajectory_->q_CtoI[k];
    for (int k = 0; k < 3; ++k) { cfg.p_CinI[k] = trajectory_->p_CinI[k]; cfg.gravity[k] = gravity[k]; }
    for (int k = 0; k < 6; ++k) cfg.imu_info[k] = imu_info[k];
    cfg.image_weight = image_weight;
    cfg.rs_padding_ns = 39000000;  // trajectory_estimator.cpp:299
    cfg.cauchy_solve = 2.0;        // :321
    cfg.cauchy_marg = 1.0;
    cfg.device = device;
    check(ctvio_create(&cfg, &h_), "ctvio_create");
  }
  ~TrajectoryEstimator() { if (h_) ctvio_destroy(h_); }
  TrajectoryEstimator(const TrajectoryEstimator&) = delete;
  TrajectoryEstimator& operator=(const TrajectoryEstimator&) = delete;

  void SetFixedIndex(int idx) { fixed_control_point_index_ = idx; }  // trajectory_estimator.h:90
  // Sliding the window: the Trajectory handed to the constructor holds only the window's slice of control points; when
  // the slice moves, shift its time origin (the reference instead keeps one growing spline and freezes old knots,
  // trajectory_manager.cpp:352-361).  Knot / bias indices of the prior are relative to the slice.
  void SetTimeOrigin(int64_t t0_ns) { check(ctvio_set_time_origin(h_, t0_ns), "ctvio_set_time_origin"); }

  // trajectory_estimator.cpp:219-263
  void AddIMUMeasurementAnalytic(int64_t timestamp, const double gyro[3], const double accel[3], double* gyro_bias,
                                 double* accel_bias, bool marg_this_factor = false) {
    imu_t_.push_back(timestamp);
    for (int k = 0; k < 3; ++k) { imu_gyro_.push_back(gyro[k]); imu_accel_.push_back(accel[k]); }
    imu_node_.push_back(biasNode(gyro_bias, accel_bias));
    imu_marg_.push_back(options.is_marg_state && marg_this_factor ? 1 : 0);
  }
  // trajectory_estimator.cpp:265-291 (sqrt_info is divided by sqrt(dt) like BiasFactor's constructor)
  void AddBiasFactor(double* bias_gyr_i, double* bias_gyr_j, double* bias_acc_i, double* bias_acc_j, double dt,
                     const double info_vec[6], bool marg_this_factor = false) {
    bf_i_.push_back(biasNode(bias_gyr_i, bias_acc_i));
    bf_j_.push_back(biasNode(bias_gyr_j, bias_acc_j));
    for (int k = 0; k < 6; ++k) bf_s_.push_back(info_vec[k] / std::sqrt(dt));
    bf_marg_.push_back(options.is_marg_state && marg_this_factor ? 1 : 0);
  }
  // trajectory_estimator.cpp:293-332; pi / pj are the undistorted normalised points (x, y, 1)
  void AddImageFeatureDelayAnalytic(int64_t ti, int rowi, const double pi[3], int64_t tj, int rowj, const double pj[3],
                                    double* inv_depth, double* line_delay, bool /*fixed_depth*/, bool marg_this_feature) {
    (void)line_delay;  // always &trajectory_->line_delay
    img_ti_.push_back(ti); img_tj_.push_back(tj); img_rowi_.push_back(rowi); img_rowj_.push_back(rowj);
    img_pi_.push_back(pi[0]); img_pi_.push_back(pi[1]); img_pj_.push_back(pj[0]); img_pj_.push_back(pj[1]);
    img_lm_.push_back(landmark(inv_depth));
    img_marg_.push_back(options.is_marg_state && marg_this_feature ? 1 : 0);
  }
  // trajectory_estimator.cpp:334-348
  void AddMarginalizationFactor(const MarginalizationInfo::Ptr& last) { prior_ = last; }

  // ---- the reference's EXACT argument shapes (trajectory_estimator.h:101-146), templated on anything that exposes
  //      .data() (Eigen::Vector3d, Eigen::Matrix<double,6,1>, std::array, ...) so that TrajectoryManager's call sites
  //      compile unchanged without Eigen being included here ----
  // AddIMUMeasurementAnalytic(const IMUData&, const Vector3d& gravity, double* bg, double* ba, const Vector6d& info, bool marg)
  template <class ImuData, class Vec3, class Vec6>
  auto AddIMUMeasurementAnalytic(const ImuData& imu_data, const Vec3& gravity, double* gyro_bias, double* accel_bias,
                                 const Vec6& info_vec, bool marg_this_factor = false)
      -> decltype(imu_data.timestamp, gravity.data(), info_vec.data(), void()) {
    (void)gravity; (void)info_vec;  // statics of the engine (ctvio_config.gravity / imu_info), checked once by the constructor
    AddIMUMeasurementAnalytic(int64_t(imu_data.timestamp), imu_data.gyro.data(), imu_data.accel.data(), gyro_bias, accel_bias,
                              marg_this_factor);
  }
  // AddBiasFactor(double*, double*, double*, double*, double dt, const Vector6d& info_vec, bool marg)
  template <class Vec6>
  auto AddBiasFactor(double* bias_gyr_i, double* bias_gyr_j, double* bias_acc_i, double* bias_acc_j, double dt,
                     const Vec6& info_vec, bool marg_this_factor = false) -> decltype(info_vec.data(), void()) {
    AddBiasFactor(bias_gyr_i, bias_gyr_j, bias_acc_i, bias_acc_j, dt, info_vec.data(), marg_this_factor);
  }
  // AddImageFeatureDelayAnalytic(int64 ti, int rowi, const Vector3d& pi, int64 tj, int rowj, const Vector3d& pj, double* inv_depth,
  //                              double* line_delay, bool fixed_depth, bool marg)
  template <class Vec3>
  auto AddImageFeatureDelayAnalytic(int64_t ti, int rowi, const Vec3& pi, int64_t tj, int rowj, const Vec3& pj, double* inv_depth,
                                    double* line_delay, bool fixed_depth = false, bool marg_this_feature = false)
      -> decltype(pi.data(), void()) {
    AddImageFeatureDelayAnalytic(ti, rowi, pi.data(), tj, rowj, pj.data(), inv_depth, line_delay, fixed_depth, marg_this_feature);
  }
  // AddMarginalizationFactor(MarginalizationInfo::Ptr, std::vector<double*>& parameter_blocks): the block list is implied by
  // the info's (kind, index) pairs; the vector is accepted for source compatibility
  void AddMarginalizationFactor(const MarginalizationInfo::Ptr& last, std::vector<double*>& /*parameter_blocks*/) { prior_ = last; }

  // PrepareMarginalizationInfo(RType_Prior, factor, NULL, parameter_blocks, drop_set) (trajectory_estimator.cpp:143-151,
  // trajectory_manager.cpp:166-203): the old prior takes part in the marginalization with an explicit drop set (indices
  // into its block list).  The engine derives the same drop set from options.ctrl_to_be_opt_now / _later and bias node 0
  // (prior.cu: ctvio_marginalize [1]); here the caller's set is CHECKED against that rule so that a divergence is loud.
  void PrepareMarginalizationInfo(ResidualType r_type, const MarginalizationInfo::Ptr& prior, const std::vector<int>& drop_set) {
    if (r_type != RType_Prior || !prior) throw Error(CTVIO_ERR_INVALID, "PrepareMarginalizationInfo: only the prior is recorded explicitly");
    std::vector<int> expect;
    for (size_t b = 0; b < prior->keep_block_type.size(); ++b) {
      const int t = prior->keep_block_type[b], i = prior->keep_block_index[b];
      const bool knot = t == CTVIO_BLK_ROT || t == CTVIO_BLK_POS;
      if ((knot && i >= options.ctrl_to_be_opt_now && i < options.ctrl_to_be_opt_later) ||
          ((t == CTVIO_BLK_BG || t == CTVIO_BLK_BA) && i == 0))
        expect.push_back(int(b));
    }
    std::vector<int> got = drop_set;
    std::sort(got.begin(), got.end());
    if (got != expect) throw Error(CTVIO_ERR_INVALID, "PrepareMarginalizationInfo: drop set differs from the window rule");
    prior_ = prior;
  }
  // SaveMarginalizationInfo(MarginalizationInfo::Ptr& out, std::vector<double*>& blocks_out) (trajectory_estimator.cpp:184-204)
  void SaveMarginalizationInfo(MarginalizationInfo::Ptr& marg_info_out, std::vector<double*>& marg_param_blocks_out) {
    marg_info_out = SaveMarginalizationInfo();
    marg_param_blocks_out.clear();
    if (!marg_info_out) return;
    for (size_t b = 0; b < marg_info_out->keep_block_type.size(); ++b)
      marg_param_blocks_out.push_back(blockPointer(marg_info_out->keep_block_type[b], marg_info_out->keep_block_index[b]));
  }
  // GetResidualSummary() (trajectory_estimator.h:168-171): evaluated on the device at the CURRENT state of the engine
  const ResidualSummary& GetResidualSummary() {
    upload();
    double sums[18];
    int32_t counts[4];
    std::vector<double> prior_sum(prior_ ? size_t(prior_->n) : 0);
    check(ctvio_residual_summary(h_, counts, sums, prior_sum.empty() ? nullptr : prior_sum.data()), "ctvio_residual_summary");
    residual_summary_ = ResidualSummary();
    residual_summary_.err_type_number[RType_Image] = counts[0];
    residual_summary_.err_type_sum[RType_Image].assign(sums, sums + 2);
    residual_summary_.err_type_number[RType_IMU] = counts[1];
    residual_summary_.err_type_sum[RType_IMU].assign(sums + 2, sums + 8);
    residual_summary_.err_type_number[RType_Bias] = counts[2];
    residual_summary_.err_type_sum[RType_Bias].assign(sums + 8, sums + 14);
    residual_summary_.err_type_number[RType_Prior] = counts[3];
    residual_summary_.err_type_sum[RType_Prior] = prior_sum;
    return residual_summary_;
  }
  // AddCallback (trajectory_estimator.cpp:350-365, CheckStateCallback): the reference prints the registered blocks after
  // every iteration.  The LM loop runs on the device; the callbacks are invoked once per Solve with the final state.
  void AddCallback(const std::vector<std::string>& descriptions, const std::vector<size_t>& block_size,
                   std::vector<double*>& param_block) {
    for (size_t i = 0; i < block_size.size(); ++i) callbacks_.push_back({descriptions[i], block_size[i], param_block[i]});
  }

  // trajectory_estimator.cpp:367-408 — uploads state + factors, solves in HBM, writes every block back in place
  SolverSummary Solve(int max_iterations = 50, bool /*progress*/ = false, int /*num_threads*/ = -1) {
    upload();
    ctvio_summary s{};
    check(ctvio_solve(h_, max_iterations, &s), "ctvio_solve");
    download();
    for (const auto& cb : callbacks_) {
      std::fprintf(stderr, "%s:", cb.name.c_str());
      for (size_t k = 0; k < cb.size; ++k) std::fprintf(stderr, " %g", cb.ptr[k]);
      std::fprintf(stderr, "\n");
    }
    SolverSummary out;
    out.iterations = s.iterations; out.num_successful_steps = s.num_successful_steps;
    out.num_unsuccessful_steps = s.num_unsuccessful_steps; out.termination = s.termination;
    out.initial_cost = s.initial_cost; out.final_cost = s.final_cost; out.device_ms = s.device_ms;
    return out;
  }

  // what ceres::Covariance (trajectory_estimator.h:23) computes for the camera-side blocks and the inverse depths, at
  // the current state (see ctvio_covariance): cov_cc [np][np] row-major in ctvio_normal_equations' column order,
  // var_rho [n_landmarks]; either may be null.  Returns rcond; throws ctvio_host::Error on a rank-deficient window.
  double GetCovariance(std::vector<double>* cov_cc, std::vector<double>* var_rho) {
    upload();
    const size_t np = 6 * (trajectory_->numKnots() + bias_nodes_.size()) + 1;
    if (cov_cc) cov_cc->assign(np * np, 0.0);
    if (var_rho) var_rho->assign(landmarks_.size(), 0.0);
    double rcond = 0.0;
    check(ctvio_covariance(h_, cov_cc ? cov_cc->data() : nullptr, var_rho ? var_rho->data() : nullptr, &rcond),
          "ctvio_covariance");
    return rcond;
  }

  // the covariance of the pose and velocity at n times t (ns), from the window covariance (see ctvio_pose_covariance):
  // cov12 [n][12][12] row-major over (dtheta, dp, domega, dv), of the body or (camera_frame) of the camera.  Knots
  // <= gauge_knot_index are held constant for this call only (-1: the options alone).  Returns rcond; throws
  // ctvio_host::Error on a rank-deficient window.
  double GetPoseCovariance(int n, const int64_t* t, int gauge_knot_index, bool camera_frame, double* cov12) {
    upload();
    double rcond = 0.0;
    check(ctvio_pose_covariance(h_, n, t, gauge_knot_index, camera_frame ? 1 : 0, cov12, &rcond),
          "ctvio_pose_covariance");
    return rcond;
  }

  // the covariance of the relative pose between t_a and t_b (ns) for n pairs, the pose at t_b in the frame of the pose
  // at t_a, from the window covariance (see ctvio_relative_pose_covariance): cov6 [n][6][6] row-major over (dtheta_ab,
  // dp_ab), of the body or (camera_frame) of the camera; cross6 [n][6][6] (may be null) the covariance of the two
  // poses' (dtheta, dp), rows a and columns b.  Knots <= gauge_knot_index are held constant for this call only (-1: the
  // options alone).  Returns rcond; throws ctvio_host::Error on a rank-deficient window.
  double GetRelativePoseCovariance(int n, const int64_t* t_a, const int64_t* t_b, int gauge_knot_index, bool camera_frame,
                                   double* cov6, double* cross6 = nullptr) {
    upload();
    double rcond = 0.0;
    check(ctvio_relative_pose_covariance(h_, n, t_a, t_b, gauge_knot_index, camera_frame ? 1 : 0, cov6, cross6, &rcond),
          "ctvio_relative_pose_covariance");
    return rcond;
  }

  // the covariance of the world points of n landmarks, each anchored at time t (ns) with the bearing (x, y, 1), from the
  // window covariance and the landmark-knot cross terms (see ctvio_point_covariance): cov9 [n][3][3] row-major, world
  // frame.  Knots <= gauge_knot_index are held constant for this call only (-1: the options alone).  Returns rcond;
  // throws ctvio_host::Error on a rank-deficient window.
  double GetPointCovariance(int n, const int32_t* landmark, const int64_t* t, const double* bearing_xy,
                            int gauge_knot_index, double* cov9) {
    upload();
    double rcond = 0.0;
    check(ctvio_point_covariance(h_, n, landmark, t, bearing_xy, gauge_knot_index, cov9, &rcond),
          "ctvio_point_covariance");
    return rcond;
  }

  // TrajectoryManager::double2vector (trajectory_manager.cpp:485-516): R0 row-major, t0; knots >= min_idx
  void GaugeRealign(int min_idx, const double R0[9], const double t0[3]) {
    check(ctvio_gauge_realign(h_, min_idx, R0, t0), "ctvio_gauge_realign");
    download();
  }

  // trajectory_estimator.cpp:184-204: every factor added with its marg flag (and the attached prior) is
  // recorded; returns nullptr when nothing can be kept
  MarginalizationInfo::Ptr SaveMarginalizationInfo() {
    upload();
    int32_t n = 0, nb = 0;
    check(ctvio_marginalize(h_, &n, &nb), "ctvio_marginalize");
    if (n <= 0) return nullptr;
    auto m = std::make_shared<MarginalizationInfo>();
    m->n = n;
    m->linearized_jacobians.resize(size_t(n) * n);
    m->linearized_residuals.resize(n);
    m->keep_block_type.resize(nb); m->keep_block_index.resize(nb); m->keep_block_idx.resize(nb);
    m->keep_block_data.resize(4 * size_t(nb));
    check(ctvio_get_prior(h_, m->linearized_jacobians.data(), m->linearized_residuals.data(), m->keep_block_type.data(),
                          m->keep_block_index.data(), m->keep_block_idx.data(), m->keep_block_data.data()),
          "ctvio_get_prior");
    return m;
  }

  // registration of the caller-owned blocks (the reference discovers them through AddParameterBlock)
  void RegisterBiasNodes(const std::vector<std::pair<double*, double*>>& bg_ba) { bias_nodes_ = bg_ba; }
  void RegisterLandmarks(const std::vector<double*>& inv_depths) { landmarks_ = inv_depths; }

  TrajectoryEstimatorOptions options;

 private:
  int biasNode(double* bg, double* ba) {
    for (size_t k = 0; k < bias_nodes_.size(); ++k)
      if (bias_nodes_[k].first == bg && bias_nodes_[k].second == ba) return int(k);
    bias_nodes_.emplace_back(bg, ba);
    return int(bias_nodes_.size()) - 1;
  }
  int landmark(double* inv_depth) {
    auto it = lm_index_.find(inv_depth);
    if (it != lm_index_.end()) return it->second;
    for (size_t k = 0; k < landmarks_.size(); ++k)
      if (landmarks_[k] == inv_depth) { lm_index_[inv_depth] = int(k); return int(k); }
    landmarks_.push_back(inv_depth);
    lm_index_[inv_depth] = int(landmarks_.size()) - 1;
    return int(landmarks_.size()) - 1;
  }
  double* blockPointer(int type, int index) {
    switch (type) {
      case CTVIO_BLK_ROT: return trajectory_->getKnotSO3(size_t(index));
      case CTVIO_BLK_POS: return trajectory_->getKnotPos(size_t(index));
      case CTVIO_BLK_BG: return bias_nodes_[size_t(index)].first;
      case CTVIO_BLK_BA: return bias_nodes_[size_t(index)].second;
      case CTVIO_BLK_LD: return &trajectory_->line_delay;
      default: return landmarks_[size_t(index)];
    }
  }
  void upload() {
    Trajectory& T = *trajectory_;
    ctvio_options o{};
    o.fixed_knot_index = fixed_control_point_index_;
    o.lock_traj = options.lock_traj; o.lock_wb = options.lock_wb; o.lock_ab = options.lock_ab;
    o.fix_ld = T.fix_ld; o.ld_lower = T.ld_lower; o.ld_upper = T.ld_upper;
    o.is_marg_state = options.is_marg_state;
    o.ctrl_to_be_opt_now = options.ctrl_to_be_opt_now; o.ctrl_to_be_opt_later = options.ctrl_to_be_opt_later;
    check(ctvio_set_options(h_, &o), "ctvio_set_options");
    check(ctvio_set_knots(h_, int32_t(T.numKnots()), T.knot_q.data(), T.knot_p.data()), "ctvio_set_knots");
    std::vector<double> b(6 * bias_nodes_.size()), r(landmarks_.size());
    for (size_t k = 0; k < bias_nodes_.size(); ++k)
      for (int c = 0; c < 3; ++c) { b[6 * k + c] = bias_nodes_[k].first[c]; b[6 * k + 3 + c] = bias_nodes_[k].second[c]; }
    for (size_t k = 0; k < landmarks_.size(); ++k) r[k] = *landmarks_[k];
    check(ctvio_set_biases(h_, int32_t(bias_nodes_.size()), b.data()), "ctvio_set_biases");
    check(ctvio_set_inv_depths(h_, int32_t(r.size()), r.data()), "ctvio_set_inv_depths");
    check(ctvio_set_line_delay(h_, T.line_delay), "ctvio_set_line_delay");
    check(ctvio_clear_factors(h_), "ctvio_clear_factors");
    if (!img_ti_.empty())
      check(ctvio_add_image_features(h_, int32_t(img_ti_.size()), img_ti_.data(), img_rowi_.data(), img_pi_.data(), img_tj_.data(),
                                     img_rowj_.data(), img_pj_.data(), img_lm_.data(), img_marg_.data()), "ctvio_add_image_features");
    if (!imu_t_.empty())
      check(ctvio_add_imu_measurements(h_, int32_t(imu_t_.size()), imu_t_.data(), imu_gyro_.data(), imu_accel_.data(),
                                       imu_node_.data(), imu_marg_.data()), "ctvio_add_imu_measurements");
    if (!bf_i_.empty())
      check(ctvio_add_bias_factors(h_, int32_t(bf_i_.size()), bf_i_.data(), bf_j_.data(), bf_s_.data(), bf_marg_.data()),
            "ctvio_add_bias_factors");
    if (prior_ && prior_->n > 0)
      check(ctvio_set_prior(h_, prior_->n, prior_->linearized_jacobians.data(), prior_->linearized_residuals.data(),
                            int32_t(prior_->keep_block_type.size()), prior_->keep_block_type.data(), prior_->keep_block_index.data(),
                            prior_->keep_block_idx.data(), prior_->keep_block_data.data()), "ctvio_set_prior");
    else
      check(ctvio_set_prior(h_, 0, nullptr, nullptr, 0, nullptr, nullptr, nullptr, nullptr), "ctvio_set_prior");
  }
  void download() {  // the reference's solver updates the caller's blocks in place
    Trajectory& T = *trajectory_;
    check(ctvio_get_knots(h_, T.knot_q.data(), T.knot_p.data()), "ctvio_get_knots");
    std::vector<double> b(6 * bias_nodes_.size()), r(landmarks_.size());
    if (!b.empty()) check(ctvio_get_biases(h_, b.data()), "ctvio_get_biases");
    if (!r.empty()) check(ctvio_get_inv_depths(h_, r.data()), "ctvio_get_inv_depths");
    for (size_t k = 0; k < bias_nodes_.size(); ++k)
      for (int c = 0; c < 3; ++c) { bias_nodes_[k].first[c] = b[6 * k + c]; bias_nodes_[k].second[c] = b[6 * k + 3 + c]; }
    for (size_t k = 0; k < landmarks_.size(); ++k) *landmarks_[k] = r[k];
    check(ctvio_get_line_delay(h_, &T.line_delay), "ctvio_get_line_delay");
  }

  std::shared_ptr<Trajectory> trajectory_;
  ctvio_handle h_ = nullptr;
  int fixed_control_point_index_ = -1;
  std::vector<std::pair<double*, double*>> bias_nodes_;
  std::vector<double*> landmarks_;
  std::map<double*, int> lm_index_;
  std::vector<int64_t> img_ti_, img_tj_, imu_t_;
  std::vector<int32_t> img_rowi_, img_rowj_, img_lm_, img_marg_, imu_node_, imu_marg_, bf_i_, bf_j_, bf_marg_;
  std::vector<double> img_pi_, img_pj_, imu_gyro_, imu_accel_, bf_s_;
  MarginalizationInfo::Ptr prior_;
  ResidualSummary residual_summary_;
  struct Callback { std::string name; size_t size; double* ptr; };
  std::vector<Callback> callbacks_;
};

}  // namespace ctvio_host
