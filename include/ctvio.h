/*
 * ctvio.h — C-ABI of the H100-native sliding-window continuous-time bundle
 * adjustment engine (libctvio_b200.so).
 *
 * This is the drop-in boundary for the ONE hot path of APRIL-ZJU/Ctrl-VIO:
 * everything behind `TrajectoryEstimator::Solve()` /
 * `TrajectoryEstimator::SaveMarginalizationInfo()`.  The reference has no FFI;
 * its seam is the C++ class `ctrlvio::TrajectoryEstimator`
 * (src/estimator/trajectory_estimator.h:61-206).  Each entry point below names
 * the reference interface it replaces (paths relative to the reference's src/).
 * Pointer identity of Ceres parameter blocks becomes INDEX identity: global
 * knot index, bias-node index, landmark index (SURVEY.md §8b).
 *
 * Conventions
 *   - plain C, no torch / CUDA types; all pointers are HOST pointers unless the
 *     name ends in `_device`.
 *   - quaternions are [x, y, z, w] (Eigen/Sophus coeff order, sophus_lib/so3.hpp:196).
 *   - times are int64 nanoseconds relative to the trajectory start.
 *   - every function returns CTVIO_OK (0) or a negative error code; the message
 *     is available from ctvio_last_error().  There is NO CPU fallback: without
 *     a usable CUDA device ctvio_create fails with CTVIO_ERR_NO_DEVICE.
 */
#ifndef CTVIO_H_
#define CTVIO_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define CTVIO_ABI_VERSION 1

enum {
  CTVIO_OK = 0,
  CTVIO_ERR_INVALID = -1,    /* bad argument / index out of range            */
  CTVIO_ERR_NO_DEVICE = -2,  /* no CUDA device / wrong architecture           */
  CTVIO_ERR_CUDA = -3,       /* CUDA runtime error (see ctvio_last_error)     */
  CTVIO_ERR_STATE = -4,      /* call sequence error (e.g. solve before state) */
  CTVIO_ERR_NCCL = -5,
  CTVIO_ERR_TIME_RANGE = -6  /* a factor time falls outside the spline (the reference asserts,
                                spline_segment.h:80) */
};

/* parameter-block kinds used by the prior (marginalization_factor.h keep_block_*) */
enum {
  CTVIO_BLK_ROT = 0, /* knot rotation, 4 stored / 3 tangent (ceres_local_param.h:125-166) */
  CTVIO_BLK_POS = 1, /* knot position, 3                                                   */
  CTVIO_BLK_BG = 2,  /* gyro bias of a bias node, 3                                        */
  CTVIO_BLK_BA = 3,  /* accel bias of a bias node, 3                                       */
  CTVIO_BLK_LD = 4,  /* camera line delay, 1                                               */
  CTVIO_BLK_RHO = 5  /* landmark inverse depth, 1                                          */
};

/* ceres::TerminationType / message analogue returned by ctvio_solve */
enum {
  CTVIO_TERM_NO_CONVERGENCE = 0, /* max_num_iterations reached */
  CTVIO_TERM_GRADIENT = 1,
  CTVIO_TERM_PARAMETER = 2,
  CTVIO_TERM_FUNCTION = 3,
  CTVIO_TERM_FAILURE = 4,
  CTVIO_TERM_MIN_RADIUS = 5
};

typedef struct ctvio_engine* ctvio_handle;

/* Static configuration of a trajectory + sensor rig.
 *   replaces: Trajectory ctor (spline/trajectory.h:45-53), InitFactorInfo
 *   (estimator/trajectory_manager.cpp:51-62: S_CtoI, p_CinI, sqrt_info),
 *   OptWeight::imu_info_vec (utils/opt_weight.h:124-126), gravity_
 *   (estimator/odometry_manager.cpp:423). */
typedef struct ctvio_config {
  int64_t t0_ns;          /* minTimeNs of knot 0                                  */
  int64_t dt_ns;          /* knot spacing (config/ct_odometry_tumrs.yaml:13 -> 50 ms) */
  double q_CtoI[4];       /* camera->IMU rotation, xyzw                           */
  double p_CinI[3];       /* camera position in IMU frame                         */
  double image_weight;    /* sqrt_info = image_weight * I2                        */
  double gravity[3];
  double imu_info[6];     /* 1/sigma_g x3, 1/sigma_a x3                           */
  int64_t rs_padding_ns;  /* rolling-shutter time padding, 39 ms (estimator.cpp:299) */
  double cauchy_solve;    /* CauchyLoss scale in Solve, 2 (estimator.cpp:321)     */
  double cauchy_marg;     /* CauchyLoss scale for marginalized features, 1        */
  int32_t device;         /* CUDA device ordinal                                  */
  int32_t reserved;
} ctvio_config;

/* Per-problem options.
 *   replaces: TrajectoryEstimatorOptions (estimator/trajectory_estimator_options.h:34-68),
 *   TrajectoryEstimator::SetFixedIndex (trajectory_estimator.h:90),
 *   Trajectory::SetLineDelay (spline/trajectory.h:55-62). */
typedef struct ctvio_options {
  int32_t fixed_knot_index; /* knots <= index are constant; -1 = none */
  int32_t lock_traj;
  int32_t lock_wb;          /* gyro biases constant  */
  int32_t lock_ab;          /* accel biases constant */
  int32_t fix_ld;           /* line delay constant   */
  int32_t is_marg_state;
  int32_t ctrl_to_be_opt_now;
  int32_t ctrl_to_be_opt_later;
  double ld_lower, ld_upper;
} ctvio_options;

/* ceres::Solver::Summary analogue (only what the caller logs / we measure). */
typedef struct ctvio_summary {
  int32_t iterations;             /* LM steps after iteration 0 (accepted + rejected + invalid) */
  int32_t num_successful_steps;   /* includes iteration 0, like Ceres */
  int32_t num_unsuccessful_steps;
  int32_t termination;            /* CTVIO_TERM_* */
  int32_t num_cost_evals;         /* cost-only passes over all residual blocks */
  int32_t num_jacobian_evals;     /* residual+Jacobian passes over all residual blocks */
  int32_t num_linear_solves;
  int32_t num_line_search_steps;
  double initial_cost, final_cost, final_radius;
  double device_ms;               /* CUDA-event time of the whole solve on the engine stream */
  int64_t kernel_launches;        /* kernels launched by this solve */
} ctvio_summary;

const char* ctvio_last_error(void);
int ctvio_abi_version(void);

/* lifecycle — replaces `new TrajectoryEstimator(trajectory, option)`
 * (estimator/trajectory_estimator.cpp:97-112); one engine may be reused across windows. */
int ctvio_create(const ctvio_config* cfg, ctvio_handle* out);
int ctvio_destroy(ctvio_handle h);
int ctvio_set_options(ctvio_handle h, const ctvio_options* opt);
/* Deterministic mode (also CTVIO_DETERMINISTIC=1 at ctvio_create): every kernel merges its per-CTA partial sums in block
 * order (a ticket) and all factor kernels run on one stream, so a solve and the prior built from it are bit-reproducible
 * run to run - like the reference's single-threaded sums (trajectory_estimator.cpp:379-383).  Slower (serialised flush);
 * off by default; single GPU only.  K5 and K7 are order-fixed in both modes. */
int ctvio_set_deterministic(ctvio_handle h, int32_t on);

/* state in — replaces the raw `double*` parameter blocks handed to
 * problem_->AddParameterBlock (estimator/trajectory_estimator.cpp:114-141,
 * 230-247, 305-318): knots of Trajectory, all_imu_bias_, para_Feature,
 * trajectory_->line_delay. Host -> HBM copies. */
int ctvio_set_knots(ctvio_handle h, int32_t n_knots, const double* q_xyzw, const double* p_xyz);
int ctvio_set_biases(ctvio_handle h, int32_t n_nodes, const double* bg_ba6);
int ctvio_set_inv_depths(ctvio_handle h, int32_t n_landmarks, const double* inv_depth);
int ctvio_set_line_delay(ctvio_handle h, double line_delay);
/* Sliding the window: the reference keeps ONE growing spline and freezes the control points below
 * fixed_control_point_index (estimator/trajectory_estimator.h:90, trajectory_manager.cpp:352-361); here the caller
 * uploads only the window's slice of control points and moves the time origin to the slice's first knot
 * (t0 must stay on the knot grid of ctvio_config.t0_ns / dt_ns). Factors and the prior are re-added by the caller
 * with knot / bias-node indices relative to the new slice. */
int ctvio_set_time_origin(ctvio_handle h, int64_t t0_ns);

/* state out — the solver updates the blocks in place in the reference; here
 * the caller reads them back. HBM -> host copies. */
int ctvio_get_knots(ctvio_handle h, double* q_xyzw, double* p_xyz);
int ctvio_get_biases(ctvio_handle h, double* bg_ba6);
int ctvio_get_inv_depths(ctvio_handle h, double* inv_depth);
int ctvio_get_line_delay(ctvio_handle h, double* line_delay);

/* factors.  `marg` arrays may be NULL (all zero). */
int ctvio_clear_factors(ctvio_handle h);
/* replaces TrajectoryEstimator::AddImageFeatureDelayAnalytic (estimator/trajectory_estimator.cpp:293-332),
 * batched: observation k links anchor (ti,rowi,pi) to (tj,rowj,pj) of landmark lm[k]. */
int ctvio_add_image_features(ctvio_handle h, int32_t n, const int64_t* ti, const int32_t* rowi,
                             const double* pi_xy, const int64_t* tj, const int32_t* rowj,
                             const double* pj_xy, const int32_t* landmark, const int32_t* marg);
/* replaces TrajectoryEstimator::AddIMUMeasurementAnalytic (:219-263), batched. */
int ctvio_add_imu_measurements(ctvio_handle h, int32_t n, const int64_t* t, const double* gyro_xyz,
                               const double* accel_xyz, const int32_t* bias_node, const int32_t* marg);
/* replaces TrajectoryEstimator::AddBiasFactor (:265-291); sqrt_info is already divided by sqrt(dt). */
int ctvio_add_bias_factors(ctvio_handle h, int32_t n, const int32_t* node_i, const int32_t* node_j,
                           const double* sqrt_info6, const int32_t* marg);
/* replaces TrajectoryEstimator::AddMarginalizationFactor (:334-348) +
 * MarginalizationInfo::{linearized_jacobians, linearized_residuals, keep_block_*}
 * (factor/analytic_diff/marginalization_factor.h:96-131).  n == 0 clears the prior. */
int ctvio_set_prior(ctvio_handle h, int32_t n, const double* J_lin_rowmajor, const double* r_lin,
                    int32_t n_blocks, const int32_t* blk_type, const int32_t* blk_index,
                    const int32_t* blk_col, const double* blk_x0_4);

/* replaces TrajectoryEstimator::Solve -> ceres::Solve (estimator/trajectory_estimator.cpp:367-408):
 * LM trust region, Jacobi scaling, Cauchy loss, bounds on the line delay; state is updated in HBM. */
int ctvio_solve(ctvio_handle h, int32_t max_iterations, ctvio_summary* summary);

/* replaces TrajectoryManager::double2vector (estimator/trajectory_manager.cpp:485-516):
 * 4-DoF (yaw + translation) re-alignment of knots >= min_idx to the pre-solve pose (R0 row-major, t0). */
int ctvio_gauge_realign(ctvio_handle h, int32_t min_idx, const double* R0_rowmajor9, const double* t0_xyz);

/* replaces TrajectoryEstimator::SaveMarginalizationInfo (:184-204) =
 * MarginalizationInfo::preMarginalize + marginalize over every factor added with marg != 0 and
 * the current prior (PrepareMarginalizationInfo, :143-182).  Returns CTVIO_OK and n_out == 0
 * when nothing can be kept (the reference hands back nullptr). */
int ctvio_marginalize(ctvio_handle h, int32_t* n_out, int32_t* n_blocks_out);
int ctvio_get_prior(ctvio_handle h, double* J_lin_rowmajor, double* r_lin, int32_t* blk_type,
                    int32_t* blk_index, int32_t* blk_col, double* blk_x0_4);
/* make the prior produced by ctvio_marginalize the active one (device-to-device, no host trip) */
int ctvio_adopt_prior(ctvio_handle h);

/* state snapshot in HBM (bench: re-run the same window without a host round trip) */
int ctvio_save_state(ctvio_handle h);
int ctvio_restore_state(ctvio_handle h);

/* ---- probes used by the parity tests (the reference's CostFunction::Evaluate seam) ---- */
/* Evaluate every image factor at the current state.
 *   replaces ImageFeatureDelayFactor::Evaluate (factor/analytic_diff/image_feature_factor.h:63-269)
 *   + the loss corrector.  Outputs (any may be NULL): r[2n], s[2n] global start knots (i-side, j-side),
 *   J[n][100]: [side][knot k][rot 2x3 row-major | pos 2x3 row-major] (96) + d/d rho (2) + d/d ld (2). */
int ctvio_eval_image_factors(ctvio_handle h, int32_t want_jacobians, double cauchy_scale, double* r,
                             int32_t* s, double* J, double* cost);
/* replaces IMUFactor::Evaluate (factor/analytic_diff/trajectory_value_factor.h:141-248).
 *   r[6n], s[n], J[n][156]: [knot k][rot 6x3 | pos 6x3] (144) + diag d/d bg (6) + diag d/d ba (6). */
int ctvio_eval_imu_factors(ctvio_handle h, int32_t want_jacobians, double* r, int32_t* s, double* J,
                           double* cost);
/* replaces ResidualSummary / TrajectoryEstimator::GetResidualSummary (estimator/trajectory_estimator.cpp:36-95, printed by every
 * UpdateVIOPrior :283): per residual type the number of blocks and the per-component sums of |r_i| evaluated WITHOUT the loss
 * at the current state.  counts4 = {image, imu, bias, prior}; err_sum18 = image[2] | imu[6] | bias[6] | pad[4];
 * prior_err_sum (may be NULL) receives the n sums of the active prior. */
int ctvio_residual_summary(ctvio_handle h, int32_t* counts4, double* err_sum18, double* prior_err_sum);
/* The structure the engine built for the current factor set (prepare's frame-pair order, work lists and landmark
 * layout), host-built or device-built alike, so that tests can compare the two builds.  The structure is built first
 * when the factor set changed.  out: int64 slab, *len: its capacity in int64 on entry, the length needed on return
 * (out == NULL: query only).  Layout:
 *   header[16]  n factors, n_desc (n, or 0 for factors with host payload), n_items, nL, n_schur_items, n_entries, np,
 *               n_marg (-1 before a ctvio_marginalize that built its blocks), n_imu_items, 0...
 *   desc[n_desc][4] (slot_i, slot_j, landmark, marg; sorted) | orig[n] (sorted position -> caller index)
 *   | K1 items[n_items][4] (start, count, wi0, wj0) | lo[nL] | hi[nL] | woff[nL + 1]
 *   | K4 items[n_schur_items][4] (ti, tj, first, count) | entries[n_entries][5] (l, lo, hi, 0, woff)
 *   | active[np + nL]
 *   | pos_cam[np] | pos_lm[nL] | marg_img[n_marg]      -- only when n_marg >= 0
 *   | K2 items[n_imu_items][4] (start, count, s, node): runs of IMU samples in sorted order
 * Traffic of the device-built structure (factors from ctvio_add_image_features_from_table): the add itself reads
 * nothing back; the build reads back one count block of 32 + 4 * ceil(n_knots / 32) bytes; ctvio_marginalize reads
 * back 8 + 4 * ceil(n_knots / 32) bytes for its image blocks.  This probe's own read-back is not counted. */
int ctvio_debug_structure(ctvio_handle h, int64_t* out, int64_t* len);
/* total cost 0.5*sum rho(|r|^2) of all factors incl. bias + prior at the current state */
int ctvio_eval_cost(ctvio_handle h, double* cost);
/* Schur-form normal equations at the current state: camera block H_cc (np x np, row-major, symmetric),
 * g_c (np), per-landmark h_l, g_l (n_landmarks each).  np = 6*n_knots + 6*n_bias + 1. */
int ctvio_normal_equations(ctvio_handle h, double* Hcc, double* gc, double* hl, double* gl, double* cost);
/* ctvio_covariance - marginal covariance of the window at the current state (ceres::Covariance with its defaults,
 *   apply_loss_function = true, which trajectory_estimator.h:23 makes available to the reference's callers).
 *   The matrix: H = J'J of the current factor set (image factors with the cauchy_solve loss applied as the solve
 *   applies it, IMU, bias and the active prior), the Gauss-Newton matrix the solve builds, without damping and without
 *   Jacobi scaling, in the tangent space of ctvio_normal_equations (3 columns per rotation).
 *   cov_cc (np x np, row-major, may be NULL): the camera-side block of H^-1, columns ordered as ctvio_normal_equations'
 *     H_cc, np = 6*n_knots + 6*n_bias + 1.  It is S^-1, S the landmark-reduced system (Schur-complement identity); the
 *     full inverse is never formed.  Exactly symmetric.
 *   var_rho (n_landmarks, may be NULL): the diagonal of H^-1 at the inverse depths, 1/h_l + v_l' S^-1 v_l with
 *     v_l = W_l / h_l, W_l the landmark's coupling row (its knot / bias range and the line delay).
 *   Dimensions the solve holds constant (knots <= fixed_knot_index, lock_traj, lock_wb, lock_ab, fix_ld) and dimensions
 *   no factor touches have zero rows and columns; a landmark no factor touches has variance 0 (Ceres returns zero
 *   covariance for constant blocks).
 *   rcond (may be NULL) = (min_i L_ii / max_i L_ii)^2, L the Cholesky factor of the Jacobi-scaled S over its free
 *   dimensions.  The call fails with CTVIO_ERR_STATE ("rank deficient") and writes nothing but rcond when the
 *   factorisation meets a non-positive or non-finite pivot, when a landmark with factors has h_l <= 0, or when
 *   rcond < 1e-14.  The threshold is Ceres' default min_reciprocal_condition_number, but the test is this pivot-ratio
 *   estimate, not Ceres' own rank test.  A window without a prior or fixed knots is always rank deficient (yaw and
 *   translation are unobservable).
 *   No side effects: state, prior, factor set and the LM driver's scalars are unchanged; a solve after the call is
 *   bitwise the solve without it in deterministic mode.  ctvio_transfer_stats counts the outputs copied (only those
 *   requested).
 *   Errors: CTVIO_ERR_STATE before the state is set and in sharded mode. */
int ctvio_covariance(ctvio_handle h, double* cov_cc, double* var_rho, double* rcond);
/* ctvio_pose_covariance - covariance of the pose and velocity at n times, from the window covariance of
 *   ctvio_covariance (same H, same rcond test and failure mode, same absence of side effects); the np x np matrix
 *   stays on the device.
 *   cov12[n][12][12] (row-major, exactly symmetric): the covariance of what ctvio_query_trajectory returns, in its
 *     order: dtheta (3, R(t) -> R(t) Exp(dtheta), the right / body perturbation of the knots), dp (3, world position),
 *     domega (3, body angular velocity), dv (3, world linear velocity).  It is J(t) Sigma_sub J(t)', Sigma_sub the
 *     24 x 24 block of the window covariance at the rotation and position dims of the four knots of t's segment, J(t)
 *     the spline's Jacobian with respect to them.
 *   camera_frame = 1: of the camera instead, R_c = R R_CI, p_c = p + R p_CI (the convention of
 *     ctvio_feature_table_map): dtheta_c = R_CI' dtheta, dp_c = dp - R [p_CI]x dtheta, domega_c = R_CI' domega,
 *     dv_c = dv - R [omega x p_CI]x dtheta - R [p_CI]x domega.
 *   gauge_knot_index: knots with index <= gauge_knot_index are held constant for this call only, on top of what the
 *     options hold constant (SetFixedIndex applied to the covariance problem alone); -1: the options alone.  A window
 *     whose solve fixes no knots (fixed_knot_index = -1) is rank deficient without it.
 *   A time whose four knots are all constant gets an exact zero matrix.
 *   rcond (may be NULL): as ctvio_covariance; on CTVIO_ERR_STATE "rank deficient" only rcond is written.
 *   Errors, checked before anything is launched, with nothing written: CTVIO_ERR_INVALID for a null handle, n < 0,
 *   a NULL t_ns or cov12 with n > 0, camera_frame not 0 or 1, gauge_knot_index outside -1 .. n_knots - 1;
 *   CTVIO_ERR_STATE in sharded mode or before the knots are set; CTVIO_ERR_TIME_RANGE for a time
 *   ctvio_query_trajectory does not accept.  n = 0 returns CTVIO_OK and launches nothing.
 *   ctvio_transfer_stats counts 8 n bytes up and 1152 n bytes down. */
int ctvio_pose_covariance(ctvio_handle h, int32_t n, const int64_t* t_ns, int32_t gauge_knot_index,
                          int32_t camera_frame, double* cov12, double* rcond);
/* ctvio_relative_pose_covariance - covariance of the relative pose between two times for n pairs (t_a_ns[k],
 *   t_b_ns[k]), the odometry edge between two keyframes, from the window covariance of ctvio_covariance (same H, same
 *   gauge argument, same rcond test and failure mode, same absence of side effects); the np x np matrix stays on the
 *   device.
 *   The poses at t_a and t_b are those of ctvio_pose_covariance: of the body, or with camera_frame = 1 of the camera
 *   (R_c = R R_CI, p_c = p + R p_CI), each perturbed as dtheta (right, R -> R Exp(dtheta)) and dp (world, additive).
 *   The relative pose is R_ab = R_a' R_b, p_ab = R_a' (p_b - p_a), perturbed as dtheta_ab (right, R_ab -> R_ab
 *   Exp(dtheta_ab)) and dp_ab (additive, in frame a):
 *     dtheta_ab = dtheta_b - R_ab' dtheta_a,   dp_ab = R_a' (dp_b - dp_a) + [p_ab]x dtheta_a  (first order).
 *   cov6[n][6][6] (row-major, exactly symmetric): the covariance of (dtheta_ab, dp_ab), G Sigma_U G' with U the union of
 *     the knots of t_a's and t_b's segments (4 to 8 knots, not contiguous when the segments are 4 or more knots apart),
 *     Sigma_U its block of the window covariance and G the relative-pose Jacobian with respect to those knots; a knot
 *     of both segments has one column, the sum of both contributions.  Unlike the absolute pose covariance it does not
 *     grow with the distance from the gauge, so it can weight an odometry edge.
 *   cross6[n][6][6] (may be NULL): Cov((dtheta_a, dp_a), (dtheta_b, dp_b)), rows a and columns b, in the convention of
 *     the first six rows and columns of ctvio_pose_covariance; with the two diagonal blocks of that call it gives the
 *     joint 12 x 12 covariance of the two poses.
 *   t_a > t_b and t_a == t_b are valid.  A pair whose knots are all constant gets exact zero matrices.
 *   rcond (may be NULL): as ctvio_covariance; on CTVIO_ERR_STATE "rank deficient" only rcond is written.
 *   Errors, checked before anything is launched, with nothing written: CTVIO_ERR_INVALID for a null handle, n < 0,
 *   a NULL t_a_ns, t_b_ns or cov6 with n > 0, camera_frame not 0 or 1, gauge_knot_index outside -1 .. n_knots - 1;
 *   CTVIO_ERR_STATE in sharded mode or before the knots are set; CTVIO_ERR_TIME_RANGE for a time
 *   ctvio_query_trajectory does not accept.  n = 0 returns CTVIO_OK and launches nothing.
 *   ctvio_transfer_stats counts 16 n bytes up and 288 n bytes down, 576 n with cross6. */
int ctvio_relative_pose_covariance(ctvio_handle h, int32_t n, const int64_t* t_a_ns, const int64_t* t_b_ns,
                                   int32_t gauge_knot_index, int32_t camera_frame, double* cov6, double* cross6,
                                   double* rcond);
/* ctvio_point_covariance - covariance of the world points of n anchored landmarks, from the window covariance of
 *   ctvio_covariance (same H, same gauge argument, same rcond test and failure mode, same absence of side effects);
 *   neither the np x np matrix nor the landmark couplings leave the device.
 *   Point k is landmark[k] (inverse depth rho) anchored at time t_anchor_ns[k] with the bearing
 *   b = (bearing_xy[2k], bearing_xy[2k+1], 1):  P = R(t) (R_CI b / rho + p_CI) + p(t), the point
 *   ctvio_feature_table_map publishes for an entry anchored in a frame at that time (the frame time, not a row time).
 *   cov9[n][3][3] (row-major, world frame, exactly symmetric): G Sigma_25 G', G = dP / d(knots of t's segment, rho) and
 *     Sigma_25 the joint covariance of those 24 knot dims and rho: the 24 x 24 block of the window covariance, the cross
 *     column -Sigma W' / h of the landmark's coupling row W and diagonal h, and its variance from ctvio_covariance.
 *   A landmark no factor touches has rho constant: only the pose part remains, and a point whose four knots and rho
 *   are all constant gets an exact zero matrix.  A rho that is not > 0 and finite gives a matrix of NaNs.
 *   rcond (may be NULL): as ctvio_covariance; on CTVIO_ERR_STATE "rank deficient" only rcond is written.
 *   Errors, checked before anything is launched, with nothing written: CTVIO_ERR_INVALID for a null handle, n < 0,
 *   a NULL array with n > 0, a landmark outside 0 .. n_landmarks - 1, gauge_knot_index outside -1 .. n_knots - 1;
 *   CTVIO_ERR_STATE in sharded mode or before the knots are set; CTVIO_ERR_TIME_RANGE for an anchor time
 *   ctvio_query_trajectory does not accept.  n = 0 returns CTVIO_OK and launches nothing.
 *   ctvio_transfer_stats counts 28 n bytes up and 72 n bytes down. */
int ctvio_point_covariance(ctvio_handle h, int32_t n, const int32_t* landmark, const int64_t* t_anchor_ns,
                           const double* bearing_xy, int32_t gauge_knot_index, double* cov9, double* rcond);

/* ---- spline query service (SURVEY §8f-2: Trajectory::poseNs / GetIMUState, spline/trajectory.cpp:27-55) ----
 * batch R(t), p(t), body angular velocity, world linear velocity and acceleration. Any output may be NULL. */
int ctvio_query_trajectory(ctvio_handle h, int32_t n, const int64_t* t, double* q_xyzw, double* p_xyz,
                           double* omega_body, double* vel_world, double* acc_world);

/* ---- front-end formats either side of the path (SURVEY §8f-3) ----
 * replaces FeatureManager::triangulate(Rs, Ps, ric, tic) (visual_odometry/feature_manager.cpp:230-275; the
 * identity-extrinsic overload :173-223 is the same call with ric = I, tic = 0): DLT depth of every landmark candidate
 * (used_num >= 2 && start_frame < window_size - 2) whose depth_inout entry is <= 0; observation k of landmark l is
 * obs_point_xyz[obs_offset[l] + k] seen from frame start_frame[l] + k; depth = V(2)/V(3) of the right singular vector
 * of the smallest singular value, replaced by init_depth (INIT_DEPTH, parameters.cpp:44) when < 0.1.
 * Rs: [n_frames][9] row-major body rotations, Ps: [n_frames][3]. */
int ctvio_triangulate(ctvio_handle h, int32_t n_frames, const double* Rs_rowmajor9, const double* Ps_xyz,
                      const double* ric_rowmajor9, const double* tic_xyz, int32_t n_landmarks,
                      const int32_t* start_frame, const int32_t* obs_offset, const double* obs_point_xyz,
                      int32_t window_size, double init_depth, double* depth_inout);

/* ---- device-resident sliding window (SURVEY §8f-1): the per-image problem build of TrajectoryManager moved behind
 * the boundary.  State (control points, bias nodes, inverse depths, line delay) and the prior stay in HBM from one
 * window to the next; only what is NEW crosses the boundary. ----
 * replaces TrajectoryManager::ExtendTrajectory (estimator/trajectory_manager.cpp:108-120, spline/se3_spline.h:201-207):
 * control points are appended on the device (copies of the last one) until maxTimeNs() >= t_ns. */
int ctvio_extend_knots_to(ctvio_handle h, int64_t t_ns, int32_t* n_knots_out);
/* replaces VisualOdometry::SlideWindow + the growing-spline convention: the first n_drop_knots control points and
 * n_drop_bias bias nodes leave the window (device-side shift, time origin advanced), n_new_bias nodes are appended as
 * copies of the newest one (Bgs_/Bas_[WINDOW_SIZE]); the ACTIVE prior's knot / bias block indices are re-based. */
int ctvio_slide_window(ctvio_handle h, int32_t n_drop_knots, int32_t n_drop_bias, int32_t n_new_bias);
/* replaces the MARGIN_SECOND_NEW half of VisualOdometry::SlideWindow (visual_odometry.cpp:253-278): bias node nB-2 takes
 * the value of node nB-1 (Bgs_/Bas_[WINDOW_SIZE-1] = [WINDOW_SIZE]); node nB-1 keeps its value and stands for the next
 * image.  Knots, time origin and prior are untouched; prior blocks keep their indices.  Use it after a solve without
 * marginalization (no ctvio_marginalize / ctvio_adopt_prior), when ctvio_check_keyframe decided against the image
 * before the new one.
 *   Errors: CTVIO_ERR_STATE with fewer than 2 bias nodes, or when the active prior holds a block of bias node nB-2 -
 *   nothing changes then. */
int ctvio_slide_window_second_new(ctvio_handle h);
/* replaces FeatureManager::addFeatureCheckParallax as VisualOdometry::AddImageToWindow uses it
 * (feature_manager.cpp:28-87, visual_odometry.cpp:180-183) on the resident frame table: no knots or state are needed,
 * only clouds ingested with ctvio_ingest_feature_cloud.
 *   frame_slots[0 .. n_frames-1] lists the window's slots oldest to newest, the last one the new image; fc = n_frames-1
 *   is the reference's frame_count.  An empty cloud is a valid slot.
 *   n_tracked (last_track_num): features of the new slot whose id occurs in any other listed slot.
 *   parallax_num / parallax_sum: the features of slot fc-1 whose id also occurs in slot fc-2 (tracks are contiguous in
 *   window positions, so this is start_frame <= fc-2 && endFrame() >= fc-1), and the sum of their parallaxes
 *   sqrt(du^2 + dv^2) between the two bearings (compensatedParallax2, :424-456; with z == 1 the compensated and the plain
 *   term coincide).  Both are 0 when fc < 2; they are computed whenever fc >= 2, also when n_tracked < 20.
 *   is_keyframe = 1 when fc < 2, n_tracked < 20 or parallax_num == 0, else parallax_sum / parallax_num >= min_parallax
 *   (MIN_PARALLAX, focal-length normalised).  0 means MARGIN_SECOND_NEW.
 *   Contract: ids are unique within a cloud, as the tracker guarantees.
 *   Difference from the reference: its feature list also forgets landmarks removed by removeFailures (depth < 0); here
 *   membership is only "the id occurs in a listed slot".
 *   Outputs other than is_keyframe may be NULL.  The sum runs in a fixed order: bitwise reproducible.  One kernel launch,
 *   the slot list up, one 24-byte result back, one stream synchronisation.
 *   Errors: CTVIO_ERR_INVALID for n_frames outside 1..16, a slot outside 0..15, a slot listed twice, or a min_parallax
 *   that is negative or not finite. */
int ctvio_check_keyframe(ctvio_handle h, int32_t n_frames, const int32_t* frame_slots, double min_parallax,
                         int32_t* is_keyframe, int32_t* n_tracked, int32_t* parallax_num, double* parallax_sum);
/* replaces FeatureManager::getDepthVector / setDepth re-indexing (visual_odometry/feature_manager.cpp:139-170): landmark l
 * of the new window takes the inverse depth of old landmark old_index[l] (>= 0), else init_inv_depth[l]. */
int ctvio_remap_landmarks(ctvio_handle h, int32_t n_landmarks, const int32_t* old_index, const double* init_inv_depth);
/* replaces FeatureManager::triangulate(Rs, Ps, ric, tic) as VisualOdometry::AddImageToWindow calls it for every new image
 * (visual_odometry.cpp:185-191, feature_manager.cpp:226-274), with the camera poses taken from the RESIDENT spline and the
 * bearings / rows from the resident frame table: only index arrays go up, only the two counts come back.
 *   Landmark l is numbered as ctvio_remap_landmarks / ctvio_set_inv_depths number it; n_landmarks must equal the engine's
 *   landmark count.  Its observations are k = obs_offset[l] .. obs_offset[l+1]-1 (obs_offset[0] == 0, non-decreasing):
 *   feature obs_idx[k] of resident frame slot obs_slot[k]; the first one is the anchor.
 *   Camera pose of an observation: the spline at frame_t[slot] + row * floor(ld * 1e9) (the current line delay, truncated
 *   to int64 like the image factor), composed with the configured extrinsic: R_c = R * R(q_CtoI), t_c = p + R * p_CinI.
 *   With ld == 0 this is the reference's triangulate at the frame poses; with ld > 0 it is its rolling-shutter variant
 *   triangulateRS (feature_manager.cpp:276-338, compiled out there) with the factor's row time and the configured
 *   extrinsic.  There is no mode flag: the line delay of the state decides.
 *   Only landmarks whose resident inverse depth is <= 0 (or NaN) are written (estimated_depth > 0 -> continue, :239-240);
 *   all others stay bitwise untouched.  Fewer than 2 observations -> 1 / init_depth; otherwise the DLT depth V(2)/V(3)
 *   of the smallest right singular vector, replaced by init_depth (INIT_DEPTH, parameters.cpp:44) when below 0.1 or not
 *   finite; written as an inverse depth.
 *   n_triangulated (may be NULL): landmarks written from a DLT depth; n_fallback (may be NULL): landmarks given init_depth.
 *   Errors: CTVIO_ERR_INVALID for a landmark-count mismatch, a bad obs_offset, a slot outside 0..15, an index >= the
 *   feature count ingested in that slot or init_depth <= 0; CTVIO_ERR_STATE before the knots / line delay are set;
 *   CTVIO_ERR_TIME_RANGE when an observation's time falls outside the spline - the resident inverse depths are then
 *   unchanged.  One kernel launch (plus the knot-pair table when stale), one stream synchronisation; bitwise
 *   reproducible (no atomics on the depths). */
int ctvio_triangulate_window(ctvio_handle h, int32_t n_landmarks, const int32_t* obs_offset, const int32_t* obs_slot,
                             const int32_t* obs_idx, double init_depth, int32_t* n_triangulated, int32_t* n_fallback);
/* The reference builds a fresh TrajectoryEstimator without the prior for InitTrajectory (trajectory_manager.cpp:297);
 * here the resident prior is switched off / on instead of being cleared and re-uploaded. */
int ctvio_enable_prior(ctvio_handle h, int32_t on);
/* (ctvio_adopt_prior above hands the prior of ctvio_marginalize over device-to-device: J_lin, r_lin and the
 *  linearisation point never visit the host unless ctvio_get_prior is called.) */

/* ---- wire formats as they are (SURVEY §8f-4) ----
 * replaces FeatureMsg2Image (visual_odometry/visual_struct.h:98-121) on the tracker's sensor_msgs::PointCloud
 * (visual_feature/feature_tracker_node.cpp:146-184): points = geometry_msgs::Point32[] (packed float32 x, y, z = 1),
 * channels[0..4] = id, u, v, velocity_x, velocity_y (float32 arrays).  The arrays are uploaded unchanged and unpacked on
 * the device into frame slot `frame_slot` (0..15) of the resident feature table.  CTVIO_ERR_STATE (nothing changes) while
 * the resident feature table (ctvio_feature_table_*) holds the slot: ctvio_feature_table_slide frees it. */
int ctvio_ingest_feature_cloud(ctvio_handle h, int32_t frame_slot, int64_t t_ns, int32_t n_points, const float* points_xyz,
                               const float* ch_id, const float* ch_u, const float* ch_v, const float* ch_vx,
                               const float* ch_vy);
/* replaces the AddImageFeatureDelayAnalytic loop of UpdateTrajectory (trajectory_manager.cpp:353-385) for factors whose
 * two observations are features idx_i / idx_j of resident frame slots slot_i / slot_j (anchor / observation): only the
 * indices cross the boundary, times / bearings / rows are gathered on the device. */
int ctvio_add_image_features_from_slots(ctvio_handle h, int32_t n, const int32_t* slot_i, const int32_t* idx_i,
                                        const int32_t* slot_j, const int32_t* idx_j, const int32_t* landmark,
                                        const int32_t* marg);
/* replaces TrajectoryManager::AddIMUData + RemoveIMUData (trajectory_manager.cpp:472-475): n packed IMUData records
 * (utils/parameter_struct.h:58-65: int64 timestamp @0, Vector3d gyro @off_gyro, Vector3d accel @off_accel, record size
 * stride_bytes) are appended to the resident IMU table as they are; samples older than drop_before_ns are retired. */
int ctvio_ingest_imu(ctvio_handle h, int32_t n, const void* imu_data, int32_t stride_bytes, int32_t off_gyro,
                     int32_t off_accel, int64_t drop_before_ns);
/* replaces the AddIMUMeasurementAnalytic loops (trajectory_manager.cpp:388-417 with kf_times / fixed_node < 0: bias node
 * from the keyframe interval; :301-310 InitTrajectory with fixed_node >= 0) over the resident samples in [t_min, t_max);
 * samples before marg_before_ns are flagged for marginalization (:239-253). */
int ctvio_add_imu_from_table(ctvio_handle h, int64_t t_min_ns, int64_t t_max_ns, int32_t n_kf, const int64_t* kf_times,
                             int32_t fixed_node, int64_t marg_before_ns, int32_t* n_added);
/* ---- resident feature table: FeatureManager's feature list on the device ----
 * One table per engine, empty at ctvio_create.  An entry is one landmark (FeaturePerId, feature_manager.h): the tracker's
 * feature id, its anchor frame slot, its observations (the feature index in each frame slot that holds one, the
 * anchor's own included), its number in the last window (or -1) and its inverse depth (estimated_depth; -1 = not
 * initialised, as the FeaturePerId constructor sets it).  Entries stay in creation order.  Frame slots are those of
 * ctvio_ingest_feature_cloud; the caller passes only slots, the association by id happens on the device.  The table's
 * indices point into the slots' clouds, so ctvio_ingest_feature_cloud refuses a slot the table holds until it is slid.
 * Two slides: ctvio_feature_table_slide drops a landmark with its anchor frame, a deliberate deviation from the
 * reference (its remaining observations leave with it, and when its id comes back in a later cloud it starts a new entry
 * anchored there).  ctvio_feature_table_slide_reanchor follows the reference instead: such a landmark is re-anchored in
 * the next frame (removeBackShiftDepth, with its depth shifted into that frame) or in the newest one (removeFront,
 * feature_manager.cpp:341-423).  A caller picks one of the two for its whole run.
 *
 * ctvio_feature_table_add - the insertion half of addFeatureCheckParallax (feature_manager.cpp:28-59) for the cloud last
 *   ingested into frame_slot: a feature whose id matches a live entry becomes that entry's observation in the slot (the
 *   count is n_tracked, the reference's last_track_num over the live list); every other feature starts a new entry
 *   anchored in the slot (n_new), appended in ascending id order (the std::map order of FeatureMsg2Image), not in cloud
 *   order.  ctvio_check_keyframe is unchanged: its tracked count means "the id occurs in a listed slot", so it also
 *   counts ids whose landmark has left the table (removeFailures, or an anchor frame that left), which this count does not.
 *   Errors: CTVIO_ERR_INVALID for a slot outside 0..15 or a slot with no ingested cloud (none yet, or none since the table
 *   slid it); CTVIO_ERR_STATE when the table still holds the slot.  One launch, one 8-byte read-back. */
int ctvio_feature_table_add(ctvio_handle h, int32_t frame_slot, int32_t* n_tracked, int32_t* n_new);
/* ctvio_feature_table_window - getDepthVector / setDepth / isLandmarkCandidate (feature_manager.cpp:111-147,
 *   feature_manager.h:58-65) for the window frame_slots[0 .. n_frames-1], oldest to newest.  First every entry numbered in
 *   the previous window takes back its resident inverse depth (setDepth).  Then the candidates - used_num >= 2 &&
 *   start_frame < window_size - 2, where start_frame is the anchor slot's position in the list and used_num is 1 + its
 *   observations in the other listed slots - are numbered 0 .. n_landmarks-1 in table order, and the resident inverse
 *   depths are re-laid out on the device to that numbering, each from its entry (a new landmark: -1).  This replaces the
 *   host's old-index table + ctvio_remap_landmarks.  The call also builds the observation CSR of
 *   ctvio_triangulate_window_from_table and the factor list of ctvio_add_image_features_from_table on the device.
 *   Errors: CTVIO_ERR_INVALID for n_frames outside 1..16, a slot outside 0..15, a repeated slot or window_size < 3;
 *   CTVIO_ERR_STATE when the listed slots are not exactly the slots the table holds, or when the resident inverse-depth
 *   count no longer equals the previous window's landmark count (ctvio_set_inv_depths / ctvio_remap_landmarks changed it).
 *   One launch, one 8-byte read-back. */
int ctvio_feature_table_window(ctvio_handle h, int32_t n_frames, const int32_t* frame_slots, int32_t window_size,
                               int32_t* n_landmarks);
/* ctvio_triangulate_window_from_table - ctvio_triangulate_window (FeatureManager::triangulate / triangulateRS,
 *   feature_manager.cpp:226-338) over the last window's landmarks, with the CSR ctvio_feature_table_window built on the
 *   device (anchor first, then the observations in window order): same kernel, same rules (only inverse depths <= 0 are
 *   written, same init_depth fallback, CTVIO_ERR_TIME_RANGE leaves the depths unchanged).  Nothing goes up.
 *   Errors: CTVIO_ERR_INVALID for init_depth <= 0; CTVIO_ERR_STATE before the knots / line delay are set, without a
 *   window since the last add / slide, or when the resident inverse-depth count differs from the window's landmark count. */
int ctvio_triangulate_window_from_table(ctvio_handle h, double init_depth, int32_t* n_triangulated, int32_t* n_fallback);
/* ctvio_add_image_features_from_table - the image-factor loops of UpdateTrajectory / UpdateVIOPrior
 *   (trajectory_manager.cpp:206-236, :359-385) over the last window's landmarks: one factor per (landmark, observation
 *   other than the anchor), landmark-major, in window order within a landmark.  With marg_oldest != 0 a factor is flagged
 *   for marginalization when its anchor is the window's oldest slot and the landmark's resident inverse depth is > 0 at
 *   the time of the call.  The 16-byte descriptors are appended to the factor set's device-side list and nothing is
 *   read back: the next solve builds the structure (frame-pair groups, work lists, landmark layout, active mask) on the
 *   device, bit for bit what the host builds for the same factors added through ctvio_add_image_features_from_slots,
 *   and reads back only its count block (see ctvio_debug_structure).  Slot-named factors may be added before or after
 *   in the same factor set; they join the device-side list in caller order.  Several calls between two
 *   ctvio_clear_factors append.  Errors found by that build are those of the host build: CTVIO_ERR_TIME_RANGE when a
 *   frame time's padded knot window leaves the spline, CTVIO_ERR_INVALID for a landmark out of range.
 *   Errors: CTVIO_ERR_STATE without a window since the last add / slide, when the resident inverse-depth count differs
 *   from the window's landmark count, or when image factors with host payload are present. */
int ctvio_add_image_features_from_table(ctvio_handle h, int32_t marg_oldest, int32_t* n_factors);
/* ctvio_feature_table_slide - the feature-list half of SlideWindowOld / SlideWindowNew for the leaving frame_slot.  First
 *   removeFailures (feature_manager.cpp:148-158): an entry numbered in the last window whose resident inverse depth is
 *   < 0 leaves (SolveFail; 0 and NaN stay).  Then the entries anchored in frame_slot leave (see the deviation above) and
 *   every other entry loses its observation there.  The slot is then free for the next ctvio_ingest_feature_cloud.
 *   Errors: CTVIO_ERR_INVALID for a slot outside 0..15; CTVIO_ERR_STATE when the table does not hold the slot or when
 *   the resident inverse-depth count differs from the last window's landmark count.  One launch, one 4-byte read-back. */
int ctvio_feature_table_slide(ctvio_handle h, int32_t frame_slot, int32_t* n_removed);
/* ctvio_feature_table_slide_reanchor - the whole feature-list half of SlideWindowOld / SlideWindowNew
 *   (visual_odometry.cpp:293-308) for the window frame_slots[0 .. n_frames-1] BEFORE the slide, oldest to newest; the
 *   leaving slot is frame_slots[0] when marg_old != 0 (MARGIN_OLD), else frame_slots[n_frames-2] (MARGIN_SECOND_NEW).
 *   First removeFailures, as ctvio_feature_table_slide.  Then, for an entry anchored in the leaving slot:
 *   - marg_old != 0 (removeBackShiftDepth(Rs_[0], Ps_[0], Rs_[1], Ps_[1]), feature_manager.cpp:341-378): the anchor
 *     observation is dropped; with fewer than 2 observations left in the listed slots the entry leaves, else its anchor
 *     becomes the earliest listed slot holding an observation (frame_slots[1] for the tracker's contiguous tracks) and
 *     its depth is shifted: depth = 1 / rho (rho: the resident inverse depth of its number in the last window, else its
 *     stored one: setDepth's value), p_w = R_c0 (x, y, 1) depth + t_c0 with (x, y) the old anchor's bearing,
 *     p_1 = R_c1^T (p_w - t_c1); the stored inverse depth becomes 1 / p_1.z when p_1.z > 0, else 1 / init_depth (a NaN
 *     falls back as well).  (R_c, t_c): the camera poses at frame_slots[0]'s and frame_slots[1]'s frame times
 *     (GetCameraPose(timestamps_[i]), the resident spline composed with the configured extrinsic), so call this after the
 *     solve and ctvio_gauge_realign and BEFORE ctvio_slide_window drops the leaving frame's knots.
 *   - marg_old == 0 (removeFront, :398-423): with an observation in the newest slot its anchor moves there and its
 *     inverse depth (as above) is kept as the stored one; without one the entry leaves.  No pose is needed.
 *   A re-anchored entry keeps its place in the table and its id, and loses its number, so the next
 *   ctvio_feature_table_window takes its stored inverse depth.  It keeps solve_flag == SovelSucc when it was numbered,
 *   which ctvio_feature_table_map's margin cloud reads.  Every other entry loses its observation in the leaving slot,
 *   and the slot is free for the next ctvio_ingest_feature_cloud.  *n_removed: the entries that left (failures
 *   included); *n_reanchored: the entries whose anchor moved (either may be NULL).
 *   Errors (nothing changes in the table or the state): CTVIO_ERR_INVALID for n_frames outside 2..16, a slot outside
 *   0..15, a repeated slot or an init_depth that is not a finite value > 0; CTVIO_ERR_STATE when the listed slots are
 *   not exactly the slots the table holds, when the resident inverse-depth count differs from the last window's landmark
 *   count, or (marg_old != 0) before the knots are set; CTVIO_ERR_TIME_RANGE (marg_old != 0) when frame_slots[0]'s or
 *   frame_slots[1]'s frame time falls outside the spline.
 *   One launch (plus the knot-pair table when it is stale, MARGIN_OLD), one 8-byte read-back; no atomics, bitwise
 *   reproducible. */
int ctvio_feature_table_slide_reanchor(ctvio_handle h, int32_t n_frames, const int32_t* frame_slots, int32_t marg_old,
                                       double init_depth, int32_t* n_removed, int32_t* n_reanchored);
/* ctvio_feature_table_landmarks - feature id, anchor slot and used_num of each landmark of the last window, in its
 *   numbering (GetLandmarksInWindow needs the id).  Errors: CTVIO_ERR_INVALID for a landmark-count mismatch or a NULL
 *   array; CTVIO_ERR_STATE without a window since the last add / slide. */
int ctvio_feature_table_landmarks(ctvio_handle h, int32_t n_landmarks, int32_t* feature_id, int32_t* anchor_slot,
                                  int32_t* used_num);
/* ctvio_feature_table_map - the landmark map and keyframe poses the reference publishes after every image, right after
 *   SlideWindow (odometry_manager.cpp:281-288): GetLandmarksInWindow, GetMarginCloud (visual_odometry.cpp:310-372) and
 *   PublishVioKeyFrame(Ps_).  Call it after either slide with frame_slots[0 .. n_frames-1], the post-slide
 *   window oldest to newest (MARGIN_OLD dropped position 0, MARGIN_SECOND_NEW the second-newest); it is valid whenever the
 *   listed slots are exactly the slots the table holds.  It only reads: neither the table nor the state changes.
 *   Per entry, in table order (the reference's std::list order): start = position of its anchor slot in the list,
 *   used_num = 1 + its observations in the other listed slots, depth = 1 / rho, where rho is the resident inverse depth
 *   of its number in the last window when it has one (what the next setDepth gives it), else its stored inverse depth
 *   (-1 for an entry never initialised).
 *   Stable (IsLandMarkStable, visual_odometry.h:82-93, as written there): used_num >= 2 && start < window_size - 2 &&
 *   !(start > window_size * 3.0 / 4.0) && !(depth <= 0), so a NaN depth passes, as in the reference.
 *   Margin cloud (GetMarginCloud): stable, start == 0, used_num <= 2 and solve_flag == SovelSucc.  setDepth gives
 *   SovelSucc to a numbered entry whose depth is not < 0 (removeFailures has already removed the others), so this is
 *   "numbered in the last window, or re-anchored by ctvio_feature_table_slide_reanchor after being numbered" (the one
 *   status the table carries across a slide); stable's depth test already makes it SovelSucc (a NaN depth included).
 *   After ctvio_feature_table_slide, an entry with start == 0 was a candidate in the last window under both slide rules
 *   (window_size >= 4): its anchor sat at position 1 (MARGIN_OLD) or 0 (MARGIN_SECOND_NEW), below window_size - 2, and a
 *   slide only takes observations away, so its used_num was at least 2 then as well.  After the re-anchoring slide the
 *   margin cloud holds the re-anchored landmarks that are down to two observations.
 *   World point (Rs_[start] * (point * estimated_depth) + Ps_[start]): p_w = R_c ((x, y, 1) depth) + t_c, (x, y) the anchor
 *   observation's bearing in the frame table, (R_c, t_c) the camera pose at the anchor slot's frame time
 *   (GetCameraPose(timestamps_[i]), :197-202, not the row time): the resident spline composed with the configured
 *   extrinsic, R_c = R R_CI, t_c = p + R p_CI.
 *   Outputs: the stable points, compacted in table order: xyz_world[k][3], feature_id[k], in_margin_cloud[k] (0 / 1).
 *   *n_points receives their count whenever the map was computed (on success, and with a capacity below it, in which case
 *   the call returns CTVIO_ERR_INVALID and writes no point).  cam_q_xyzw[n_frames][4] and cam_p_xyz[n_frames][3] (either
 *   may be NULL) receive the listed frames' camera poses at the frame time: the reference's Rs_ / Ps_.
 *   After ctvio_feature_table_slide (the table's deviation, see above) the entries anchored in the leaving frame have
 *   left with it, so they are not in the map; after ctvio_feature_table_slide_reanchor they are, as in the reference.
 *   Errors (nothing is written to the caller's arrays): CTVIO_ERR_INVALID for n_frames outside 1..16, a slot outside
 *   0..15, a repeated slot, window_size < 3, a negative or too small capacity, or NULL point arrays with capacity > 0;
 *   CTVIO_ERR_STATE before the knots are set, when the listed slots are not exactly the slots the table holds, or when the
 *   resident inverse-depth count differs from the last window's landmark count; CTVIO_ERR_TIME_RANGE when a listed frame
 *   time falls outside the spline.
 *   One launch (plus the knot-pair table when it is stale), nothing goes up (the slots travel as launch parameters), one
 *   stream synchronise: the kernel writes the points, the poses and the count straight into mapped host memory.
 *   ctvio_transfer_stats counts d2h = 8 + 56 n_frames + 32 n_points bytes (count, 7 doubles per pose, 32-byte records). */
int ctvio_feature_table_map(ctvio_handle h, int32_t n_frames, const int32_t* frame_slots, int32_t window_size,
                            int32_t capacity, double* xyz_world, int32_t* feature_id, uint8_t* in_margin_cloud,
                            int32_t* n_points, double* cam_q_xyzw, double* cam_p_xyz);
/* ctvio_feature_table_point_covariance - ctvio_point_covariance for every landmark of the feature table's last window,
 *   in the numbering of ctvio_feature_table_window / ctvio_feature_table_landmarks: cov9[n_landmarks][3][3].  Landmark
 *   l's anchor is the first entry of its observation CSR (anchor slot, feature index): the bearing is that feature's in
 *   the frame table, the time the anchor slot's frame time.  rcond as ctvio_point_covariance.
 *   When it applies to a map point: call it after the solve and ctvio_gauge_realign and before the slide (after the
 *   slide H no longer matches the state).  A map entry that keeps its anchor and its number across the slide is the
 *   same function of the same state in ctvio_feature_table_map: for it, the matrix of its number is the covariance of
 *   the point the map publishes.  An entry re-anchored by ctvio_feature_table_slide_reanchor loses its number, and its
 *   new point has no covariance from this call.
 *   Errors, checked before anything is launched, with nothing written: CTVIO_ERR_INVALID for a null handle,
 *   gauge_knot_index outside -1 .. n_knots - 1, n_landmarks other than the window's landmark count, or a NULL cov9
 *   with n_landmarks > 0; CTVIO_ERR_STATE in sharded mode, without a window since the last add / slide, when the
 *   resident inverse-depth count differs from the window's landmark count, or before the knots are set;
 *   CTVIO_ERR_TIME_RANGE when the frame time of a slot the table holds falls outside the spline.  n_landmarks = 0
 *   returns CTVIO_OK and launches nothing.
 *   Nothing goes up; ctvio_transfer_stats counts 72 n_landmarks bytes down. */
int ctvio_feature_table_point_covariance(ctvio_handle h, int32_t n_landmarks, int32_t gauge_knot_index, double* cov9,
                                         double* rcond);

/* bytes moved host<->device by the C-ABI calls since the last reset (state, factors, priors, index tables) */
int ctvio_transfer_stats(ctvio_handle h, int64_t* h2d_bytes, int64_t* d2h_bytes, int32_t reset);
/* host waits on the device (stream synchronisations, and spins on the scalars an LM step publishes to mapped memory) by
 * the C-ABI calls made on the calling thread since the last reset: a debug counter for measuring how often the host
 * stops for the device. */
int ctvio_sync_stats(ctvio_handle h, int64_t* host_waits, int32_t reset);

/* ---- the per-image odometry cycle: OdometryManager::ProcessVIOData (odometry_manager.cpp:178-299) behind two calls ----
 * The resident window (SURVEY §8f-1) driven as the reference drives it after every image, with every stage of the
 * section above in the reference's order and the bookkeeping a caller of those calls keeps itself (frame slots, the
 * window's frames and frame times, the knot range of each frame, bias nodes) held by the library.  The caller passes
 * only messages: the tracker's PointClouds and the IMUData records.  The cycle can also publish the uncertainty of what
 * it publishes (ctvio_cycle_covariances).  Not covered: the host-association and rho0 modes of the separate calls,
 * sharded engines and the initialisers.
 * Every image takes a frame slot: frame f (counting the frames since ctvio_odometry_start, the first one 0) takes slot
 * f % 16 when the feature table does not hold it, else the lowest free slot. */

/* One tracker message: sensor_msgs::PointCloud as ctvio_ingest_feature_cloud takes it. */
typedef struct ctvio_image_msg {
  int64_t t_ns;          /* image time                                                   */
  int32_t n_points;
  int32_t reserved;
  const float* points_xyz;  /* geometry_msgs::Point32[] (x, y, z = 1)                     */
  const float* ch_id;       /* channels[0..4]: id, u, v, velocity_x, velocity_y           */
  const float* ch_u;
  const float* ch_v;
  const float* ch_vx;
  const float* ch_vy;
} ctvio_image_msg;

/* IMUData records as ctvio_ingest_imu takes them: int64 timestamp at offset 0, Vector3d gyro at off_gyro, Vector3d
 * accel at off_accel, record size stride_bytes. */
typedef struct ctvio_imu_msgs {
  int32_t n;
  int32_t stride_bytes;
  int32_t off_gyro;
  int32_t off_accel;
  const void* data;
} ctvio_imu_msgs;

/* Options of the cycle, fixed by ctvio_odometry_start for the whole run.  ctvio_cycle_default_options fills the values
 * in brackets. */
typedef struct ctvio_cycle_options {
  int32_t window_size;          /* WINDOW_SIZE (parameters.h:8): the window holds window_size + 1 frames, 2..15 [10] */
  int32_t solve_iterations;     /* UpdateTrajectory's Solve (odometry_manager.cpp:264)                        [15]  */
  int32_t predictor_iterations; /* InitTrajectory's Solve (trajectory_manager.cpp:288-315)                    [8]   */
  int32_t fix_ld;               /* line delay constant in the main solve                                      [0]   */
  double min_parallax;          /* MIN_PARALLAX, focal-length normalised; <= 0: every image is a keyframe       [0]   */
  double init_depth;            /* INIT_DEPTH (parameters.cpp:44): triangulation fallback and depth shift      [5]   */
  int64_t extend_ns;            /* the spline is extended to image time + extend_ns (odometry_manager.cpp:246) [40 ms] */
  double ld_lower, ld_upper;    /* line-delay bounds of the main solve                                   [0, 35e-6] */
  double sigma_wb_discrete;     /* bias random walk (trajectory_manager.cpp:420-450)                          [2e-5] */
  double sigma_ab_discrete;     /*                                                                            [4e-4] */
  int32_t reanchor;             /* the feature list slides as the reference's does (ctvio_feature_table_slide_reanchor)
                                   instead of dropping a landmark with its anchor frame (ctvio_feature_table_slide) [0] */
  int32_t publish_map;          /* ctvio_feature_table_map of the post-slide window after every image         [1]   */
  /* the covariance publications (ctvio_cycle_covariances), each 0 or 1: */
  int32_t publish_pose_covariance;     /* the camera pose and velocity at the TF time, 12 x 12                  [0]   */
  int32_t publish_odometry_covariance; /* the relative camera pose of each consecutive frame pair, 6 x 6         [0]   */
  int32_t publish_map_covariance;      /* each map point's world point, 3 x 3; requires publish_map             [0]   */
  int32_t covariance_gauge_knot;       /* -1..3: knots <= it are held constant for the covariances only (the
                                          gauge_knot_index of the separate calls)                               [3]   */
} ctvio_cycle_options;

/* Optional outputs; a NULL pointer means the output is not wanted. */
typedef struct ctvio_cycle_outputs {
  /* the window's knots and line delay after ctvio_gauge_realign, before the slide (what the reference publishes) */
  int32_t knot_capacity;   /* rows of q_xyzw / p_xyz; CTVIO_ERR_INVALID (after the cycle ran) when below the knot count */
  int32_t map_capacity;    /* rows of the map point arrays, as ctvio_feature_table_map's capacity                    */
  double* q_xyzw;          /* [knot_capacity][4]                                                                     */
  double* p_xyz;           /* [knot_capacity][3]                                                                     */
  double* line_delay;      /* [1]                                                                                    */
  /* ctvio_feature_table_map of the post-slide window (publish_map only) */
  double* map_xyz;         /* [map_capacity][3]                                                                      */
  int32_t* map_feature_id; /* [map_capacity]                                                                         */
  uint8_t* map_in_margin_cloud;
  double* cam_q_xyzw;      /* [16][4]: the post-slide window's camera poses, oldest to newest                       */
  double* cam_p_xyz;       /* [16][3]                                                                                */
} ctvio_cycle_outputs;

/* What one cycle did. */
typedef struct ctvio_cycle_result {
  int32_t marg_flag;        /* 0 MARGIN_OLD, 1 MARGIN_SECOND_NEW                                                    */
  int32_t n_tracked;        /* ctvio_check_keyframe's counts; -1 / 0 when no check ran                              */
  int32_t parallax_num;
  int32_t frame_slot;       /* the slot the image took (ctvio_odometry_start: the newest frame's)                   */
  double parallax_sum;
  int32_t n_frames;         /* frames of the window that was solved                                                 */
  int32_t n_knots;          /* its knots; knot 0 sits at knot_t0_ns                                                 */
  int64_t knot_t0_ns;
  int32_t n_landmarks, n_image_factors, n_imu_factors, n_predictor_imu, n_triangulated, n_fallback;
  ctvio_summary predictor;  /* all zero when the predictor did not run (window 0, or no IMU sample in its range)    */
  ctvio_summary solve;
  int32_t prior_dim;        /* dimension of the active prior after the cycle                                        */
  int32_t n_removed;        /* entries that left the feature table                                                  */
  int32_t n_reanchored;     /* reanchor only, else 0                                                                */
  int32_t n_map_points;     /* publish_map only, else 0                                                             */
  int32_t n_margin_points;
  int32_t n_knots_after;    /* knots of the engine's window after the slide                                         */
  double host_ms;           /* the call's own host wall clock                                                       */
} ctvio_cycle_result;

/* the defaults in brackets above */
int ctvio_cycle_default_options(ctvio_cycle_options* opt);
/* What ctvio_cycle_covariances returns besides the matrices. */
typedef struct ctvio_cycle_covariance_info {
  int32_t requested;        /* the last cycle's publications (bits): 1 pose, 2 odometry edges, 4 map points     */
  int32_t available;        /* the same bits for what it published; 0 when ctvio_cycle_covariances fails        */
  int32_t status;           /* CTVIO_OK when available; CTVIO_ERR_STATE: rank deficient, nothing requested or no
                               completed cycle; CTVIO_ERR_TIME_RANGE: a time outside the spline or the evaluation */
  int32_t gauge_knot;       /* covariance_gauge_knot of the run                                                  */
  double rcond;             /* of the window covariance, as ctvio_covariance reports it; NaN when not formed     */
  int64_t pose_t_ns;        /* the TF time of cov12                                                              */
  int32_t n_pairs;          /* rows of cov6 / pair_t_ns (0 unless the odometry edges are available)              */
  int32_t n_map_points;     /* rows of map_cov9: the cycle's map points (0 unless the map's are available)      */
  int32_t n_map_points_without_cov; /* of those, the rows of NaN                                                  */
  int32_t reserved;
} ctvio_cycle_covariance_info;

/* ctvio_odometry_start - SetInitialState + InitWindow + the first UpdateTrajectory (odometry_manager.cpp:230-264), which
 *   runs no predictor (first_opt_flag): the initializer's window of n_frames = window_size + 1 images goes up once.
 *   Knots q_xyzw / p_xyz [n_knots] start at t0_ns (knot 0, on the configured knot grid), bg_ba6 [n_frames] holds one
 *   bias node per frame, line_delay the initial line delay; imu: every IMUData record up to the newest image (may be
 *   NULL when there is none).  The engine's earlier run, if any, is forgotten: feature table, frame slots, IMU table and
 *   prior start empty.  Then the window is solved as ctvio_process_image solves it, without the predictor.
 *   marg_flag_override: -1 lets the keyframe decision choose, 0 / 1 force MARGIN_OLD / MARGIN_SECOND_NEW.
 *   Errors: see ctvio_process_image; CTVIO_ERR_INVALID also for n_frames != window_size + 1, n_knots < 4 or a NULL
 *   array, all checked before anything changes. */
int ctvio_odometry_start(ctvio_handle h, const ctvio_cycle_options* opt, int64_t t0_ns, int32_t n_knots, const double* q_xyzw,
                         const double* p_xyz, int32_t n_frames, const ctvio_image_msg* frames, const double* bg_ba6,
                         double line_delay, const ctvio_imu_msgs* imu, int32_t marg_flag_override, ctvio_cycle_outputs* out,
                         ctvio_cycle_result* result);
/* ctvio_process_image - one image of OdometryManager::ProcessVIOData (odometry_manager.cpp:178-299) on the resident
 *   window.  imu: the IMUData records since the last call (may be NULL).  In order:
 *    1. the cloud goes into the image's frame slot and joins the feature table (ctvio_ingest_feature_cloud,
 *       ctvio_feature_table_add; AddImageToWindow, visual_odometry.cpp:180-183);
 *    2. the keyframe decision: ctvio_check_keyframe over the window's slots when min_parallax > 0, else MARGIN_OLD,
 *       unless marg_flag_override says otherwise;
 *    3. ExtendTrajectory to the image time + extend_ns (trajectory_manager.cpp:108-120), then the IMU records go in,
 *       samples before the window's first knot retired (AddIMUData / RemoveIMUData, :472-475);
 *    4. ctvio_feature_table_window (setDepth + getDepthVector);
 *    5. InitTrajectory (:288-315): IMU factors over [end of the spline before the extension, end after it) with the
 *       newest bias node, prior off, knots up to the last one before the extension fixed, biases locked, line delay
 *       fixed, predictor_iterations LM steps (skipped without a sample in that range);
 *    6. ctvio_triangulate_window_from_table (FeatureManager::triangulate, visual_odometry.cpp:185-191);
 *    7. UpdateTrajectory's factors (:317-453): the prior, the table's image factors, IMU factors over [first knot,
 *       min(end of spline, image time + 1 ns)) with bias nodes from the keyframe intervals, and the bias random-walk
 *       factors between consecutive frames; MARGIN_OLD flags for marginalization the oldest frame's image factors, the
 *       IMU samples before the second frame and the first bias factor (:206-263);
 *    8. Solve(solve_iterations);
 *    9. double2vector (:485-516): ctvio_gauge_realign to knot 0 as it was before the solve;
 *   10. MARGIN_OLD: UpdateVIOPrior (:122-286): ctvio_marginalize, and the new prior becomes the active one
 *       (ctvio_get_prior still returns it afterwards, until the next marginalization);
 *   11. reanchor: ctvio_feature_table_slide_reanchor;
 *   12. SlideWindow: ctvio_slide_window(knots of the oldest frame, 1, 1) or ctvio_slide_window_second_new;
 *   13. without reanchor: ctvio_feature_table_slide of the leaving frame's slot;
 *   14. publish_map: ctvio_feature_table_map of the post-slide window.
 *   With a publish_*_covariance flag set, the covariances of ctvio_cycle_covariances are formed right after step 9.
 *   Computed on the device from what it already holds, where a caller of the separate calls computes them on the host:
 *   - the bias random-walk weights (trajectory_manager.cpp:420-450): for frames i, i+1, with s2 the sum of dt^2 over the
 *     IMU intervals that start at or after frame i's time and end before frame i+1's, sqrt_info = 1 / sqrt(s2 sigma^2)
 *     per axis (0 when s2 == 0).  s2 is the difference of two entries of a sequential prefix sum of dt^2 that runs over
 *     every sample ingested since ctvio_odometry_start, in sample order, with dt = (t_k - t_{k-1}) * 1e-9;
 *   - the pre-solve pose of knot 0 for the re-alignment, a device-to-device snapshot taken before the main solve
 *     (trajectory_manager.cpp:325-327).
 *   The host still reads back what it decides on or sizes launches with: the keyframe flag, the feature table's counts,
 *   the LM step scalars, the marginalization's block bookkeeping.
 *   Errors (through ctvio_last_error): CTVIO_ERR_INVALID for a NULL handle, options (start) or result, options out of
 *   range (window_size outside 2..15, iterations < 1 or predictor_iterations < 0, init_depth not finite and > 0,
 *   extend_ns <= 0, a min_parallax that is not finite, a publish_*_covariance flag other than 0 / 1,
 *   covariance_gauge_knot outside -1..3, publish_map_covariance without publish_map), a bad message (NULL arrays, n_points outside 0..1024) or IMU
 *   layout (as ctvio_ingest_imu), marg_flag_override outside -1..1; CTVIO_ERR_STATE before ctvio_odometry_start, on a
 *   sharded engine (world > 1), or when the feature table holds all 16 frame slots so the image has none.  These are
 *   checked before any device work and leave the engine unchanged.  An error of a stage (CTVIO_ERR_TIME_RANGE, ...)
 *   stops the cycle there; the engine must then be restarted with ctvio_odometry_start. */
int ctvio_process_image(ctvio_handle h, const ctvio_image_msg* img, const ctvio_imu_msgs* imu, int32_t marg_flag_override,
                        ctvio_cycle_outputs* out, ctvio_cycle_result* result);
/* ctvio_cycle_covariances - the covariances the last ctvio_odometry_start / ctvio_process_image published, with the
 *   options' publish_*_covariance flags.  The cycle forms them right after step 9, on the solved window's H, before
 *   the marginalization and the slide change it: the window covariance Sigma once (as ctvio_covariance forms it, with
 *   the knots <= covariance_gauge_knot held constant), then its projections on the device, all in the camera frame:
 *   - cov12 [12][12]: ctvio_pose_covariance at pose_t_ns = the solved window's maxTimeNs() - 50 ms, the time of the
 *     reference's TF (odometry_manager.cpp:287-288);
 *   - cov6 [n_pairs][6][6]: ctvio_relative_pose_covariance of the solved window's consecutive frames, pair_t_ns
 *     [n_pairs][2] their times (the odometry edges a pose graph fuses);
 *   - map_cov9 [n_map_points][3][3]: the covariance of each point of that cycle's map output, in its order: the
 *     point's matrix from ctvio_feature_table_point_covariance by the entry's number in the solved window, attached by
 *     the map kernel.  A point without a number there, or re-anchored by the slide (reanchor), gets NaNs.
 *   Sigma never leaves the device, and the cycle waits for nothing more: the rank test (as ctvio_covariance's) reads
 *   its inputs after the synchronisation the slide makes anyway.  A rank-deficient window does not stop the cycle:
 *   info->status is CTVIO_ERR_STATE with info->rcond, and nothing is available.
 *   Every pointer but the handle may be NULL.  The call copies from host memory the cycle filled: no device work, no
 *   synchronisation.  Each cycle clears what the last one published before it starts.
 *   Errors (info, when given, is filled first): CTVIO_ERR_INVALID for a NULL handle, a negative map_capacity, or a
 *   map_capacity below n_map_points with map_cov9; CTVIO_ERR_STATE "not available" before any cycle, after a cycle
 *   that stopped on an error or published nothing (flags off, rank deficient, ...).
 *   ctvio_transfer_stats counts, in the cycle: 8 bytes up for the TF time and 8 n_frames for the frame times, 1152
 *   bytes down for cov12, 288 n_pairs for cov6 and 72 n_map_points for map_cov9. */
int ctvio_cycle_covariances(ctvio_handle h, double* cov12, int64_t* pose_t_ns, double* cov6, int64_t* pair_t_ns,
                            int32_t map_capacity, double* map_cov9, ctvio_cycle_covariance_info* info);
/* ctvio_odometry_checkpoint - the run of the odometry cycle as one self-describing blob, from which
 *   ctvio_odometry_restore continues it on this or another engine: a later ctvio_process_image computes, bit for bit,
 *   what it computes on the engine that took the checkpoint.  Valid after any ctvio_odometry_start /
 *   ctvio_process_image that returned CTVIO_OK.
 *   The blob holds what the next cycle reads: the knots, bias nodes, inverse depths and line delay with their counts,
 *   the time origin as the slides moved it, the active prior (J, r, x0, block lists, whether it is enabled), the clouds
 *   of the frame slots the feature table holds (up to each point count) with their times, the live rows of the
 *   resident IMU table with their dt^2 prefix values and the prefix carry, the feature table's live entries (id, anchor,
 *   number, per-slot feature indices, masks, inverse depths, sorted keys) and counts, and the cycle's options, window
 *   frames and frame counter.  Not held: what the next call rebuilds (factor structures, knot-pair table, scales,
 *   workspaces), the last cycle's covariance publications, and the engine's deterministic mode.
 *   Format: little-endian; a magic number, the format version (1), CTVIO_ABI_VERSION, the length, a 64-bit checksum
 *   of everything after the header, a section table, then the counts and the configuration (ctvio_config without
 *   device), the prior's block lists and the device sections.  The device sections are gathered by one kernel
 *   launch into a staging buffer that also sums their checksum terms, then come back in one copy.
 *   buf NULL: only *len is written (the size the checkpoint needs; no device work).  Otherwise the blob's *len bytes are
 *   written to buf.
 *   Transfers: *len bytes down, nothing up.  Synchronises the engine stream once.
 *   Errors (nothing is written but *len): CTVIO_ERR_INVALID for a NULL len, capacity < 0, a NULL handle, or (buf
 *   given) capacity below the size needed; CTVIO_ERR_STATE before ctvio_odometry_start, after a cycle that stopped on
 *   an error, on a sharded engine, or when the active prior came from ctvio_set_prior after the cycle. */
int ctvio_odometry_checkpoint(ctvio_handle h, void* buf, int64_t capacity, int64_t* len);
/* ctvio_odometry_restore - replaces the engine's run, if any, with the one of a blob of ctvio_odometry_checkpoint; the
 *   next call is ctvio_process_image.  The engine must have been created with an equal configuration (every
 *   ctvio_config field but device and t0_ns; the blob's time origin must lie on the engine's knot grid); the device
 *   ordinal may differ.  The engine keeps its deterministic mode.  Until the next cycle, ctvio_cycle_covariances
 *   reports "not available" and ctvio_get_prior "no prior has been produced".
 *   The host checks the header, counts and section table; the blob then goes up in one copy, and a kernel recomputes
 *   the checksum and checks the section table on the device, into scratch buffers.  Only a blob that passes is
 *   written into the engine's buffers (a second launch), so a refused blob leaves the engine's run bitwise unchanged.
 *   Transfers: len bytes up, the device check's 4-byte verdict down.  Synchronises the engine stream once.
 *   Errors: CTVIO_ERR_INVALID for len < 0, a NULL buf with len > 0, a NULL handle, a malformed blob (bad magic number,
 *   a format version other than 1, another CTVIO_ABI_VERSION, a length other than the blob's, counts or a section
 *   table that do not agree, a checksum mismatch) or a configuration that differs from the engine's; CTVIO_ERR_STATE
 *   on a sharded engine.  All of them leave the engine unchanged. */
int ctvio_odometry_restore(ctvio_handle h, const void* buf, int64_t len);
/* test support: the bias random-walk weights ctvio_process_image computes, for the keyframe times kf_t_ns[0 .. n_kf-1]
 *   (2..16, ascending) over the resident IMU table as the last cycle left it; sqrt_info6 [n_kf - 1][6]. */
int ctvio_debug_bias_weights(ctvio_handle h, int32_t n_kf, const int64_t* kf_t_ns, double sigma_wb_discrete,
                             double sigma_ab_discrete, double* sqrt_info6);

/* ---- measurement support (bench.py roofline) ----
 * Average CUDA-event duration (ms, on the engine stream) of one launch of each stage of an LM step at the
 * current state, over `reps` launches after 3 warm-up launches.  flush_l2 != 0 writes a 256 MiB scratch
 * buffer (> the 50 MB L2) between timed launches.
 *   out_ms[0] visual residual+Jacobian+accumulate kernel (K1)   out_ms[1] IMU kernel (K2)
 *   out_ms[2] bias + prior kernels (K3)                          out_ms[3] reduced system + landmark Schur (K4)
 *   out_ms[4] blocked Cholesky + triangular solves (K5)          out_ms[5] step vectors / back-substitution (K6)
 *   out_ms[6] apply step + knot-pair table (K6/K0)               out_ms[7] cost-only visual kernel */
int ctvio_profile_kernels(ctvio_handle h, int32_t reps, int32_t flush_l2, double* out_ms8);
/* fp64 FMA micro-benchmark (8 independent DFMA chains per thread, all SMs): measured TFLOP/s, the compute
 * roofline denominator of the fp64-bound kernels (MEASURED_PEAKS.json has only HBM and bf16). */
int ctvio_measure_fp64_tflops(ctvio_handle h, double* tflops);
/* fp64 tensor-core micro-benchmark (8 independent mma.sync.m8n8k4.f64 chains per warp, all SMs): measured TFLOP/s,
 * the compute roofline denominator of the kernels built on DMMA (the dense solve K5, the Schur update K4). */
int ctvio_measure_fp64_tensor_tflops(ctvio_handle h, double* tflops);
/* Self-check of the dense solver (K5) on the reduced system of the current state: the system is built once, then
 * factored + solved `reps` times from the same input.  mismatches = number of repetitions whose solution differs
 * BITWISE from the first one (must be 0: the sharded mode relies on a reproducible replicated solve);
 * rel_residual = max_i |M x - rhs|_i / max_i |rhs|_i of the first solve, evaluated on the host. */
int ctvio_selfcheck_solver(ctvio_handle h, int32_t reps, int32_t* mismatches, double* rel_residual);

/* ---- multi-GPU: landmark-sharded residuals, one allreduce of the reduced system per LM step ----
 * Every rank holds the full (replicated) state and its own shard of image factors; rank 0 also holds
 * IMU / bias / prior factors. unique_id is the 128-byte ncclUniqueId from ctvio_nccl_unique_id on rank 0. */
int ctvio_nccl_unique_id(uint8_t* id128);
int ctvio_comm_init(ctvio_handle h, int32_t rank, int32_t world_size, const uint8_t* id128);

#ifdef __cplusplus
}
#endif
#endif /* CTVIO_H_ */
