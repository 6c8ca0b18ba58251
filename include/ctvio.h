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
/* total cost 0.5*sum rho(|r|^2) of all factors incl. bias + prior at the current state */
int ctvio_eval_cost(ctvio_handle h, double* cost);
/* Schur-form normal equations at the current state: camera block H_cc (np x np, row-major, symmetric),
 * g_c (np), per-landmark h_l, g_l (n_landmarks each).  np = 6*n_knots + 6*n_bias + 1. */
int ctvio_normal_equations(ctvio_handle h, double* Hcc, double* gc, double* hl, double* gl, double* cost);

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
/* replaces FeatureManager::getDepthVector / setDepth re-indexing (visual_odometry/feature_manager.cpp:139-170): landmark l
 * of the new window takes the inverse depth of old landmark old_index[l] (>= 0), else init_inv_depth[l]. */
int ctvio_remap_landmarks(ctvio_handle h, int32_t n_landmarks, const int32_t* old_index, const double* init_inv_depth);
/* The reference builds a fresh TrajectoryEstimator without the prior for InitTrajectory (trajectory_manager.cpp:297);
 * here the resident prior is switched off / on instead of being cleared and re-uploaded. */
int ctvio_enable_prior(ctvio_handle h, int32_t on);
/* (ctvio_adopt_prior above hands the prior of ctvio_marginalize over device-to-device: J_lin, r_lin and the
 *  linearisation point never visit the host unless ctvio_get_prior is called.) */

/* ---- wire formats as they are (SURVEY §8f-4) ----
 * replaces FeatureMsg2Image (visual_odometry/visual_struct.h:98-121) on the tracker's sensor_msgs::PointCloud
 * (visual_feature/feature_tracker_node.cpp:146-184): points = geometry_msgs::Point32[] (packed float32 x, y, z = 1),
 * channels[0..4] = id, u, v, velocity_x, velocity_y (float32 arrays).  The arrays are uploaded unchanged and unpacked on
 * the device into frame slot `frame_slot` (0..15) of the resident feature table. */
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
/* bytes moved host<->device by the C-ABI calls since the last reset (state, factors, priors, index tables) */
int ctvio_transfer_stats(ctvio_handle h, int64_t* h2d_bytes, int64_t* d2h_bytes, int32_t reset);

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
