// The per-image odometry cycle (include/ctvio.h: ctvio_odometry_start, ctvio_process_image): the stages of the resident
// window's entry points in OdometryManager::ProcessVIOData's order, with the window's frame bookkeeping held here and the
// last two host computations of a caller of those entry points (the bias random-walk weights and the pre-solve pose of
// knot 0) done on the device.
#include <atomic>
#include <chrono>
#include <cmath>

#include "engine_state.h"

namespace ctvio {
namespace {

constexpr int kMaxKf = 16;

struct KfTimes { int64_t t[kMaxKf]; };

// carry[0]: the prefix of dt^2 at the last sample ingested, carry[1]: that sample's time (int64 bits), carry[2]: != 0
// once a sample was ingested.  The prefix of table sample k is kept in the .y of its {t, .y} record, which no reader of
// the resident table uses (ingestion writes 0 there) and which the table's shift and growth move with the sample.
__device__ __forceinline__ double prefix_of(const longlong2& r) { return __longlong_as_double(r.y); }

// Extends the prefix over the samples [first, first + n) just appended, sequentially in sample order: the prefix of the
// first sample ever ingested is 0, every later one adds (dt * 1e-9)^2 to its predecessor's, dt the int64 time step.  The
// same operations as numpy's cumsum over np.diff(t) * 1e-9 squared (synthetic.bias_sqrt_info); no contraction.
__global__ void imu_prefix_kernel(longlong2* tab, int first, int n, double* carry) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  double c = carry[0];
  int64_t t_prev = __double_as_longlong(carry[1]);
  bool valid = carry[2] != 0.0;
  for (int k = first; k < first + n; ++k) {
    const int64_t t = tab[k].x;
    if (valid) {
      const double dt = __dmul_rn(double(t - t_prev), 1e-9);
      c = __dadd_rn(c, __dmul_rn(dt, dt));
    } else {
      c = 0.0;
      valid = true;
    }
    tab[k].y = __double_as_longlong(c);
    t_prev = t;
  }
  carry[0] = c;
  carry[1] = __longlong_as_double(t_prev);
  carry[2] = valid ? 1.0 : 0.0;
}

// first table index with t >= v (n if none)
__device__ __forceinline__ int lower_bound_t(const longlong2* tab, int n, int64_t v) {
  int lo = 0, hi = n;
  while (lo < hi) {
    const int m = (lo + hi) >> 1;
    if (tab[m].x < v) lo = m + 1;
    else hi = m;
  }
  return lo;
}

// The bias random-walk weights of trajectory_manager.cpp:420-450 for the keyframe pairs (kf_i, kf_i+1), one thread per
// pair, as synthetic.bias_sqrt_info computes them: a = first sample >= kf_i, b = first sample >= kf_i+1,
// s2 = prefix[b - 1] - prefix[a] when b - 1 > a (else 0), sqrt_info = 1 / sqrt(s2 sigma^2) per axis when s2 > 0 (else 0).
// sig2: sigma_wb^2, sigma_ab^2.  out: [n_kf - 1][6].
__global__ void bias_sqrt_info_kernel(const longlong2* tab, int n_tab, KfTimes kf, int n_kf, double sig2_wb, double sig2_ab,
                                      double* out) {
  const int i = threadIdx.x;
  if (i >= n_kf - 1) return;
  double s2 = 0.0;
  if (n_tab >= 2) {
    const int a = lower_bound_t(tab, n_tab, kf.t[i]);
    const int b = lower_bound_t(tab, n_tab, kf.t[i + 1]);
    if (b - 1 > a) s2 = __dsub_rn(prefix_of(tab[b - 1]), prefix_of(tab[a]));
  }
  double w = 0.0, x = 0.0;
  if (s2 > 0.0) {
    w = __ddiv_rn(1.0, __dsqrt_rn(__dmul_rn(s2, sig2_wb)));
    x = __ddiv_rn(1.0, __dsqrt_rn(__dmul_rn(s2, sig2_ab)));
  }
  for (int c = 0; c < 3; ++c) {
    out[6 * i + c] = w;
    out[6 * i + 3 + c] = x;
  }
}

}  // namespace
}  // namespace ctvio

namespace {

using Clock = std::chrono::steady_clock;
constexpr size_t kMaxKfPairs = ctvio::kMaxKf - 1;

// the samples ingested from `first` on extend the dt^2 prefix
int extend_imu_prefix(ctvio_engine* e, int first, int n) {
  if (n <= 0) return CTVIO_OK;
  ctvio::imu_prefix_kernel<<<1, 32, 0, e->stream>>>(e->d_imu_tab_t.p, first, n, e->cyc.imu_carry.p);
  ++e->launches;
  return CTVIO_OK;
}

// the weights of the window's consecutive frames (n_kf times) into out, from the resident IMU table
int launch_bias_weights(ctvio_engine* e, int n_kf, const int64_t* kf_t, double sigma_wb, double sigma_ab, double* out) {
  ctvio::KfTimes k;
  for (int i = 0; i < n_kf; ++i) k.t[i] = kf_t[i];
  // sigma^2 as the host forms it (sigma * sigma, trajectory_manager.cpp:420-421)
  ctvio::bias_sqrt_info_kernel<<<1, 32, 0, e->stream>>>(e->d_imu_tab_t.p, int(e->h_imu_tab_t.size()), k, n_kf,
                                                         sigma_wb * sigma_wb, sigma_ab * sigma_ab, out);
  ++e->launches;
  return CTVIO_OK;
}

int check_options(const ctvio_cycle_options* o) {
  if (!o) return fail(CTVIO_ERR_INVALID, "null options");
  if (o->window_size < 2 || o->window_size > 15) return fail(CTVIO_ERR_INVALID, "window_size must be 2..15");
  if (o->solve_iterations < 1 || o->predictor_iterations < 0) return fail(CTVIO_ERR_INVALID, "bad iteration count");
  if (!(o->init_depth > 0.0) || !std::isfinite(o->init_depth)) return fail(CTVIO_ERR_INVALID, "init_depth must be positive");
  if (o->extend_ns <= 0) return fail(CTVIO_ERR_INVALID, "extend_ns must be positive");
  if (!std::isfinite(o->min_parallax)) return fail(CTVIO_ERR_INVALID, "min_parallax must be finite");
  if (!std::isfinite(o->sigma_wb_discrete) || !std::isfinite(o->sigma_ab_discrete))
    return fail(CTVIO_ERR_INVALID, "bias sigmas must be finite");
  for (const int32_t f : {o->publish_pose_covariance, o->publish_odometry_covariance, o->publish_map_covariance})
    if (f != 0 && f != 1) return fail(CTVIO_ERR_INVALID, "the publish_*_covariance options must be 0 or 1");
  if (o->covariance_gauge_knot < -1 || o->covariance_gauge_knot > 3)
    return fail(CTVIO_ERR_INVALID, "covariance_gauge_knot must be -1..3");
  if (o->publish_map_covariance && !o->publish_map)
    return fail(CTVIO_ERR_INVALID, "publish_map_covariance requires publish_map");
  return CTVIO_OK;
}

// ---- the covariance publications (ctvio_cycle_covariances) ----
constexpr int64_t kTfLagNs = 50'000'000;  // the TF time: maxTimeNs() - 50 ms (odometry_manager.cpp:287-288)

// a cycle starts: nothing it or an earlier one published is available until it completes
void clear_covariances(ctvio_engine* e) {
  auto& cv = e->cyc.cov;
  const ctvio_cycle_options& o = e->cyc.opt;
  cv.ran = false;
  cv.requested = (o.publish_pose_covariance ? 1 : 0) | (o.publish_odometry_covariance ? 2 : 0) |
                 (o.publish_map_covariance ? 4 : 0);
  cv.available = 0;
  cv.status = CTVIO_ERR_STATE;
  cv.rcond = NAN;
  cv.n_frames = cv.n_lm = cv.n_map = cv.n_map_nan = 0;
  cv.pending = false;
  cv.why = "the last cycle stopped on an error";
}

// step 9 done: Sigma of the solved window and its projections go on the stream, unless a time they need lies outside
// the spline (then the status says so and the cycle goes on)
int start_covariances(ctvio_engine* e, int64_t max_t, int n_lm) {
  auto& c = e->cyc;
  auto& cv = c.cov;
  const bool pose = cv.requested & 1, rel = cv.requested & 2, points = cv.requested & 4;
  cv.pose_t = max_t - kTfLagNs;
  cv.n_frames = c.n_frames;
  for (int k = 0; k < c.n_frames; ++k) cv.frame_t[k] = c.t[k];
  cv.n_lm = n_lm;
  // the ranges the separate calls check: the query times, and every held slot's frame time (the anchors)
  if ((pose && !times_inside(e->sp, 1, &cv.pose_t)) || (rel && !times_inside(e->sp, c.n_frames, c.t)) ||
      (points && !held_frames_inside(e))) {
    cv.status = CTVIO_ERR_TIME_RANGE;
    cv.why = "a covariance time falls outside the spline";
    return CTVIO_OK;
  }
  if (const int rc = cycle_covariance_enqueue(e, c.opt.covariance_gauge_knot, pose, rel, points)) return rc;
  cv.pending = true;
  return CTVIO_OK;
}

// after a stream synchronisation that follows start_covariances: the rank test on the published block
int finish_covariances(ctvio_engine* e) {
  auto& cv = e->cyc.cov;
  if (!cv.pending) return CTVIO_OK;
  cv.pending = false;
  const LmPublished& pub = *const_cast<const LmPublished*>(&e->cyc.cov_host->pub);
  if (*reinterpret_cast<const volatile unsigned long long*>(&pub.seq) != cv.seq)
    return fail(CTVIO_ERR_CUDA, "the window covariance was not published before the cycle's synchronisation");
  std::atomic_thread_fence(std::memory_order_acquire);
  cv.rcond = pub.rcond;
  cv.status = rank_test(pub, "window covariance", &cv.why);
  if (cv.status == CTVIO_OK) cv.available = cv.requested & 3;  // the map's bit comes with the map
  return CTVIO_OK;
}

int check_image(const ctvio_image_msg* m) {
  if (!m) return fail(CTVIO_ERR_INVALID, "null image message");
  if (m->n_points < 0 || m->n_points > ctvio_engine::kFrameCap) return fail(CTVIO_ERR_INVALID, "n_points must be 0..1024");
  if (m->n_points > 0 && (!m->points_xyz || !m->ch_id || !m->ch_v)) return fail(CTVIO_ERR_INVALID, "bad image message");
  return CTVIO_OK;
}

int check_imu(const ctvio_imu_msgs* m) {
  if (!m) return CTVIO_OK;
  if (m->n < 0 || (m->n > 0 && !m->data) || m->stride_bytes < 56 || m->off_gyro < 8 || m->off_accel < 8 ||
      m->off_gyro + 24 > m->stride_bytes || m->off_accel + 24 > m->stride_bytes)
    return fail(CTVIO_ERR_INVALID, "bad IMU record layout");
  return CTVIO_OK;
}

int check_engine(ctvio_engine* e, int32_t marg_flag_override, ctvio_cycle_result* r) {
  if (!r) return fail(CTVIO_ERR_INVALID, "null result");
  if (marg_flag_override < -1 || marg_flag_override > 1) return fail(CTVIO_ERR_INVALID, "marg_flag_override must be -1, 0 or 1");
  if (!e) return fail(CTVIO_ERR_INVALID, "null handle");
  if (e->world > 1) return fail(CTVIO_ERR_STATE, "the odometry cycle runs on a single engine, not sharded");
  return CTVIO_OK;
}

// the frame slot of the next frame: f % 16 when the feature table does not hold it, else the lowest free one (-1: none)
int free_slot(const ctvio_engine* e, int64_t f) {
  const uint32_t held = e->ft.held;
  const int s = int(f % ctvio_engine::kFrameSlots);
  if (!(held >> s & 1u)) return s;
  for (int k = 0; k < ctvio_engine::kFrameSlots; ++k)
    if (!(held >> k & 1u)) return k;
  return -1;
}

// the image's cloud into `slot`, appended to the window, added to the feature table
int take_image(ctvio_engine* e, int slot, const ctvio_image_msg* m) {
  auto& c = e->cyc;
  if (const int rc = ingest_feature_cloud_body(e, slot, m->t_ns, m->n_points, m->points_xyz, m->ch_id, m->ch_v, false)) return rc;
  c.slot[c.n_frames] = slot;
  c.t[c.n_frames] = m->t_ns;
  ++c.n_frames;
  ++c.next_frame;
  return ctvio_feature_table_add(e, slot, nullptr, nullptr);
}

int take_imu(ctvio_engine* e, const ctvio_imu_msgs* m, int64_t drop_before_ns) {
  const int n = m ? m->n : 0;
  int first = 0;
  if (!m) {
    // still retire what left the window
    return ingest_imu_body(e, 0, nullptr, 56, 8, 32, drop_before_ns, false, &first);
  }
  if (const int rc = ingest_imu_body(e, n, m->data, m->stride_bytes, m->off_gyro, m->off_accel, drop_before_ns, false, &first))
    return rc;
  return extend_imu_prefix(e, first, n);
}

ctvio_options make_opt() {
  ctvio_options o;
  std::memset(&o, 0, sizeof(o));
  o.fixed_knot_index = -1;
  return o;
}

// knot index (of the engine's window) of time t
int knot_of(const ctvio_engine* e, int64_t t) { return int((t - e->cfg.t0_ns) / e->cfg.dt_ns); }

// everything after the image and the IMU records went in: ResidentRunner.step()'s order from the feature-table window on
int run_cycle(ctvio_engine* e, bool first, int32_t marg_flag_override, int64_t nK_before, ctvio_cycle_outputs* out,
              ctvio_cycle_result* r) {
  auto& c = e->cyc;
  const ctvio_cycle_options& o = c.opt;
  const int nf = c.n_frames;
  int rc;
  // 2. the keyframe decision
  r->marg_flag = 0;
  r->n_tracked = -1;
  r->parallax_num = 0;
  r->parallax_sum = 0.0;
  if (marg_flag_override >= 0) {
    r->marg_flag = marg_flag_override;
  } else if (o.min_parallax > 0.0) {
    int32_t is_kf = 1;
    if ((rc = ctvio_check_keyframe(e, nf, c.slot, o.min_parallax, &is_kf, &r->n_tracked, &r->parallax_num, &r->parallax_sum)))
      return rc;
    r->marg_flag = is_kf ? 0 : 1;
  }
  const bool marg = r->marg_flag == 0;
  // 4. setDepth + getDepthVector
  int32_t n_lm = 0;
  if ((rc = ctvio_feature_table_window(e, nf, c.slot, o.window_size, &n_lm))) return rc;
  r->n_landmarks = n_lm;
  const int64_t dt = e->cfg.dt_ns, t0 = e->cfg.t0_ns;
  const int64_t max_t = t0 + int64_t(e->nK - 3) * dt;
  const int64_t t_newest = c.t[nf - 1];
  // the pre-solve pose of knot 0 (trajectory_manager.cpp:325-327): the predictor fixes it, so any time before the main
  // solve gives the same value
  CUDA_OK(c.snap.reserve(4 + 3 + 12));
  CUDA_OK(cudaMemcpyAsync(c.snap.p, e->x[e->cur].q.p, 4 * sizeof(double), cudaMemcpyDeviceToDevice, e->stream));
  CUDA_OK(cudaMemcpyAsync(c.snap.p + 4, e->x[e->cur].p.p, 3 * sizeof(double), cudaMemcpyDeviceToDevice, e->stream));
  // 5. InitTrajectory
  std::memset(&r->predictor, 0, sizeof(r->predictor));
  r->n_predictor_imu = 0;
  if (!first) {
    ctvio_options po = make_opt();
    po.fixed_knot_index = int32_t(nK_before - 1);
    po.lock_wb = po.lock_ab = po.fix_ld = 1;
    const int64_t max_bef_ns = t0 + (nK_before - 3) * dt;
    ctvio_set_options(e, &po);
    ctvio_clear_factors(e);
    ctvio_enable_prior(e, 0);
    if ((rc = ctvio_add_imu_from_table(e, max_bef_ns, max_t, 0, nullptr, nf - 1, -(int64_t(1) << 62), &r->n_predictor_imu)))
      return rc;
    if (r->n_predictor_imu > 0 && (rc = ctvio_solve(e, o.predictor_iterations, &r->predictor))) return rc;
  }
  // 6. FeatureManager::triangulate
  if ((rc = ctvio_triangulate_window_from_table(e, o.init_depth, &r->n_triangulated, &r->n_fallback))) return rc;
  // 7. UpdateTrajectory's problem
  ctvio_options mo = make_opt();
  mo.fix_ld = o.fix_ld;
  mo.ld_lower = o.ld_lower;
  mo.ld_upper = o.ld_upper;
  mo.is_marg_state = marg ? 1 : 0;
  mo.ctrl_to_be_opt_now = 0;
  mo.ctrl_to_be_opt_later = knot_of(e, c.t[1]);
  ctvio_set_options(e, &mo);
  ctvio_clear_factors(e);
  ctvio_enable_prior(e, 1);
  if ((rc = ctvio_add_image_features_from_table(e, marg ? 1 : 0, &r->n_image_factors))) return rc;
  const int64_t t_imu_max = std::min(max_t, t_newest + 1);
  if ((rc = ctvio_add_imu_from_table(e, t0, t_imu_max, nf, c.t, -1, marg ? c.t[1] : -(int64_t(1) << 62), &r->n_imu_factors)))
    return rc;
  CUDA_OK(c.bias_w.reserve(6 * kMaxKfPairs));
  launch_bias_weights(e, nf, c.t, o.sigma_wb_discrete, o.sigma_ab_discrete, c.bias_w.p);
  int32_t bi[16], bj[16], bm[16];
  for (int i = 0; i < nf - 1; ++i) { bi[i] = i; bj[i] = i + 1; bm[i] = (marg && i == 0) ? 1 : 0; }
  if ((rc = add_bias_factors_device(e, nf - 1, bi, bj, c.bias_w.p, bm))) return rc;
  // 8. Solve
  if ((rc = ctvio_solve(e, o.solve_iterations, &r->solve))) return rc;
  // 9. double2vector, from the snapshot (the R0 / t0 it formed land behind it)
  e->launches += ctvio::launch_gauge_realign_snapshot(e->x[e->cur].ptrs(), e->nK, 0, c.snap.p, c.snap.p + 7, e->stream);
  e->table_valid = true;
  e->mirror_valid = false;
  // the covariance publications, on the solved window's H: Sigma once, then its projections, all enqueued; the rank
  // test is read after the slide's synchronisation below
  if (c.cov.requested && (rc = start_covariances(e, max_t, n_lm))) return rc;
  r->n_frames = nf;
  r->n_knots = e->nK;
  r->knot_t0_ns = e->cfg.t0_ns;
  const bool want_knots = out && (out->q_xyzw || out->p_xyz || out->line_delay);
  if (want_knots) {
    if ((out->q_xyzw || out->p_xyz) && out->knot_capacity < e->nK)
      return fail(CTVIO_ERR_INVALID, "knot_capacity is smaller than the window's knot count");
    if ((rc = refresh_mirror(e))) return rc;  // read below, after the next synchronisation
  }
  // 10. UpdateVIOPrior
  if (marg) {
    int32_t n_out = 0, nb_out = 0;
    if ((rc = ctvio_marginalize(e, &n_out, &nb_out))) return rc;
    if (n_out > 0 && (rc = adopt_prior_body(e, true))) return rc;
    r->prior_dim = n_out;
  } else {
    r->prior_dim = e->prior.n;
  }
  // 11 - 13. the slide
  const int leave = marg ? 0 : nf - 2;
  const int leave_slot = c.slot[leave];
  const int drop_knots = mo.ctrl_to_be_opt_later;
  r->n_reanchored = 0;
  if (o.reanchor) {
    if ((rc = ctvio_feature_table_slide_reanchor(e, nf, c.slot, marg ? 1 : 0, o.init_depth, &r->n_removed, &r->n_reanchored)))
      return rc;
  }
  if (want_knots) {
    CUDA_OK(stream_sync(e->stream));  // (after the reanchoring slide's read-back this returns at once)
    const double* mq = e->h_mirror;
    const double* mp = mq + 4 * size_t(e->nK);
    if (out->q_xyzw) std::memcpy(out->q_xyzw, mq, 4 * size_t(e->nK) * sizeof(double));
    if (out->p_xyz) for (int k = 0; k < e->nK; ++k) for (int d = 0; d < 3; ++d) out->p_xyz[3 * k + d] = mp[kPStride * k + d];
    if (out->line_delay)
      *out->line_delay = e->h_mirror[(4 + kPStride) * size_t(e->nK) + 6 * size_t(std::max(e->nB, 1)) + size_t(std::max(e->nL, 1))];
    e->d2h_bytes += size_t(e->nK) * (((out->q_xyzw) ? 32 : 0) + ((out->p_xyz) ? 32 : 0));
  }
  if (marg) rc = ctvio_slide_window(e, drop_knots, 1, 1);
  else rc = ctvio_slide_window_second_new(e);
  if (rc) return rc;
  if (!o.reanchor && (rc = ctvio_feature_table_slide(e, leave_slot, &r->n_removed))) return rc;
  r->n_knots_after = e->nK;
  for (int k = leave; k + 1 < nf; ++k) { c.slot[k] = c.slot[k + 1]; c.t[k] = c.t[k + 1]; }
  --c.n_frames;
  // both branches have synchronised since step 9 (the feature table's slide reads its counts back)
  if ((rc = finish_covariances(e))) return rc;
  // 14. the map of the post-slide window, with each point's covariance when Sigma passed the rank test
  r->n_map_points = r->n_margin_points = 0;
  if (o.publish_map) {
    const bool pts = out && out->map_xyz && out->map_feature_id && out->map_in_margin_cloud;
    const bool cov = (c.cov.requested & 4) && c.cov.status == CTVIO_OK;
    auto& t = e->ft;
    if ((rc = feature_table_map_body(e, c.n_frames, c.slot, o.window_size, pts ? out->map_capacity : 0, pts ? out->map_xyz : nullptr,
                                     pts ? out->map_feature_id : nullptr, pts ? out->map_in_margin_cloud : nullptr,
                                     &r->n_map_points, out ? out->cam_q_xyzw : nullptr, out ? out->cam_p_xyz : nullptr,
                                     cov ? cycle_point_covariances(e) : nullptr, cov ? c.cov.n_lm : 0,
                                     cov ? &c.cov_host->map_cov9[0] : nullptr))) {
      if (!(rc == CTVIO_ERR_INVALID && !pts)) return rc;  // a map without point buffers: only the count is wanted
    }
    int nm = 0;
    for (int k = 0; k < r->n_map_points; ++k) nm += t.h_map_points[k].in_margin_cloud ? 1 : 0;
    r->n_margin_points = nm;
    if (!pts) e->d2h_bytes -= sizeof(ctvio::MapPoint) * size_t(r->n_map_points);  // the points stayed in the mapped buffer
    if (cov) {
      int nan_rows = 0;
      for (int k = 0; k < r->n_map_points; ++k) nan_rows += std::isnan(c.cov_host->map_cov9[9 * size_t(k)]) ? 1 : 0;
      c.cov.n_map = r->n_map_points;
      c.cov.n_map_nan = nan_rows;
      c.cov.available |= 4;
    }
  }
  c.cov.ran = true;
  if (!c.cov.requested) c.cov.why = "the cycle's options publish no covariances";
  return CTVIO_OK;
}

}  // namespace

int ctvio::host::check_cycle_options(const ctvio_cycle_options* o) { return check_options(o); }

extern "C" {

int ctvio_cycle_default_options(ctvio_cycle_options* o) {
  if (!o) return fail(CTVIO_ERR_INVALID, "null options");
  std::memset(o, 0, sizeof(*o));
  o->window_size = 10;
  o->solve_iterations = 15;
  o->predictor_iterations = 8;
  o->fix_ld = 0;
  o->min_parallax = 0.0;
  o->init_depth = 5.0;
  o->extend_ns = 40'000'000;
  o->ld_lower = 0.0;
  o->ld_upper = 35e-6;
  o->sigma_wb_discrete = 2.0e-5;
  o->sigma_ab_discrete = 4.0e-4;
  o->reanchor = 0;
  o->publish_map = 1;
  o->covariance_gauge_knot = 3;
  return CTVIO_OK;
}

int ctvio_odometry_start(ctvio_handle e, const ctvio_cycle_options* opt, int64_t t0_ns, int32_t n_knots, const double* q,
                         const double* p, int32_t n_frames, const ctvio_image_msg* frames, const double* bg_ba6, double ld,
                         const ctvio_imu_msgs* imu, int32_t marg_flag_override, ctvio_cycle_outputs* out,
                         ctvio_cycle_result* r) {
  const auto t_start = Clock::now();
  int rc;
  if ((rc = check_options(opt))) return rc;
  if (n_frames != opt->window_size + 1) return fail(CTVIO_ERR_INVALID, "n_frames must be window_size + 1");
  if (n_knots < 4 || !q || !p || !frames || !bg_ba6) return fail(CTVIO_ERR_INVALID, "bad initial state");
  for (int k = 0; k < n_frames; ++k)
    if ((rc = check_image(&frames[k]))) return rc;
  if ((rc = check_imu(imu))) return rc;
  if ((rc = check_engine(e, marg_flag_override, r))) return rc;
  cudaSetDevice(e->cfg.device);
  std::memset(r, 0, sizeof(*r));
  auto& c = e->cyc;
  // a fresh run: feature table, frame slots, IMU table and prior start empty
  c.started = false;
  c.opt = *opt;
  clear_covariances(e);
  c.n_frames = 0;
  c.next_frame = 0;
  e->ft.held = 0;
  e->ft.n_entries = 0;
  e->ft.n_lm = -1;
  e->ft.window_current = false;
  e->h_frame_ingested = 0;
  e->h_imu_tab_t.clear();
  CUDA_OK(c.imu_carry.reserve(3));
  CUDA_OK(cudaMemsetAsync(c.imu_carry.p, 0, 3 * sizeof(double), e->stream));
  ctvio_clear_factors(e);
  if ((rc = ctvio_set_prior(e, 0, nullptr, nullptr, 0, nullptr, nullptr, nullptr, nullptr))) return rc;
  e->new_prior = ctvio::PriorHost();
  if ((rc = ctvio_set_time_origin(e, t0_ns))) return rc;
  if ((rc = ctvio_set_knots(e, n_knots, q, p))) return rc;
  if ((rc = ctvio_set_biases(e, n_frames, bg_ba6))) return rc;
  if ((rc = ctvio_set_line_delay(e, ld))) return rc;
  for (int k = 0; k < n_frames; ++k) {
    const int slot = free_slot(e, c.next_frame);
    if ((rc = take_image(e, slot, &frames[k]))) return rc;
  }
  r->frame_slot = c.slot[n_frames - 1];
  if ((rc = take_imu(e, imu, e->cfg.t0_ns + int64_t(knot_of(e, c.t[0])) * e->cfg.dt_ns))) return rc;
  c.started = true;
  rc = run_cycle(e, true, marg_flag_override, e->nK, out, r);
  if (rc) c.started = false;
  r->host_ms = std::chrono::duration<double, std::milli>(Clock::now() - t_start).count();
  return rc;
}

int ctvio_process_image(ctvio_handle e, const ctvio_image_msg* img, const ctvio_imu_msgs* imu, int32_t marg_flag_override,
                        ctvio_cycle_outputs* out, ctvio_cycle_result* r) {
  const auto t_start = Clock::now();
  int rc;
  if ((rc = check_image(img))) return rc;
  if ((rc = check_imu(imu))) return rc;
  if ((rc = check_engine(e, marg_flag_override, r))) return rc;
  auto& c = e->cyc;
  if (!c.started) return fail(CTVIO_ERR_STATE, "ctvio_odometry_start has not run (or its run stopped on an error)");
  const int slot = free_slot(e, c.next_frame);
  if (slot < 0 || c.n_frames >= ctvio_engine::kFrameSlots) return fail(CTVIO_ERR_STATE, "no free frame slot: all 16 are held");
  cudaSetDevice(e->cfg.device);
  std::memset(r, 0, sizeof(*r));
  c.started = false;  // until the cycle completes
  clear_covariances(e);
  // 1. the cloud joins the window and the feature table
  if ((rc = take_image(e, slot, img))) return rc;
  r->frame_slot = slot;
  // 3. ExtendTrajectory, then the IMU records (retiring what is older than the window's first knot)
  const int64_t nK_before = e->nK;
  if ((rc = ctvio_extend_knots_to(e, img->t_ns + c.opt.extend_ns, nullptr))) return rc;
  if ((rc = take_imu(e, imu, e->cfg.t0_ns + int64_t(knot_of(e, c.t[0])) * e->cfg.dt_ns))) return rc;
  rc = run_cycle(e, false, marg_flag_override, nK_before, out, r);
  if (!rc) c.started = true;
  r->host_ms = std::chrono::duration<double, std::milli>(Clock::now() - t_start).count();
  return rc;
}

int ctvio_cycle_covariances(ctvio_handle e, double* cov12, int64_t* pose_t_ns, double* cov6, int64_t* pair_t_ns,
                            int32_t map_capacity, double* map_cov9, ctvio_cycle_covariance_info* info) {
  if (!e) return fail(CTVIO_ERR_INVALID, "null handle");
  if (map_capacity < 0) return fail(CTVIO_ERR_INVALID, "map_capacity must be >= 0");
  const auto& cv = e->cyc.cov;
  const bool ok = cv.ran && cv.available;
  const int n_pairs = (ok && (cv.available & 2)) ? cv.n_frames - 1 : 0;
  const int n_map = (ok && (cv.available & 4)) ? cv.n_map : 0;
  if (info) {
    std::memset(info, 0, sizeof(*info));
    info->requested = cv.requested;
    info->available = ok ? cv.available : 0;
    info->status = cv.ran ? cv.status : CTVIO_ERR_STATE;
    info->gauge_knot = e->cyc.opt.covariance_gauge_knot;
    info->rcond = cv.ran ? cv.rcond : NAN;
    info->pose_t_ns = cv.pose_t;
    info->n_pairs = n_pairs;
    info->n_map_points = n_map;
    info->n_map_points_without_cov = (ok && (cv.available & 4)) ? cv.n_map_nan : 0;
  }
  if (!ok) return fail(CTVIO_ERR_STATE, "ctvio_cycle_covariances: not available: " + cv.why);
  if (map_cov9 && map_capacity < n_map)
    return fail(CTVIO_ERR_INVALID, "ctvio_cycle_covariances: map_capacity is smaller than the map's point count");
  const CycleCovHost* h = e->cyc.cov_host;
  if (cv.available & 1) {
    if (cov12) std::memcpy(cov12, h->cov12, 144 * sizeof(double));
    if (pose_t_ns) *pose_t_ns = cv.pose_t;
  }
  if (cov6) std::memcpy(cov6, h->cov6, 36 * size_t(n_pairs) * sizeof(double));
  for (int k = 0; pair_t_ns && k < n_pairs; ++k) {
    pair_t_ns[2 * k] = cv.frame_t[k];
    pair_t_ns[2 * k + 1] = cv.frame_t[k + 1];
  }
  if (map_cov9) std::memcpy(map_cov9, h->map_cov9, 9 * size_t(n_map) * sizeof(double));
  return CTVIO_OK;
}

int ctvio_debug_bias_weights(ctvio_handle e, int32_t n_kf, const int64_t* kf_t, double sigma_wb, double sigma_ab,
                             double* out) {
  if (!e) return fail(CTVIO_ERR_INVALID, "null handle");
  if (n_kf < 2 || n_kf > ctvio::kMaxKf || !kf_t || !out) return fail(CTVIO_ERR_INVALID, "bad argument");
  for (int i = 1; i < n_kf; ++i)
    if (kf_t[i] < kf_t[i - 1]) return fail(CTVIO_ERR_INVALID, "keyframe times must ascend");
  cudaSetDevice(e->cfg.device);
  auto& c = e->cyc;
  CUDA_OK(c.bias_w.reserve(6 * kMaxKfPairs));
  launch_bias_weights(e, n_kf, kf_t, sigma_wb, sigma_ab, c.bias_w.p);
  CUDA_OK(cudaMemcpyAsync(out, c.bias_w.p, 6 * size_t(n_kf - 1) * sizeof(double), cudaMemcpyDeviceToHost, e->stream));
  CUDA_OK(stream_sync(e->stream));
  return CTVIO_OK;
}

}  // extern "C"
