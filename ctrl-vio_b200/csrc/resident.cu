// Host side of the device-resident window: the entry points of include/ctvio.h's sections device-resident sliding window,
// keyframe, wire formats, resident feature table and front-end DLT, which launch the kernels of frontend.cu.
#include <cmath>

#include "engine_state.h"

namespace {

// the inverse depths just written into the other state buffer become the current ones
void swap_rho(ctvio_engine* e) { swap(e->x[e->cur].rho, e->x[e->cur ^ 1].rho); }

// the caller's window of 1..kFrameSlots frame slots (n_frames checked by the caller), oldest to newest, each listed once
int parse_window_slots(int32_t n_frames, const int32_t* frame_slots, ctvio::WindowSlots& w) {
  w.n_frames = n_frames;
  w.listed = 0;
  for (int s = 0; s < ctvio_engine::kFrameSlots; ++s) w.position[s] = -1;
  for (int k = 0; k < n_frames; ++k) {
    const int s = frame_slots[k];
    if (s < 0 || s >= ctvio_engine::kFrameSlots) return fail(CTVIO_ERR_INVALID, "frame slot out of range");
    if (w.listed & (1u << s)) return fail(CTVIO_ERR_INVALID, "a frame slot is listed twice");
    w.listed |= 1u << s;
    w.slot[k] = s;
    w.position[s] = k;
  }
  return CTVIO_OK;
}

// What a call needs of the feature table's last window (ctvio_feature_table_window).  kCurrent: the window still
// describes the table (no add / slide since).  kCurrentNumbered: that, and the resident inverse depths follow the
// window's numbering.  kNumbered: the resident inverse depths follow the last window's numbering, if there was a window.
enum class TableWindow { kCurrent, kCurrentNumbered, kNumbered };
int check_numbering(ctvio_engine* e, TableWindow need) {
  if (need != TableWindow::kNumbered && !e->ft.window_current)
    return fail(CTVIO_ERR_STATE, "no feature-table window since the last add / slide");
  const int n_lm = e->ft.n_lm;
  const bool numbered = need == TableWindow::kCurrent || e->nL == n_lm || (need == TableWindow::kNumbered && n_lm < 0);
  if (!numbered) return fail(CTVIO_ERR_STATE, "the resident inverse depths no longer follow the table's numbering");
  return CTVIO_OK;
}

// DLT of the resident window (ctvio_triangulate_window, ctvio_triangulate_window_from_table) from a device-resident
// observation CSR
int triangulate_window_device(ctvio_engine* e, int nl, const int32_t* d_off, const int32_t* d_slot, const int32_t* d_idx,
                              double init_depth, int32_t* n_triangulated, int32_t* n_fallback) {
  cudaStream_t st = e->stream;
  ensure_table(e);
  const int other = e->cur ^ 1;
  CUDA_OK(e->x[other].rho.reserve(size_t(nl) + 1));
  CUDA_OK(e->d_tri_cnt.reserve(2));
  CUDA_OK(cudaMemsetAsync(e->d_tri_cnt.p, 0, 2 * sizeof(int32_t), st));
  ctvio::TriangulateWindowArgs a;
  a.n_landmarks = nl; a.obs_offset = d_off; a.obs_slot = d_slot; a.obs_idx = d_idx;
  a.table = e->d_frames.p; a.frame_t = e->d_frame_t.p; a.frame_cap = ctvio_engine::kFrameCap;
  a.st = e->x[e->cur].ptrs(); a.sp = e->sp; a.R_CI = e->rig.R_CI; a.p_CI = e->rig.p_CI;
  a.init_depth = init_depth;
  // written into the other state buffer's array and swapped in only on success: after CTVIO_ERR_TIME_RANGE the
  // resident inverse depths are the ones before the call
  a.rho_in = e->x[e->cur].rho.p; a.rho_out = e->x[other].rho.p;
  a.counts = e->d_tri_cnt.p;
  e->launches += ctvio::launch_triangulate_window(a, st);
  int32_t cnt[2];
  if (const int rc = read_result(e, cnt, e->d_tri_cnt.p, 2)) return rc;
  if (cnt[0] < 0) return fail(CTVIO_ERR_TIME_RANGE, "an observation's row time falls outside the spline");
  swap_rho(e);
  e->mirror_valid = false;
  if (n_triangulated) *n_triangulated = cnt[0];
  if (n_fallback) *n_fallback = cnt[1];
  return CTVIO_OK;
}

}  // namespace

// the resident feature table's arrays, at full size (kFeatureTableMaxEntries entries), on first use
int ctvio::host::ensure_feature_table(ctvio_engine* e) {
  auto& t = e->ft;
  if (t.id.p) return CTVIO_OK;
  const size_t cap = ctvio::kFeatureTableMaxEntries, slots = ctvio_engine::kFrameSlots;
  CUDA_OK(e->d_frames.reserve(slots * ctvio_engine::kFrameCap));
  CUDA_OK(t.id.reserve(cap)); CUDA_OK(t.anchor.reserve(cap)); CUDA_OK(t.lm.reserve(cap)); CUDA_OK(t.mask.reserve(cap));
  CUDA_OK(t.rho.reserve(cap)); CUDA_OK(t.idx.reserve(slots * cap)); CUDA_OK(t.new_index.reserve(cap));
  CUDA_OK(t.key[0].reserve(cap)); CUDA_OK(t.key[1].reserve(cap));
  CUDA_OK(t.obs_offset.reserve(cap + 1)); CUDA_OK(t.obs_slot.reserve(slots * cap)); CUDA_OK(t.obs_idx.reserve(slots * cap));
  CUDA_OK(t.lm_id.reserve(cap)); CUDA_OK(t.lm_anchor.reserve(cap)); CUDA_OK(t.lm_used.reserve(cap));
  CUDA_OK(t.result.reserve(2));
  CUDA_OK(t.desc.reserve((slots - 1) * cap));
  return CTVIO_OK;
}

namespace {

// room for n descriptors in the factor set's device-side list, keeping the ones it holds
int reserve_device_descriptors(ctvio_engine* e, size_t n) {
  if (n > e->d_img_in.cap) CUDA_OK(e->d_img_in.grow(2 * n, 0, size_t(e->n_img_dev), e->stream));
  return CTVIO_OK;
}

// append descriptors to the factor set's device-side list (staged through the caller's arena)
int append_device_descriptors(ctvio_engine* e, const std::vector<ctvio::FactorDesc>& d) {
  const size_t base = size_t(e->n_img_dev), bytes = d.size() * sizeof(ctvio::FactorDesc);
  if (const int rc = reserve_device_descriptors(e, base + d.size())) return rc;
  CUDA_OK(staged_h2d(e->d_img_in.p + base, d.data(), bytes, e->stream));
  e->h2d_bytes += bytes;
  e->n_img_dev += int(d.size());
  return CTVIO_OK;
}

}  // namespace


namespace ctvio::host {

// ctvio_ingest_feature_cloud after its argument checks; sync = false leaves the copies in flight (the odometry cycle
// synchronises later in the same call, before its caller's buffers can go away)
int ingest_feature_cloud_body(ctvio_engine* e, int32_t slot, int64_t t_ns, int32_t n, const float* points, const float* ch_id,
                              const float* ch_v, bool sync) {
  cudaStream_t st = e->stream;
  CUDA_OK(e->d_frames.reserve(size_t(ctvio_engine::kFrameSlots) * ctvio_engine::kFrameCap));
  CUDA_OK(e->d_frame_t.reserve(ctvio_engine::kFrameSlots));
  CUDA_OK(e->d_cloud_stage.reserve(5 * size_t(ctvio_engine::kFrameCap)));
  e->h_frame_t[slot] = t_ns;
  e->h_frame_n[slot] = n;
  e->h_frame_ingested |= 1u << slot;
  CUDA_OK(cudaMemcpyAsync(e->d_frame_t.p + slot, &e->h_frame_t[slot], sizeof(int64_t), cudaMemcpyHostToDevice, st));
  if (n) {
    // the message arrays go up AS THEY ARE (packed float32 triples + float32 channels); conversion happens on the device
    CUDA_OK(cudaMemcpyAsync(e->d_cloud_stage.p, points, 3 * size_t(n) * sizeof(float), cudaMemcpyHostToDevice, st));
    CUDA_OK(cudaMemcpyAsync(e->d_cloud_stage.p + 3 * size_t(n), ch_id, size_t(n) * sizeof(float), cudaMemcpyHostToDevice, st));
    CUDA_OK(cudaMemcpyAsync(e->d_cloud_stage.p + 4 * size_t(n), ch_v, size_t(n) * sizeof(float), cudaMemcpyHostToDevice, st));
    e->h2d_bytes += 5 * size_t(n) * sizeof(float) + 8;
    ctvio::UnpackCloudArgs a;
    a.n = n; a.points = e->d_cloud_stage.p; a.ch_id = e->d_cloud_stage.p + 3 * size_t(n); a.ch_v = e->d_cloud_stage.p + 4 * size_t(n);
    a.out = e->d_frames.p + size_t(slot) * ctvio_engine::kFrameCap;
    e->launches += ctvio::launch_unpack_cloud(a, st);
  }
  if (sync) CUDA_OK(stream_sync(st));
  return CTVIO_OK;
}

// ctvio_ingest_imu after its argument checks.  *first_new (may be null): the table index of the first appended sample.
int ingest_imu_body(ctvio_engine* e, int32_t n, const void* records, int32_t stride, int32_t off_gyro, int32_t off_accel,
                    int64_t drop_before_ns, bool sync, int* first_new) {
  cudaStream_t st = e->stream;
  // retire samples older than drop_before_ns (RemoveIMUData, trajectory_manager.cpp:472-475): a device-side shift
  size_t keep_from = 0;
  while (keep_from < e->h_imu_tab_t.size() && e->h_imu_tab_t[keep_from] < drop_before_ns) ++keep_from;
  const size_t kept = e->h_imu_tab_t.size() - keep_from, total = kept + size_t(n);
  if (e->d_imu_tab_t.cap < total) {
    CUDA_OK(e->d_imu_tab_t.grow(2 * total + 256, keep_from, kept, st));
    CUDA_OK(e->d_imu_tab_ga.grow(3 * (2 * total + 256), 3 * keep_from, 3 * kept, st));
  } else if (keep_from > 0 && kept > 0) {
    CUDA_OK(e->d_tmp.reserve(8 * kept));
    e->launches += ctvio::launch_shift_imu_table(e->d_imu_tab_t.p, e->d_imu_tab_ga.p, int(keep_from), int(kept), e->d_tmp.p, st);
  }
  e->h_imu_tab_t.erase(e->h_imu_tab_t.begin(), e->h_imu_tab_t.begin() + keep_from);
  if (first_new) *first_new = int(kept);
  if (n) {
    CUDA_OK(e->d_imu_raw.reserve(size_t(n) * stride));
    CUDA_OK(cudaMemcpyAsync(e->d_imu_raw.p, records, size_t(n) * stride, cudaMemcpyHostToDevice, st));  // records as they are
    e->h2d_bytes += size_t(n) * stride;
    ctvio::UnpackImuArgs a;
    a.n = n; a.raw = e->d_imu_raw.p; a.stride = stride; a.off_gyro = off_gyro; a.off_accel = off_accel;
    a.kf_t = nullptr; a.n_kf = 0; a.dst0 = int(kept); a.t_node = e->d_imu_tab_t.p; a.ga = e->d_imu_tab_ga.p;
    e->launches += ctvio::launch_unpack_imu(a, st);
    const unsigned char* rec = static_cast<const unsigned char*>(records);
    for (int k = 0; k < n; ++k) {
      int64_t t;
      std::memcpy(&t, rec + size_t(k) * stride, sizeof(t));
      e->h_imu_tab_t.push_back(t);
    }
    if (sync) CUDA_OK(stream_sync(st));
  }
  return CTVIO_OK;
}

}  // namespace ctvio::host

// =================================================================================================
extern "C" {

int ctvio_triangulate(ctvio_handle e, int32_t n_frames, const double* Rs, const double* Ps, const double* ric,
                      const double* tic, int32_t nl, const int32_t* start_frame, const int32_t* obs_offset,
                      const double* obs_point, int32_t window_size, double init_depth, double* depth) {
  if (!e || n_frames <= 0 || !Rs || !Ps || !ric || !tic || nl < 0 || (nl > 0 && (!start_frame || !obs_offset || !obs_point || !depth)))
    return fail(CTVIO_ERR_INVALID, "bad argument");
  if (nl == 0) return CTVIO_OK;
  cudaSetDevice(e->cfg.device);
  const int total = obs_offset[nl];
  if (total < 0) return fail(CTVIO_ERR_INVALID, "obs_offset must be non-decreasing");
  for (int l = 0; l < nl; ++l)
    if (obs_offset[l + 1] < obs_offset[l]) return fail(CTVIO_ERR_INVALID, "obs_offset must be non-decreasing");
  cudaStream_t st = e->stream;
  // one staging buffer: [Rs | Ps | obs points | depth] doubles, [start | offsets] ints
  const size_t nd = 12 * size_t(n_frames) + 3 * size_t(total) + size_t(nl);
  CUDA_OK(e->d_tmp.reserve(nd));
  CUDA_OK(e->d_tri_idx.reserve(2 * size_t(nl) + 1));
  double* dRs = e->d_tmp.p;
  double* dPs = dRs + 9 * size_t(n_frames);
  double* dobs = dPs + 3 * size_t(n_frames);
  double* ddepth = dobs + 3 * size_t(total);
  CUDA_OK(cudaMemcpyAsync(dRs, Rs, 9 * size_t(n_frames) * sizeof(double), cudaMemcpyHostToDevice, st));
  CUDA_OK(cudaMemcpyAsync(dPs, Ps, 3 * size_t(n_frames) * sizeof(double), cudaMemcpyHostToDevice, st));
  if (total) CUDA_OK(cudaMemcpyAsync(dobs, obs_point, 3 * size_t(total) * sizeof(double), cudaMemcpyHostToDevice, st));
  CUDA_OK(cudaMemcpyAsync(ddepth, depth, size_t(nl) * sizeof(double), cudaMemcpyHostToDevice, st));
  CUDA_OK(cudaMemcpyAsync(e->d_tri_idx.p, start_frame, size_t(nl) * sizeof(int32_t), cudaMemcpyHostToDevice, st));
  CUDA_OK(cudaMemcpyAsync(e->d_tri_idx.p + nl, obs_offset, (size_t(nl) + 1) * sizeof(int32_t), cudaMemcpyHostToDevice, st));
  ctvio::TriangulateArgs a;
  a.n_frames = n_frames; a.Rs = dRs; a.Ps = dPs;
  for (int k = 0; k < 9; ++k) a.ric.m[k] = ric[k];
  a.tic = V3{tic[0], tic[1], tic[2]};
  a.n_landmarks = nl; a.start_frame = e->d_tri_idx.p; a.obs_offset = e->d_tri_idx.p + nl; a.obs_point = dobs;
  a.window_size = window_size; a.init_depth = init_depth; a.depth = ddepth;
  e->launches += ctvio::launch_triangulate(a, st);
  CUDA_OK(cudaMemcpyAsync(depth, ddepth, size_t(nl) * sizeof(double), cudaMemcpyDeviceToHost, st));
  CUDA_OK(stream_sync(st));
  return CTVIO_OK;
}

// ---- device-resident sliding window (SURVEY 8f-1) -------------------------------------------------
int ctvio_extend_knots_to(ctvio_handle e, int64_t t_ns, int32_t* n_out) {
  if (!e || !e->have_knots) return fail(CTVIO_ERR_STATE, "knots have not been set");
  cudaSetDevice(e->cfg.device);
  int n = e->nK;
  while (n < 4 || e->cfg.t0_ns + int64_t(n - 3) * e->cfg.dt_ns < t_ns) ++n;  // se3_spline.h:201-207
  if (n != e->nK) {
    const int old = e->nK;
    // grow both state buffers, keeping the current knots (the knot-pair table is rebuilt)
    for (int b = 0; b < 2; ++b) {
      DevState& x = e->x[b];
      if (x.q.cap < 4 * size_t(n) || x.p.cap < kPStride * size_t(n) || x.tab.cap < size_t(n)) {
        CUDA_OK(x.q.grow(4 * size_t(n) + 64, 0, b == e->cur ? 4 * size_t(old) : 0, e->stream));
        CUDA_OK(x.p.grow(kPStride * size_t(n) + 64, 0, b == e->cur ? kPStride * size_t(old) : 0, e->stream));
        CUDA_OK(x.tab.grow(size_t(n) + 16, 0, 0, e->stream));
      }
    }
    e->launches += ctvio::launch_extend_knots(e->x[e->cur].ptrs(), old, n, e->stream);
    e->nK = n;
    e->sp.n_knots = n;
    e->structure_dirty = true;
    e->table_valid = false;
    e->mirror_valid = false;
  }
  if (n_out) *n_out = n;
  return CTVIO_OK;
}

int ctvio_slide_window(ctvio_handle e, int32_t drop_knots, int32_t drop_bias, int32_t new_bias) {
  if (!e || !e->have_knots) return fail(CTVIO_ERR_STATE, "knots have not been set");
  if (drop_knots < 0 || drop_bias < 0 || new_bias < 0 || e->nK - drop_knots < 4 || drop_bias > e->nB)
    return fail(CTVIO_ERR_INVALID, "slide out of range");
  cudaSetDevice(e->cfg.device);
  const int nB_new = e->nB - drop_bias + new_bias;
  for (int b = 0; b < 2; ++b)
    if (e->x[b].bias.cap < 6 * size_t(std::max(nB_new, 1)))
      CUDA_OK(e->x[b].bias.grow(6 * size_t(nB_new) + 96, 0, b == e->cur ? 6 * size_t(e->nB) : 0, e->stream));
  // the shift runs in a scratch copy (overlapping ranges), all on the device
  CUDA_OK(e->d_tmp.reserve(size_t(8) * e->nK + 6 * size_t(std::max(e->nB, 1)) + 16));
  e->launches += ctvio::launch_slide_state(e->x[e->cur].ptrs(), e->nK, e->nB, drop_knots, drop_bias, new_bias, e->d_tmp.p, e->stream);
  e->nK -= drop_knots;
  e->sp.n_knots = e->nK;
  e->nB = nB_new;
  e->cfg.t0_ns += int64_t(drop_knots) * e->cfg.dt_ns;
  e->sp.t0_ns = e->cfg.t0_ns;
  // the active prior's blocks follow the window: knot / bias-node indices are window relative
  for (size_t b = 0; b < e->prior.type.size(); ++b) {
    const int t = e->prior.type[b];
    if (!ctvio::block_is_knot(t) && !ctvio::block_is_bias(t)) continue;
    e->prior.index[b] -= ctvio::block_is_knot(t) ? drop_knots : drop_bias;
    if (e->prior.index[b] < 0) return fail(CTVIO_ERR_STATE, "a block of the active prior left the window");
  }
  e->prior_dirty = true;
  e->masks_dirty = true;
  e->structure_dirty = true;
  e->table_valid = false;
  e->mirror_valid = false;
  return CTVIO_OK;
}

int ctvio_remap_landmarks(ctvio_handle e, int32_t n_new, const int32_t* old_index, const double* init_rho) {
  if (!e || n_new < 0 || (n_new > 0 && (!old_index || !init_rho))) return fail(CTVIO_ERR_INVALID, "bad argument");
  cudaSetDevice(e->cfg.device);
  for (int k = 0; k < n_new; ++k)
    if (old_index[k] >= e->nL) return fail(CTVIO_ERR_INVALID, "old landmark index out of range");
  cudaStream_t st = e->stream;
  CUDA_OK(e->d_tmp.reserve(size_t(n_new) + 8));
  CUDA_OK(e->d_tri_idx.reserve(size_t(n_new) + 1));
  const int other = e->cur ^ 1;
  for (int b = 0; b < 2; ++b) CUDA_OK(e->x[b].rho.reserve(size_t(std::max(n_new, e->nL)) + 1));
  if (n_new) {
    CUDA_OK(cudaMemcpyAsync(e->d_tmp.p, init_rho, size_t(n_new) * sizeof(double), cudaMemcpyHostToDevice, st));
    CUDA_OK(cudaMemcpyAsync(e->d_tri_idx.p, old_index, size_t(n_new) * sizeof(int32_t), cudaMemcpyHostToDevice, st));
    e->h2d_bytes += size_t(n_new) * 12;
    // gather into the other state buffer's array, then swap the pointers (no aliasing)
    e->launches += ctvio::launch_remap_rho(e->x[e->cur].rho.p, e->d_tri_idx.p, e->d_tmp.p, n_new, e->x[other].rho.p, st);
    CUDA_OK(stream_sync(st));
    swap_rho(e);
  }
  if (n_new != e->nL) e->structure_dirty = true;
  e->mirror_valid = false;
  e->nL = n_new;
  e->have_rho = true;
  return CTVIO_OK;
}

int ctvio_triangulate_window(ctvio_handle e, int32_t nl, const int32_t* obs_offset, const int32_t* obs_slot, const int32_t* obs_idx,
                             double init_depth, int32_t* n_triangulated, int32_t* n_fallback) {
  if (!e) return fail(CTVIO_ERR_INVALID, "null handle");
  if (!e->have_knots) return fail(CTVIO_ERR_STATE, "knots have not been set");
  if (!e->x[e->cur].ld.p) return fail(CTVIO_ERR_STATE, "the line delay has not been set");
  if (nl != e->nL) return fail(CTVIO_ERR_INVALID, "n_landmarks differs from the engine's landmark count");
  if (!(init_depth > 0.0) || !std::isfinite(init_depth)) return fail(CTVIO_ERR_INVALID, "init_depth must be positive");
  if (nl > 0 && !obs_offset) return fail(CTVIO_ERR_INVALID, "null obs_offset");
  if (nl > 0 && obs_offset[0] != 0) return fail(CTVIO_ERR_INVALID, "obs_offset[0] must be 0");
  for (int l = 0; l < nl; ++l)
    if (obs_offset[l + 1] < obs_offset[l]) return fail(CTVIO_ERR_INVALID, "obs_offset must be non-decreasing");
  const int total = nl > 0 ? obs_offset[nl] : 0;
  if (total > 0 && (!obs_slot || !obs_idx)) return fail(CTVIO_ERR_INVALID, "null observation array");
  for (int k = 0; k < total; ++k) {
    const int s = obs_slot[k];
    if (s < 0 || s >= ctvio_engine::kFrameSlots || obs_idx[k] < 0 || obs_idx[k] >= e->h_frame_n[s])
      return fail(CTVIO_ERR_INVALID, "feature slot / index out of range");
  }
  if (n_triangulated) *n_triangulated = 0;
  if (n_fallback) *n_fallback = 0;
  if (nl == 0) return CTVIO_OK;
  cudaSetDevice(e->cfg.device);
  ArenaScope arena(e);
  cudaStream_t st = e->stream;
  CUDA_OK(e->d_tri_idx.reserve(size_t(nl) + 1 + 2 * size_t(total)));
  int32_t* d_off = e->d_tri_idx.p;
  int32_t* d_slot = d_off + nl + 1;
  int32_t* d_idx = d_slot + total;
  // only the three index arrays go up: bearings, rows, frame times, knots and the line delay are resident
  CUDA_OK(staged_h2d(d_off, obs_offset, (size_t(nl) + 1) * sizeof(int32_t), st));
  CUDA_OK(staged_h2d(d_slot, obs_slot, size_t(total) * sizeof(int32_t), st));
  CUDA_OK(staged_h2d(d_idx, obs_idx, size_t(total) * sizeof(int32_t), st));
  e->h2d_bytes += (size_t(nl) + 1 + 2 * size_t(total)) * sizeof(int32_t);
  return triangulate_window_device(e, nl, d_off, d_slot, d_idx, init_depth, n_triangulated, n_fallback);
}

int ctvio_triangulate_window_from_table(ctvio_handle e, double init_depth, int32_t* n_triangulated, int32_t* n_fallback) {
  if (!e) return fail(CTVIO_ERR_INVALID, "null handle");
  if (!e->have_knots) return fail(CTVIO_ERR_STATE, "knots have not been set");
  if (!e->x[e->cur].ld.p) return fail(CTVIO_ERR_STATE, "the line delay has not been set");
  if (!(init_depth > 0.0) || !std::isfinite(init_depth)) return fail(CTVIO_ERR_INVALID, "init_depth must be positive");
  if (const int rc = check_numbering(e, TableWindow::kCurrentNumbered)) return rc;
  if (n_triangulated) *n_triangulated = 0;
  if (n_fallback) *n_fallback = 0;
  if (e->nL == 0) return CTVIO_OK;
  cudaSetDevice(e->cfg.device);
  // the CSR was built on the device by ctvio_feature_table_window: nothing goes up
  return triangulate_window_device(e, e->nL, e->ft.obs_offset.p, e->ft.obs_slot.p, e->ft.obs_idx.p, init_depth, n_triangulated,
                                   n_fallback);
}

int ctvio_feature_table_add(ctvio_handle e, int32_t frame_slot, int32_t* n_tracked, int32_t* n_new) {
  if (!e) return fail(CTVIO_ERR_INVALID, "null handle");
  if (frame_slot < 0 || frame_slot >= ctvio_engine::kFrameSlots) return fail(CTVIO_ERR_INVALID, "frame slot out of range");
  if (!(e->h_frame_ingested >> frame_slot & 1u)) return fail(CTVIO_ERR_INVALID, "no feature cloud was ingested into the slot");
  if (e->ft.held >> frame_slot & 1u) return fail(CTVIO_ERR_STATE, "the feature table still holds the slot");
  cudaSetDevice(e->cfg.device);
  if (const int rc = ensure_feature_table(e)) return rc;
  cudaStream_t st = e->stream;
  auto& t = e->ft;
  ctvio::FeatureTableAddArgs a;
  a.t = t.ptrs(); a.n_entries = t.n_entries;
  a.key_in = t.key[t.cur_key].p; a.key_out = t.key[t.cur_key ^ 1].p;
  a.cloud = e->d_frames.p + size_t(frame_slot) * ctvio_engine::kFrameCap;
  a.n_features = e->h_frame_n[frame_slot];
  a.slot = frame_slot; a.out = t.result.p;
  e->launches += ctvio::launch_feature_table_add(a, st);
  int32_t r[2];
  if (const int rc = read_result(e, r, t.result.p, 2)) return rc;
  t.cur_key ^= 1;
  t.n_entries += r[1];
  t.held |= 1u << frame_slot;
  t.window_current = false;
  if (n_tracked) *n_tracked = r[0];
  if (n_new) *n_new = r[1];
  return CTVIO_OK;
}

int ctvio_feature_table_window(ctvio_handle e, int32_t n_frames, const int32_t* frame_slots, int32_t window_size,
                               int32_t* n_landmarks) {
  if (!e) return fail(CTVIO_ERR_INVALID, "null handle");
  if (!frame_slots) return fail(CTVIO_ERR_INVALID, "null argument");
  if (n_frames < 1 || n_frames > ctvio_engine::kFrameSlots) return fail(CTVIO_ERR_INVALID, "n_frames must be 1..16");
  if (window_size < 3) return fail(CTVIO_ERR_INVALID, "window_size must be >= 3");
  ctvio::FeatureTableWindowArgs a;
  if (const int rc = parse_window_slots(n_frames, frame_slots, a.w)) return rc;
  auto& t = e->ft;
  if (a.w.listed != t.held) return fail(CTVIO_ERR_STATE, "the listed frame slots are not the slots the feature table holds");
  if (const int rc = check_numbering(e, TableWindow::kNumbered)) return rc;
  cudaSetDevice(e->cfg.device);
  if (const int rc = ensure_feature_table(e)) return rc;
  cudaStream_t st = e->stream;
  const int other = e->cur ^ 1;
  const size_t cap = ctvio::kFeatureTableMaxEntries;
  CUDA_OK(e->x[other].rho.reserve(cap + 1));  // only the other buffer: reserve() does not keep the contents
  a.t = t.ptrs(); a.n_entries = t.n_entries; a.window_size = window_size;
  a.rho_in = e->x[e->cur].rho.p; a.n_rho_in = std::max(t.n_lm, 0);
  a.rho_out = e->x[other].rho.p;  // the re-laid-out depths go into the other state buffer, then the pointers swap
  a.obs_offset = t.obs_offset.p; a.obs_slot = t.obs_slot.p; a.obs_idx = t.obs_idx.p;
  a.lm_id = t.lm_id.p; a.lm_anchor = t.lm_anchor.p; a.lm_used = t.lm_used.p; a.out = t.result.p;
  e->h2d_bytes += size_t(n_frames) * sizeof(int32_t);  // the slot list goes up with the launch
  e->launches += ctvio::launch_feature_table_window(a, st);
  int32_t r[2];
  if (const int rc = read_result(e, r, t.result.p, 2)) return rc;
  swap_rho(e);
  if (r[0] != e->nL) e->structure_dirty = true;
  e->nL = r[0];
  e->have_rho = true;
  e->mirror_valid = false;
  t.n_lm = r[0];
  t.n_obs = r[1];
  t.oldest_slot = a.w.slot[0];
  t.window_current = true;
  if (n_landmarks) *n_landmarks = r[0];
  return CTVIO_OK;
}

int ctvio_add_image_features_from_table(ctvio_handle e, int32_t marg_oldest, int32_t* n_factors) {
  if (!e) return fail(CTVIO_ERR_INVALID, "null handle");
  if (const int rc = check_numbering(e, TableWindow::kCurrentNumbered)) return rc;
  if (!e->img.empty() && e->img_desc.empty()) return fail(CTVIO_ERR_STATE, "image factors with host payload are already present");
  cudaSetDevice(e->cfg.device);
  cudaStream_t st = e->stream;
  auto& t = e->ft;
  const int n = t.n_obs - t.n_lm;
  if (n_factors) *n_factors = n;
  if (n > 0) {
    ctvio::FeatureTableFactorArgs a;
    a.n_landmarks = t.n_lm; a.obs_offset = t.obs_offset.p; a.obs_slot = t.obs_slot.p; a.obs_idx = t.obs_idx.p;
    a.rho = e->x[e->cur].rho.p; a.oldest_slot = t.oldest_slot; a.marg_oldest = marg_oldest ? 1 : 0;
    a.frame_cap = ctvio_engine::kFrameCap;
    // the descriptors are appended to the factor set's device-side list and never come back: the structure build
    // runs on the device (structure.cu).  Slot-named factors added before go up first, so that the list keeps the
    // caller order.
    if (!e->img_desc.empty()) {
      ArenaScope arena(e);
      if (const int rc = append_device_descriptors(e, e->img_desc)) return rc;
      e->img.clear();
      e->img_desc.clear();
    }
    const size_t base = size_t(e->n_img_dev);
    if (const int rc = reserve_device_descriptors(e, base + size_t(n))) return rc;
    a.out = e->d_img_in.p + base;
    e->launches += ctvio::launch_feature_table_factors(a, st);
    e->n_img_dev += n;
  }
  e->structure_dirty = true;
  return CTVIO_OK;
}

int ctvio_feature_table_slide(ctvio_handle e, int32_t frame_slot, int32_t* n_removed) {
  if (!e) return fail(CTVIO_ERR_INVALID, "null handle");
  if (frame_slot < 0 || frame_slot >= ctvio_engine::kFrameSlots) return fail(CTVIO_ERR_INVALID, "frame slot out of range");
  auto& t = e->ft;
  if (!(t.held >> frame_slot & 1u)) return fail(CTVIO_ERR_STATE, "the feature table does not hold the slot");
  if (const int rc = check_numbering(e, TableWindow::kNumbered)) return rc;
  cudaSetDevice(e->cfg.device);
  cudaStream_t st = e->stream;
  ctvio::FeatureTableSlideArgs a;
  a.t = t.ptrs(); a.n_entries = t.n_entries;
  a.key_in = t.key[t.cur_key].p; a.key_out = t.key[t.cur_key ^ 1].p; a.new_index = t.new_index.p;
  a.slot = frame_slot; a.rho = e->x[e->cur].rho.p; a.n_rho = std::max(t.n_lm, 0); a.out = t.result.p;
  e->launches += ctvio::launch_feature_table_slide(a, st);
  int32_t r;
  if (const int rc = read_result(e, &r, t.result.p)) return rc;
  t.cur_key ^= 1;
  t.n_entries -= r;
  t.held &= ~(1u << frame_slot);
  t.window_current = false;
  e->h_frame_ingested &= ~(1u << frame_slot);
  if (n_removed) *n_removed = r;
  return CTVIO_OK;
}

int ctvio_feature_table_slide_reanchor(ctvio_handle e, int32_t n_frames, const int32_t* frame_slots, int32_t marg_old,
                                       double init_depth, int32_t* n_removed, int32_t* n_reanchored) {
  if (!e) return fail(CTVIO_ERR_INVALID, "null handle");
  if (!frame_slots) return fail(CTVIO_ERR_INVALID, "null argument");
  if (n_frames < 2 || n_frames > ctvio_engine::kFrameSlots) return fail(CTVIO_ERR_INVALID, "n_frames must be 2..16");
  if (!(init_depth > 0.0) || !std::isfinite(init_depth)) return fail(CTVIO_ERR_INVALID, "init_depth must be positive");
  ctvio::FeatureTableSlideArgs a;
  if (const int rc = parse_window_slots(n_frames, frame_slots, a.w)) return rc;
  auto& t = e->ft;
  if (a.w.listed != t.held) return fail(CTVIO_ERR_STATE, "the listed frame slots are not the slots the feature table holds");
  if (const int rc = check_numbering(e, TableWindow::kNumbered)) return rc;
  a.marg_old = marg_old ? 1 : 0;
  if (a.marg_old) {
    // removeBackShiftDepth's poses: the cameras at the leaving frame's and the next frame's time
    if (!e->have_knots) return fail(CTVIO_ERR_STATE, "knots have not been set");
    for (int k = 0; k < 2; ++k) {
      int32_t s;
      double u;
      if (!spline_index(e->sp, e->h_frame_t[a.w.slot[k]], s, u))
        return fail(CTVIO_ERR_TIME_RANGE, "a frame time of the depth shift falls outside the spline");
    }
  }
  const int frame_slot = a.w.slot[a.marg_old ? 0 : n_frames - 2];
  cudaSetDevice(e->cfg.device);
  cudaStream_t st = e->stream;
  if (a.marg_old) ensure_table(e);
  a.t = t.ptrs(); a.n_entries = t.n_entries;
  a.key_in = t.key[t.cur_key].p; a.key_out = t.key[t.cur_key ^ 1].p; a.new_index = t.new_index.p;
  a.slot = frame_slot; a.rho = e->x[e->cur].rho.p; a.n_rho = std::max(t.n_lm, 0); a.out = t.result.p;
  a.init_depth = init_depth;
  a.table = e->d_frames.p; a.frame_cap = ctvio_engine::kFrameCap; a.frame_t = e->d_frame_t.p;
  a.st = e->x[e->cur].ptrs(); a.sp = e->sp; a.R_CI = e->rig.R_CI; a.p_CI = e->rig.p_CI;
  // the slot list goes up with the launch parameters
  e->h2d_bytes += size_t(n_frames) * sizeof(int32_t);
  e->launches += ctvio::launch_feature_table_slide_reanchor(a, st);
  int32_t r[2];
  if (const int rc = read_result(e, r, t.result.p, 2)) return rc;
  t.cur_key ^= 1;
  t.n_entries -= r[0];
  t.held &= ~(1u << frame_slot);
  t.window_current = false;
  e->h_frame_ingested &= ~(1u << frame_slot);
  if (n_removed) *n_removed = r[0];
  if (n_reanchored) *n_reanchored = r[1];
  return CTVIO_OK;
}

int ctvio_feature_table_landmarks(ctvio_handle e, int32_t n_landmarks, int32_t* feature_id, int32_t* anchor_slot,
                                  int32_t* used_num) {
  if (!e) return fail(CTVIO_ERR_INVALID, "null handle");
  if (const int rc = check_numbering(e, TableWindow::kCurrent)) return rc;
  if (n_landmarks != e->ft.n_lm) return fail(CTVIO_ERR_INVALID, "n_landmarks differs from the window's landmark count");
  if (n_landmarks > 0 && (!feature_id || !anchor_slot || !used_num)) return fail(CTVIO_ERR_INVALID, "null argument");
  if (n_landmarks == 0) return CTVIO_OK;
  cudaSetDevice(e->cfg.device);
  cudaStream_t st = e->stream;
  const size_t bytes = size_t(n_landmarks) * sizeof(int32_t);
  CUDA_OK(cudaMemcpyAsync(feature_id, e->ft.lm_id.p, bytes, cudaMemcpyDeviceToHost, st));
  CUDA_OK(cudaMemcpyAsync(anchor_slot, e->ft.lm_anchor.p, bytes, cudaMemcpyDeviceToHost, st));
  CUDA_OK(cudaMemcpyAsync(used_num, e->ft.lm_used.p, bytes, cudaMemcpyDeviceToHost, st));
  e->d2h_bytes += 3 * bytes;
  CUDA_OK(stream_sync(st));
  return CTVIO_OK;
}

int ctvio_feature_table_map(ctvio_handle e, int32_t n_frames, const int32_t* frame_slots, int32_t window_size,
                            int32_t capacity, double* xyz_world, int32_t* feature_id, uint8_t* in_margin_cloud,
                            int32_t* n_points, double* cam_q_xyzw, double* cam_p_xyz) {
  return feature_table_map_body(e, n_frames, frame_slots, window_size, capacity, xyz_world, feature_id, in_margin_cloud,
                                n_points, cam_q_xyzw, cam_p_xyz, nullptr, 0, nullptr);
}

}  // extern "C"

namespace ctvio::host {

int feature_table_map_body(ctvio_engine* e, int32_t n_frames, const int32_t* frame_slots, int32_t window_size,
                           int32_t capacity, double* xyz_world, int32_t* feature_id, uint8_t* in_margin_cloud,
                           int32_t* n_points, double* cam_q_xyzw, double* cam_p_xyz, const double* lm_cov9, int32_t n_cov,
                           double* point_cov9) {
  if (!e) return fail(CTVIO_ERR_INVALID, "null handle");
  if (!frame_slots || !n_points) return fail(CTVIO_ERR_INVALID, "null argument");
  if (n_frames < 1 || n_frames > ctvio_engine::kFrameSlots) return fail(CTVIO_ERR_INVALID, "n_frames must be 1..16");
  if (window_size < 3) return fail(CTVIO_ERR_INVALID, "window_size must be >= 3");
  if (capacity < 0) return fail(CTVIO_ERR_INVALID, "capacity must be >= 0");
  if (capacity > 0 && (!xyz_world || !feature_id || !in_margin_cloud)) return fail(CTVIO_ERR_INVALID, "null point array");
  ctvio::FeatureTableMapArgs a;
  if (const int rc = parse_window_slots(n_frames, frame_slots, a.w)) return rc;
  auto& t = e->ft;
  if (!e->have_knots) return fail(CTVIO_ERR_STATE, "knots have not been set");
  if (a.w.listed != t.held) return fail(CTVIO_ERR_STATE, "the listed frame slots are not the slots the feature table holds");
  if (const int rc = check_numbering(e, TableWindow::kNumbered)) return rc;
  for (int k = 0; k < n_frames; ++k) {
    int32_t s;
    double u;
    if (!spline_index(e->sp, e->h_frame_t[a.w.slot[k]], s, u))
      return fail(CTVIO_ERR_TIME_RANGE, "a listed frame time falls outside the spline");
  }
  cudaSetDevice(e->cfg.device);
  if (!t.h_map_head) {
    void* p = nullptr;
    const size_t bytes = sizeof(ctvio::MapHeader) + size_t(ctvio::kFeatureTableMaxEntries) * sizeof(ctvio::MapPoint);
    if (cudaHostAlloc(&p, bytes, cudaHostAllocMapped) != cudaSuccess) {
      cudaGetLastError();
      return fail(CTVIO_ERR_CUDA, "could not allocate the mapped map buffer");
    }
    t.h_map_head = static_cast<ctvio::MapHeader*>(p);
    t.h_map_points = reinterpret_cast<ctvio::MapPoint*>(t.h_map_head + 1);
  }
  cudaStream_t st = e->stream;
  ensure_table(e);
  a.t = t.ptrs(); a.n_entries = t.n_entries; a.window_size = window_size;
  a.table = e->d_frames.p; a.frame_t = e->d_frame_t.p; a.frame_cap = ctvio_engine::kFrameCap;
  a.st = e->x[e->cur].ptrs(); a.sp = e->sp; a.R_CI = e->rig.R_CI; a.p_CI = e->rig.p_CI;
  a.rho = e->x[e->cur].rho.p; a.n_rho = std::max(t.n_lm, 0);
  a.head = t.h_map_head; a.points = t.h_map_points;
  a.lm_cov9 = lm_cov9; a.n_cov = n_cov; a.point_cov9 = point_cov9;
  // the slot list goes with the launch parameters; the kernel writes the result straight into mapped host memory
  e->launches += point_cov9 ? ctvio::launch_feature_table_map_cov(a, st) : ctvio::launch_feature_table_map(a, st);
  CUDA_OK(stream_sync(st));
  const ctvio::MapHeader& h = *t.h_map_head;
  const int n = h.n_points;
  e->d2h_bytes += 8 + 56 * size_t(n_frames) + sizeof(ctvio::MapPoint) * size_t(n);
  if (point_cov9) e->d2h_bytes += 9 * sizeof(double) * size_t(n);
  *n_points = n;
  if (n > capacity) return fail(CTVIO_ERR_INVALID, "capacity is smaller than the number of map points");
  for (int k = 0; k < n; ++k) {
    const ctvio::MapPoint& p = t.h_map_points[k];
    xyz_world[3 * k] = p.xyz[0]; xyz_world[3 * k + 1] = p.xyz[1]; xyz_world[3 * k + 2] = p.xyz[2];
    feature_id[k] = p.id;
    in_margin_cloud[k] = uint8_t(p.in_margin_cloud);
  }
  for (int k = 0; k < n_frames; ++k) {
    if (cam_q_xyzw) for (int c = 0; c < 4; ++c) cam_q_xyzw[4 * k + c] = h.cam[k][c];
    if (cam_p_xyz) for (int c = 0; c < 3; ++c) cam_p_xyz[3 * k + c] = h.cam[k][4 + c];
  }
  return CTVIO_OK;
}

}  // namespace ctvio::host

extern "C" {

int ctvio_check_keyframe(ctvio_handle e, int32_t n_frames, const int32_t* frame_slots, double min_parallax,
                         int32_t* is_keyframe, int32_t* n_tracked, int32_t* parallax_num, double* parallax_sum) {
  if (!e) return fail(CTVIO_ERR_INVALID, "null handle");
  if (!frame_slots || !is_keyframe) return fail(CTVIO_ERR_INVALID, "null argument");
  if (n_frames < 1 || n_frames > ctvio_engine::kFrameSlots) return fail(CTVIO_ERR_INVALID, "n_frames must be 1..16");
  if (!(min_parallax >= 0.0) || !std::isfinite(min_parallax)) return fail(CTVIO_ERR_INVALID, "min_parallax must be finite and >= 0");
  ctvio::KeyframeArgs a;
  if (const int rc = parse_window_slots(n_frames, frame_slots, a.w)) return rc;
  for (int k = 0; k < n_frames; ++k) a.count[k] = e->h_frame_n[a.w.slot[k]];  // 0 for a slot that never received a cloud
  cudaSetDevice(e->cfg.device);
  cudaStream_t st = e->stream;
  CUDA_OK(e->d_frames.reserve(size_t(ctvio_engine::kFrameSlots) * ctvio_engine::kFrameCap));
  CUDA_OK(e->d_kf_result.reserve(1));
  a.table = e->d_frames.p; a.frame_cap = ctvio_engine::kFrameCap;
  a.min_parallax = min_parallax; a.out = e->d_kf_result.p;
  // the slot list goes up with the launch; ids and bearings are resident
  e->h2d_bytes += size_t(n_frames) * sizeof(int32_t);
  e->launches += ctvio::launch_keyframe_parallax(a, st);
  ctvio::KeyframeResult r;
  if (const int rc = read_result(e, &r, e->d_kf_result.p)) return rc;
  *is_keyframe = r.is_keyframe;
  if (n_tracked) *n_tracked = r.n_tracked;
  if (parallax_num) *parallax_num = r.parallax_num;
  if (parallax_sum) *parallax_sum = r.parallax_sum;
  return CTVIO_OK;
}

int ctvio_slide_window_second_new(ctvio_handle e) {
  if (!e) return fail(CTVIO_ERR_INVALID, "null handle");
  if (e->nB < 2) return fail(CTVIO_ERR_STATE, "the window has fewer than 2 bias nodes");
  const int gone = e->nB - 2;
  // the prior is kept as it is (trajectory_manager.cpp:270-280), so none of its blocks may belong to the leaving node
  for (size_t b = 0; b < e->prior.type.size(); ++b)
    if (ctvio::block_is_bias(e->prior.type[b]) && e->prior.index[b] == gone)
      return fail(CTVIO_ERR_STATE, "the active prior holds a block of the second-newest bias node");
  cudaSetDevice(e->cfg.device);
  // Bgs_/Bas_[WINDOW_SIZE - 1] = [WINDOW_SIZE] (visual_odometry.cpp:253-278); node nB-1 keeps its value and stands for the
  // next image, as the node ctvio_slide_window appends does.  Knots, time origin and prior block indices do not move.
  double* bias = e->x[e->cur].bias.p;
  CUDA_OK(cudaMemcpyAsync(bias + 6 * size_t(gone), bias + 6 * size_t(gone + 1), 6 * sizeof(double), cudaMemcpyDeviceToDevice,
                          e->stream));
  e->mirror_valid = false;
  return CTVIO_OK;
}

// ---- wire-format ingestion (SURVEY 8f-4) ----------------------------------------------------------
int ctvio_ingest_feature_cloud(ctvio_handle e, int32_t slot, int64_t t_ns, int32_t n, const float* points, const float* ch_id,
                               const float* ch_u, const float* ch_v, const float* ch_vx, const float* ch_vy) {
  (void)ch_u; (void)ch_vx; (void)ch_vy;  // carried by the message, not used by the estimator's factors
  if (!e || slot < 0 || slot >= ctvio_engine::kFrameSlots || n < 0 || n > ctvio_engine::kFrameCap ||
      (n > 0 && (!points || !ch_id || !ch_v)))
    return fail(CTVIO_ERR_INVALID, "bad feature cloud");
  // the feature table's indices point into the slot's cloud until ctvio_feature_table_slide frees it
  if (e->ft.held >> slot & 1u) return fail(CTVIO_ERR_STATE, "the feature table holds the slot");
  cudaSetDevice(e->cfg.device);
  return ingest_feature_cloud_body(e, slot, t_ns, n, points, ch_id, ch_v, true);  // the caller's message buffers may go away
}

int ctvio_add_image_features_from_slots(ctvio_handle e, int32_t n, const int32_t* slot_i, const int32_t* idx_i,
                                        const int32_t* slot_j, const int32_t* idx_j, const int32_t* lm, const int32_t* marg) {
  if (!e || n < 0 || (n > 0 && (!slot_i || !idx_i || !slot_j || !idx_j || !lm))) return fail(CTVIO_ERR_INVALID, "null argument");
  if (!e->img.empty() && e->img_desc.empty()) return fail(CTVIO_ERR_STATE, "image factors with host payload are already present");
  // the factors before the first bad one are added, as the call always did
  std::vector<ctvio::FactorDesc> desc;
  int rc = CTVIO_OK;
  for (int k = 0; k < n; ++k) {
    const int si = slot_i[k], sj = slot_j[k];
    if (si < 0 || si >= ctvio_engine::kFrameSlots || sj < 0 || sj >= ctvio_engine::kFrameSlots || idx_i[k] < 0 ||
        idx_i[k] >= e->h_frame_n[si] || idx_j[k] < 0 || idx_j[k] >= e->h_frame_n[sj]) {
      rc = fail(CTVIO_ERR_INVALID, "feature slot / index out of range");
      break;
    }
    desc.push_back(ctvio::FactorDesc{si * ctvio_engine::kFrameCap + idx_i[k], sj * ctvio_engine::kFrameCap + idx_j[k], lm[k],
                                     marg ? marg[k] : 0});
  }
  if (e->n_img_dev > 0) {
    // the set already holds table-built factors: these join them on the device, in caller order
    cudaSetDevice(e->cfg.device);
    ArenaScope arena(e);
    if (const int rc2 = append_device_descriptors(e, desc)) return rc2;
  } else {
    for (const ctvio::FactorDesc& d : desc)
      e->img.push_back(HostImage{e->h_frame_t[d.slot_i / ctvio_engine::kFrameCap], e->h_frame_t[d.slot_j / ctvio_engine::kFrameCap],
                                 0, 0, {0, 0}, {0, 0}, d.lm, d.marg});
    e->img_desc.insert(e->img_desc.end(), desc.begin(), desc.end());
  }
  e->structure_dirty = true;
  return rc;
}

int ctvio_ingest_imu(ctvio_handle e, int32_t n, const void* records, int32_t stride, int32_t off_gyro, int32_t off_accel,
                     int64_t drop_before_ns) {
  if (!e || n < 0 || (n > 0 && !records) || stride < 56 || off_gyro < 8 || off_accel < 8 || off_gyro + 24 > stride ||
      off_accel + 24 > stride)
    return fail(CTVIO_ERR_INVALID, "bad IMU record layout");
  cudaSetDevice(e->cfg.device);
  return ingest_imu_body(e, n, records, stride, off_gyro, off_accel, drop_before_ns, true, nullptr);
}

int ctvio_add_imu_from_table(ctvio_handle e, int64_t t_min, int64_t t_max, int32_t n_kf, const int64_t* kf_t, int32_t fixed_node,
                             int64_t marg_before_ns, int32_t* n_added) {
  if (!e || (fixed_node < 0 && (n_kf <= 0 || !kf_t))) return fail(CTVIO_ERR_INVALID, "bad argument");
  if (!e->imu.empty() && e->imu_src.empty()) return fail(CTVIO_ERR_STATE, "IMU factors with host payload are already present");
  int added = 0;
  for (size_t k = 0; k < e->h_imu_tab_t.size(); ++k) {
    const int64_t t = e->h_imu_tab_t[k];
    if (t < t_min) continue;      // trajectory_manager.cpp:391-394
    if (t >= t_max) break;
    int node = fixed_node;
    if (node < 0) {               // bias index of the sample (:396-412)
      if (t < kf_t[0]) node = 0;
      else if (t >= kf_t[n_kf - 1]) node = n_kf - 1;
      else
        for (int i = 1; i < n_kf; ++i)
          if (t >= kf_t[i - 1] && t < kf_t[i]) { node = i - 1; break; }
    }
    HostImu o{t, {0, 0, 0}, {0, 0, 0}, node, t < marg_before_ns ? 1 : 0};
    e->imu.push_back(o);
    e->imu_src.push_back(int32_t(k));
    ++added;
  }
  if (n_added) *n_added = added;
  e->structure_dirty = true;
  return CTVIO_OK;
}

}  // extern "C"
