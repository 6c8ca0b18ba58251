// Front-end data formats either side of the hot path (SURVEY §8f-3, f-4).
//
//   triangulate_kernel   replaces FeatureManager::triangulate (visual_odometry/feature_manager.cpp:173-223 and the
//                        camera-extrinsic overload :230-275): per-landmark DLT, depth = V(2)/V(3) of the right singular
//                        vector of the smallest singular value of the 2m x 4 system, INIT_DEPTH fallback below 0.1.
//   triangulate_window_kernel  the same DLT for the landmarks of the resident window (AddImageToWindow,
//                        visual_odometry.cpp:185-191), camera poses from the resident spline at each observation's row
//                        time (the rolling-shutter variant triangulateRS, feature_manager.cpp:276-338, when ld > 0).
//   keyframe_parallax_kernel  replaces FeatureManager::addFeatureCheckParallax (feature_manager.cpp:28-87) as
//                        VisualOdometry::AddImageToWindow uses it (visual_odometry.cpp:180-183), on the resident frame
//                        slots: tracked count of the new image and mean parallax between the two frames before it.
//   feature_table_*_kernel  the feature list of FeatureManager (feature_manager.cpp:28-59 insertion, :111-147
//                        getDepthVector / setDepth, :148-158 removeFailures, :341-423 the slide, dropping or re-anchoring
//                        the leaving frame's landmarks) as a resident table keyed
//                        by the tracker's feature id, and the image-factor loops of trajectory_manager.cpp:206-236, :359-385.
//                        feature_table_map_kernel publishes its landmark map (GetLandmarksInWindow / GetMarginCloud,
//                        visual_odometry.cpp:310-372) and the keyframe camera poses (PublishVioKeyFrame).
//   unpack_cloud_kernel  replaces FeatureMsg2Image (visual_odometry/visual_struct.h:98-121) on the tracker's message
//                        (visual_feature/feature_tracker_node.cpp:146-184): sensor_msgs::PointCloud arrives as packed
//                        float32 triples + five float32 channels and is converted ON THE DEVICE into the resident
//                        per-frame feature table (id, bearing xy, pixel row).
//   unpack_imu_kernel    IMUData (utils/parameter_struct.h:58-65) records -> {t, gyro, accel} table.
//   gather_factors_kernel builds the sorted SoA image-factor arrays of K1 from the resident tables and an 8-byte
//                        (slot_i, slot_j) descriptor per factor: the payload never passes through host marshalling.
//
// The DLT itself (streaming Givens QR + 4x4 one-sided Jacobi SVD, one thread per landmark) is in dlt.cuh.
#include "frontend.h"

#include <algorithm>

#include "dlt.cuh"

namespace ctvio {

namespace {

__global__ void triangulate_kernel(TriangulateArgs a) {
  const int l = blockIdx.x * blockDim.x + threadIdx.x;
  if (l >= a.n_landmarks) return;
  const int o0 = a.obs_offset[l], used = a.obs_offset[l + 1] - o0;
  const int start = a.start_frame[l];
  // feature_manager.cpp:236-240: candidates only, already-initialised depths are kept
  if (!(used >= 2 && start < a.window_size - 2)) return;
  if (a.depth[l] > 0.0) return;
  if (start < 0 || start + used > a.n_frames) { a.depth[l] = a.init_depth; return; }
  auto cam_pose = [&](int f, M3& Rc, V3& tc) {
    M3 Rf;
#pragma unroll
    for (int e = 0; e < 9; ++e) Rf.m[e] = a.Rs[9 * f + e];
    const V3 Pf{a.Ps[3 * f], a.Ps[3 * f + 1], a.Ps[3 * f + 2]};
    Rc = m3_mul(Rf, a.ric);          // R0 = Rs[i] * ric        (:246)
    tc = Pf + m3_vec(Rf, a.tic);     // t0 = Ps[i] + Rs[i] tic  (:245)
  };
  M3 R0;
  V3 t0;
  cam_pose(start, R0, t0);
  R4 Rq;
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) Rq.r[i][j] = 0.0;
  for (int k = 0; k < used; ++k) {
    M3 R1;
    V3 t1;
    cam_pose(start + k, R1, t1);
    const V3 f{a.obs_point[3 * (o0 + k)], a.obs_point[3 * (o0 + k) + 1], a.obs_point[3 * (o0 + k) + 2]};
    dlt_push_observation(Rq, R0, t0, R1, t1, f);
  }
  double v[4];
  smallest_right_singular_vector(Rq, v);
  double d = v[2] / v[3];
  if (!(d >= 0.1)) d = a.init_depth;  // :268-271 (NaN / inf from v[3] == 0 also fall back)
  if (!isfinite(d)) d = a.init_depth;
  a.depth[l] = d;
}

// ---- DLT of the resident window (triangulate at the row time, feature_manager.cpp:226-274 / :276-338) ----------------
// One CTA per kTriLmPerCta consecutive landmarks.  Their observations are processed in chunks of kTriObsChunk: every
// thread evaluates observation poses (the ~11 spline evaluations per landmark are the bulk of the work) into shared
// memory, then the thread of each landmark folds the rows of its observations in that chunk into its R (registers,
// kept across chunks, so a landmark may have any number of observations).  Rows enter in observation order, the SVD
// runs once per landmark: no atomics on the result, bitwise reproducible.
constexpr int kTriThreads = 128;
constexpr int kTriLmPerCta = 32;
constexpr int kTriObsChunk = 256;
constexpr int kTriPoseWords = 14;  // camera R (9) | camera t (3) | bearing x, y

__global__ void __launch_bounds__(kTriThreads) triangulate_window_kernel(TriangulateWindowArgs a) {
  __shared__ double s_pose[kTriObsChunk][kTriPoseWords];
  __shared__ int32_t s_off[kTriLmPerCta + 1];
  __shared__ uint8_t s_todo[kTriLmPerCta];
  const int tid = threadIdx.x;
  const int l0 = blockIdx.x * kTriLmPerCta;
  const int nl = min(kTriLmPerCta, a.n_landmarks - l0);
  const int l = l0 + tid;
  const bool owner = tid < nl;
  const double rho_old = owner ? a.rho_in[l] : 0.0;
  // feature_manager.cpp:239-240: an initialised depth (> 0) is kept; NaN is not > 0 and is re-triangulated
  const bool want = owner && !(rho_old > 0.0);
  if (tid <= nl) s_off[tid] = a.obs_offset[l0 + tid];
  if (owner) s_todo[tid] = want && a.obs_offset[l + 1] - a.obs_offset[l] >= 2;
  __syncthreads();
  const int o_begin = s_off[0], o_end = s_off[nl];
  const int lo = owner ? s_off[tid] : 0, hi = owner ? s_off[tid + 1] : 0;
  const bool dlt = owner && s_todo[tid];
  const int64_t ld_ns = int64_t(*a.st.ld * 1e9);  // image_feature_factor.h:72 (truncation), as K1
  bool out_of_range = false;
  R4 Rq = {};
  M3 R0{};
  V3 t0{0.0, 0.0, 0.0};
  for (int c0 = o_begin; c0 < o_end; c0 += kTriObsChunk) {
    const int c1 = min(c0 + kTriObsChunk, o_end);
    for (int k = c0 + tid; k < c1; k += kTriThreads) {
      const int slot = a.obs_slot[k];
      const FrameFeature f = a.table[size_t(slot) * a.frame_cap + a.obs_idx[k]];
      int32_t s;
      double u;
      // every observation's time is checked; poses are evaluated only for the landmarks that are triangulated
      if (!spline_index(a.sp, a.frame_t[slot] + int64_t(f.row) * ld_ns, s, u)) { out_of_range = true; continue; }
      int j = 0;  // landmark of observation k: last j with s_off[j] <= k
      for (int step = kTriLmPerCta / 2; step > 0; step >>= 1)
        if (j + step < nl && s_off[j + step] <= k) j += step;
      if (!s_todo[j]) continue;
      SideEval ev;
      eval_side<false, kPStride>(a.sp, a.st.q, a.st.p, a.st.tab, s, u, ev);
      const M3 Rc = m3_mul(ev.R, a.R_CI);        // R_c = R * R_CI         (:246)
      const V3 tc = ev.p + m3_vec(ev.R, a.p_CI);  // t_c = p + R * p_CI     (:245)
      double* w = s_pose[k - c0];
#pragma unroll
      for (int e = 0; e < 9; ++e) w[e] = Rc.m[e];
      w[9] = tc.x; w[10] = tc.y; w[11] = tc.z;
      w[12] = f.x; w[13] = f.y;
    }
    __syncthreads();
    if (dlt) {
      const int k1 = min(hi, c1);
      for (int k = max(lo, c0); k < k1; ++k) {
        const double* w = s_pose[k - c0];
        M3 R1;
#pragma unroll
        for (int e = 0; e < 9; ++e) R1.m[e] = w[e];
        const V3 t1{w[9], w[10], w[11]};
        if (k == lo) { R0 = R1; t0 = t1; }  // the anchor
        dlt_push_observation(Rq, R0, t0, R1, t1, V3{w[12], w[13], 1.0});
      }
    }
    __syncthreads();
  }
  bool triangulated = false;
  if (want) {
    double d = a.init_depth;  // fewer than 2 observations: INIT_DEPTH
    if (dlt) {
      double v[4];
      smallest_right_singular_vector(Rq, v);
      const double dd = v[2] / v[3];
      if (dd >= 0.1 && isfinite(dd)) { d = dd; triangulated = true; }  // :266-271 (NaN / inf fall back as well)
    }
    a.rho_out[l] = 1.0 / d;
  } else if (owner) {
    a.rho_out[l] = rho_old;
  }
  const int n_tri = __syncthreads_count(triangulated);
  const int n_fb = __syncthreads_count(want && !triangulated);
  const int bad = __syncthreads_or(out_of_range);
  if (tid == 0) {
    if (n_tri) atomicAdd(&a.counts[0], n_tri);
    if (n_fb) atomicAdd(&a.counts[1], n_fb);
    if (bad) atomicOr(&a.counts[0], int(0x80000000u));
  }
}

// ---- keyframe decision (addFeatureCheckParallax + compensatedParallax2, feature_manager.cpp:28-87 / :424-456) ------------
// One CTA, one thread per feature index.  The (id, index) keys of the new slot and of slot fc-2 are sorted in shared
// memory (bitonic, both arrays at once); the features of the other listed slots binary-search the new slot's keys and
// mark the hits (an idempotent store), the features of slot fc-1 search slot fc-2's keys and store their parallax at
// their own index.  The counts come from __syncthreads_count, the parallax sum from a fixed tree over the feature
// indices: no atomics, bitwise reproducible.
constexpr int kKfThreads = kKeyframeMaxFeatures;

// sort key of (id, index): the signed id ordered as unsigned in the high word, the index in the low word
__device__ __forceinline__ uint64_t kf_key(int32_t id, int i) {
  return (uint64_t(uint32_t(id) ^ 0x80000000u) << 32) | uint32_t(i);
}
// index (in its slot) of the feature with this id among the n sorted keys, or -1
__device__ __forceinline__ int kf_find(const uint64_t* keys, int n, int32_t id) {
  const uint64_t lo = kf_key(id, 0);
  int a = 0, b = n;  // first key >= lo
  while (a < b) {
    const int m = (a + b) >> 1;
    if (keys[m] < lo) a = m + 1; else b = m;
  }
  return (a < n && (keys[a] >> 32) == (lo >> 32)) ? int(uint32_t(keys[a])) : -1;
}
// number of the n sorted keys whose id is smaller than the id of x
__device__ __forceinline__ int kf_rank(const uint64_t* keys, int n, uint64_t x) {
  const uint64_t lo = x & 0xffffffff00000000ull;
  int a = 0, b = n;
  while (a < b) {
    const int m = (a + b) >> 1;
    if (keys[m] < lo) a = m + 1; else b = m;
  }
  return a;
}
// ascending bitonic sort of N keys in shared memory.  Every thread of the block calls it (it synchronises the block after
// each pass); the threads with `active` set each work on compare pair p, 0 <= p < N/2.
template <int N>
__device__ __forceinline__ void bitonic_sort_shared(uint64_t* keys, int p, bool active) {
  for (int k = 2; k <= N; k <<= 1)
    for (int j = k >> 1; j > 0; j >>= 1) {
      if (active) {
        const int i = 2 * j * (p / j) + p % j;
        const uint64_t x = keys[i], y = keys[i + j];
        if ((x > y) == ((i & k) == 0)) { keys[i] = y; keys[i + j] = x; }
      }
      __syncthreads();
    }
}

__global__ void __launch_bounds__(kKfThreads) keyframe_parallax_kernel(KeyframeArgs a) {
  __shared__ uint64_t s_key[2][kKeyframeMaxFeatures];  // [0]: the new slot, [1]: slot fc-2
  __shared__ double s_par[kKeyframeMaxFeatures];       // parallax of feature i of slot fc-1 (0: not a parallax feature)
  __shared__ uint8_t s_tracked[kKeyframeMaxFeatures];  // feature i of the new slot occurs in another listed slot
  const int tid = threadIdx.x;
  const int fc = a.w.n_frames - 1;  // frame_count
  const int n_new = a.count[fc];
  const int n_old = fc >= 2 ? a.count[fc - 2] : 0;
  const FrameFeature* t_new = a.table + size_t(a.w.slot[fc]) * a.frame_cap;
  const FrameFeature* t_old = fc >= 2 ? a.table + size_t(a.w.slot[fc - 2]) * a.frame_cap : nullptr;
  s_key[0][tid] = tid < n_new ? kf_key(t_new[tid].id, tid) : ~0ull;
  s_key[1][tid] = tid < n_old ? kf_key(t_old[tid].id, tid) : ~0ull;
  s_par[tid] = 0.0;
  s_tracked[tid] = 0;
  __syncthreads();
  // bitonic sort of both key arrays: threads [0, N/2) work on s_key[0], [N/2, N) on s_key[1]
  constexpr int N = kKeyframeMaxFeatures;
  bitonic_sort_shared<N>(s_key[tid / (N / 2)], tid % (N / 2), true);
  // last_track_num (:38-57): the new image's features whose id is already in the window
  for (int f = 0; f < fc; ++f) {
    const FrameFeature* t = a.table + size_t(a.w.slot[f]) * a.frame_cap;
    for (int i = tid; i < a.count[f]; i += kKfThreads) {
      const int hit = kf_find(s_key[0], n_new, t[i].id);
      if (hit >= 0) s_tracked[hit] = 1;
    }
  }
  // parallax features (:62-72): start_frame <= fc-2 && endFrame() >= fc-1, i.e. seen in slots fc-2 and fc-1
  bool parallax_feature = false;
  if (fc >= 2 && tid < a.count[fc - 1]) {
    const FrameFeature fj = a.table[size_t(a.w.slot[fc - 1]) * a.frame_cap + tid];
    const int i = kf_find(s_key[1], n_old, fj.id);
    if (i >= 0) {
      // compensatedParallax2 (:424-456) with z == 1: the compensated and the plain distance coincide.  The products are
      // rounded separately (no FMA) so that every per-feature value is the one a host restatement computes.
      const FrameFeature fi = t_old[i];
      const double du = fi.x - fj.x, dv = fi.y - fj.y;
      s_par[tid] = sqrt(__dadd_rn(__dmul_rn(du, du), __dmul_rn(dv, dv)));
      parallax_feature = true;
    }
  }
  __syncthreads();
  const int n_tracked = __syncthreads_count(tid < n_new && s_tracked[tid]);
  const int parallax_num = __syncthreads_count(parallax_feature);
  for (int stride = kKfThreads / 2; stride > 0; stride >>= 1) {
    if (tid < stride) s_par[tid] += s_par[tid + stride];
    __syncthreads();
  }
  if (tid == 0) {
    const double sum = s_par[0];
    KeyframeResult r;
    r.n_tracked = n_tracked;
    r.parallax_num = parallax_num;
    r.parallax_sum = sum;
    r.pad = 0;
    // :59-60 and :74-86
    if (fc < 2 || n_tracked < 20 || parallax_num == 0) r.is_keyframe = 1;
    else r.is_keyframe = sum / parallax_num >= a.min_parallax;
    *a.out = r;
  }
}

// ---- resident feature table (FeatureManager's feature list, feature_manager.cpp:28-59, :111-158, :341-423) --------------
// Add, Slide and Window run as one CTA of kFtThreads threads; the counts come from block scans and __syncthreads_count.
// Every entry and key is written by exactly one thread: no atomics, bitwise reproducible.
constexpr int kFtThreads = kKeyframeMaxFeatures;
static_assert(kFtThreads == 1024, "block_exclusive_scan covers 32 warps");

// exclusive prefix sum of v over the block (kFtThreads threads, in thread order); `total` receives the block sum.
// s: 32 ints of shared memory.  Synchronises the block (so every read issued before the call is complete on return).
__device__ __forceinline__ int block_exclusive_scan(int v, int* s, int& total) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  int x = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int y = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= o) x += y;
  }
  if (lane == 31) s[w] = x;
  __syncthreads();
  if (w == 0) {
    int t = s[lane];
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int y = __shfl_up_sync(0xffffffffu, t, o);
      if (lane >= o) t += y;
    }
    s[lane] = t;
  }
  __syncthreads();
  const int before = (w ? s[w - 1] : 0) + x - v;
  total = s[31];
  __syncthreads();
  return before;
}

// Add: the new slot's (id, index) keys are sorted; each binary-searches the live entries' sorted (id, entry) keys.  A hit
// becomes that entry's observation in the slot; the misses, ranked in ascending id order, are appended as new entries.
// The sorted key array is rebuilt by a rank merge into key_out (ids are distinct between the live entries and the misses).
__global__ void __launch_bounds__(kFtThreads) feature_table_add_kernel(FeatureTableAddArgs a) {
  __shared__ uint64_t s_key[kFtThreads];  // the new slot's keys, sorted
  __shared__ uint64_t s_new[kFtThreads];  // (id, new entry) of the misses, ascending id
  __shared__ int s_scan[32];
  const int tid = threadIdx.x;
  const int n_live = a.n_entries;
  const FeatureTablePtrs& t = a.t;
  s_key[tid] = tid < a.n_features ? kf_key(a.cloud[tid].id, tid) : ~0ull;
  __syncthreads();
  bitonic_sort_shared<kFtThreads>(s_key, tid, tid < kFtThreads / 2);
  const uint64_t k = s_key[tid];
  const bool valid = tid < a.n_features;
  const int32_t id = int32_t(uint32_t(k >> 32) ^ 0x80000000u);
  const int i = int(uint32_t(k));
  const int hit = valid ? kf_find(a.key_in, n_live, id) : -1;
  if (hit >= 0) {  // ids are unique within a cloud: one thread per entry
    t.idx[size_t(a.slot) * kFeatureTableMaxEntries + hit] = i;
    t.mask[hit] |= 1u << a.slot;
  }
  const bool miss = valid && hit < 0;
  int n_new;
  const int r = block_exclusive_scan(miss, s_scan, n_new);
  const int n_tracked = __syncthreads_count(hit >= 0);
  if (miss) {
    const int e = n_live + r;
    t.id[e] = id;
    t.anchor[e] = a.slot;
    t.mask[e] = 1u << a.slot;
    t.lm[e] = -1;
    t.rho[e] = -1.0;  // FeaturePerId: estimated_depth = -1
    t.idx[size_t(a.slot) * kFeatureTableMaxEntries + e] = i;
    s_new[r] = (k & 0xffffffff00000000ull) | uint32_t(e);
  }
  __syncthreads();
  for (int j = tid; j < n_live; j += kFtThreads) {
    const uint64_t x = a.key_in[j];
    a.key_out[j + kf_rank(s_new, n_new, x)] = x;
  }
  if (tid < n_new) a.key_out[tid + kf_rank(a.key_in, n_live, s_new[tid])] = s_new[tid];
  if (tid == 0) { a.out[0] = n_tracked; a.out[1] = n_new; }
}

// camera pose at time t (GetCameraPose, visual_odometry.cpp:197-202): the resident spline composed with the extrinsic,
// R_c = R R_CI, t_c = p + R p_CI (as triangulate_window_kernel).  t must lie inside the spline.
__device__ __forceinline__ void camera_pose_at(const StatePtrs& st, const SplineParams& sp, const M3& R_CI, const V3& p_CI,
                                               int64_t t, M3& Rc, V3& tc) {
  int32_t s;
  double u;
  spline_index(sp, t, s, u);
  SideEval ev;
  eval_side<false, kPStride>(sp, st.q, st.p, st.tab, s, u, ev);
  Rc = m3_mul(ev.R, R_CI);
  tc = ev.p + m3_vec(ev.R, p_CI);
}

// Slide: removeFailures (an entry numbered in the last window whose resident inverse depth is < 0), then the entries
// anchored in the leaving slot go and every other one drops its observation there.  A stable in-place compaction of the
// entries (a chunk is read completely before the scan's barrier, and lands at or below its own positions), then of the
// sorted key array into key_out with the entries' new indices (a stable filter of a sorted array stays sorted).
// kReanchor: an entry anchored in the leaving slot is re-anchored instead where the reference keeps it.  MARGIN_OLD
// (removeBackShiftDepth, feature_manager.cpp:341-378): with >= 2 observations left, its anchor becomes the earliest
// listed slot holding one and its depth is shifted from the camera at w.slot[0] into the camera at w.slot[1] (poses
// evaluated first into shared memory), INIT_DEPTH when the shifted depth is not > 0.  MARGIN_SECOND_NEW (removeFront,
// :398-423): with an observation in the newest slot, its anchor moves there and its depth is kept.  Either way the entry
// keeps its place and id (the key array stays a stable filter), stores its inverse depth, loses its number and carries
// solve_flag in kFeatureSolvedBit.
template <bool kReanchor>
__global__ void __launch_bounds__(kFtThreads) feature_table_slide_kernel(FeatureTableSlideArgs a) {
  __shared__ int s_scan[32];
  const int tid = threadIdx.x;
  const FeatureTablePtrs& t = a.t;
  const uint32_t bit = 1u << a.slot;
  constexpr size_t S = kFeatureTableMaxEntries;
  int kept = 0;
  [[maybe_unused]] int n_reanchored = 0;
  [[maybe_unused]] __shared__ double s_cam[2][12];  // kReanchor: camera R (9) | t (3) at w.slot[0], w.slot[1]
  if constexpr (kReanchor) {
    if (a.marg_old && tid < 2) {
      M3 Rc;
      V3 tc;
      camera_pose_at(a.st, a.sp, a.R_CI, a.p_CI, a.frame_t[a.w.slot[tid]], Rc, tc);
#pragma unroll
      for (int k = 0; k < 9; ++k) s_cam[tid][k] = Rc.m[k];
      s_cam[tid][9] = tc.x; s_cam[tid][10] = tc.y; s_cam[tid][11] = tc.z;
    }
    __syncthreads();
  }
  for (int c = 0; c < a.n_entries; c += kFtThreads) {
    const int e = c + tid;
    const bool in = e < a.n_entries;
    int32_t id = 0, anchor = 0, lm = -1, idx[kKeyframeMaxSlots];
    uint32_t mask = 0;
    double rho = 0.0;
    bool keep = false;
    [[maybe_unused]] bool reanchored = false;
    if (in) {
      id = t.id[e]; anchor = t.anchor[e]; lm = t.lm[e]; mask = t.mask[e]; rho = t.rho[e];
#pragma unroll
      for (int s = 0; s < kKeyframeMaxSlots; ++s) idx[s] = (mask >> s) & 1u ? t.idx[s * S + e] : -1;
      const bool failed = lm >= 0 && lm < a.n_rho && a.rho[lm] < 0.0;  // SolveFail (feature_manager.cpp:148-158)
      keep = !failed && anchor != a.slot;
      if constexpr (kReanchor) {
        if (!failed && anchor == a.slot) {
          const bool numbered = lm >= 0 && lm < a.n_rho;
          const double r_now = numbered ? a.rho[lm] : rho;  // setDepth's value, else the stored one
          const uint32_t rest = mask & ~bit & a.w.listed;
          if (a.marg_old) {
            if (__popc(rest) >= 2) {
              int k = 1;
              while (!((rest >> a.w.slot[k]) & 1u)) ++k;  // the earliest listed slot holding an observation
              const FrameFeature f = a.table[size_t(anchor) * a.frame_cap + t.idx[anchor * S + e]];
              const double depth = 1.0 / r_now;
              const double* c0 = s_cam[0];
              const double* c1 = s_cam[1];
              const V3 pc{f.x * depth, f.y * depth, depth};  // uv_i * estimated_depth
              double d[3];
#pragma unroll
              for (int r = 0; r < 3; ++r)  // w_pts_i - new_P
                d[r] = c0[3 * r] * pc.x + c0[3 * r + 1] * pc.y + c0[3 * r + 2] * pc.z + c0[9 + r] - c1[9 + r];
              const double z = c1[2] * d[0] + c1[5] * d[1] + c1[8] * d[2];  // (new_R^T (w_pts_i - new_P)).z
              rho = 1.0 / (z > 0.0 ? z : a.init_depth);  // dep_j > 0, else INIT_DEPTH (a NaN falls back as well)
              anchor = a.w.slot[k];
              reanchored = true;
            }
          } else if ((rest >> a.w.slot[a.w.n_frames - 1]) & 1u) {
            anchor = a.w.slot[a.w.n_frames - 1];
            rho = r_now;
            reanchored = true;
          }
          if (reanchored) {
            if (numbered) mask |= kFeatureSolvedBit;  // setDepth set SovelSucc (SolveFail has left above)
            lm = -1;
            keep = true;
          }
        }
      }
    }
    if constexpr (kReanchor) n_reanchored += __syncthreads_count(reanchored);
    int total;
    const int r = block_exclusive_scan(keep, s_scan, total);
    if (keep) {
      const int d = kept + r;
      t.id[d] = id; t.anchor[d] = anchor; t.lm[d] = lm; t.rho[d] = rho; t.mask[d] = mask & ~bit;
#pragma unroll
      for (int s = 0; s < kKeyframeMaxSlots; ++s)
        if (((mask & ~bit) >> s) & 1u) t.idx[s * S + d] = idx[s];
    }
    if (in) a.new_index[e] = keep ? kept + r : -1;
    kept += total;
  }
  __syncthreads();  // new_index complete (global memory written by this block)
  int placed = 0;
  for (int c = 0; c < a.n_entries; c += kFtThreads) {
    const int j = c + tid;
    const uint64_t x = j < a.n_entries ? a.key_in[j] : 0;
    const int ne = j < a.n_entries ? a.new_index[uint32_t(x)] : -1;
    int total;
    const int r = block_exclusive_scan(ne >= 0, s_scan, total);
    if (ne >= 0) a.key_out[placed + r] = (x & 0xffffffff00000000ull) | uint32_t(ne);
    placed += total;
  }
  if (tid == 0) {
    a.out[0] = a.n_entries - kept;
    if constexpr (kReanchor) a.out[1] = n_reanchored;
  }
}

// Window: setDepth of the last window's landmarks, then the numbering of getDepthVector (isLandmarkCandidate: used_num >= 2
// && start_frame < window_size - 2) in table order, the inverse depths re-laid out to it (rho_out) and the observation CSR
// (anchor first, then the listed slots in window order) with per-landmark records.
__global__ void __launch_bounds__(kFtThreads) feature_table_window_kernel(FeatureTableWindowArgs a) {
  __shared__ int s_scan[32];
  const int tid = threadIdx.x;
  const FeatureTablePtrs& t = a.t;
  constexpr size_t S = kFeatureTableMaxEntries;
  int n_lm = 0, n_obs = 0;
  for (int c = 0; c < a.n_entries; c += kFtThreads) {
    const int e = c + tid;
    const bool in = e < a.n_entries;
    bool cand = false;
    int used = 0, anchor = 0;
    uint32_t mask = 0;
    double rho = 0.0;
    if (in) {
      const int lm = t.lm[e];
      rho = t.rho[e];
      if (lm >= 0 && lm < a.n_rho_in) { rho = a.rho_in[lm]; t.rho[e] = rho; }  // setDepth (feature_manager.cpp:126-147)
      mask = t.mask[e];
      anchor = t.anchor[e];
      used = __popc(mask & a.w.listed);
      cand = used >= 2 && a.w.position[anchor] < a.window_size - 2;
    }
    int n_cand, n_used;
    const int rl = block_exclusive_scan(cand, s_scan, n_cand);
    const int ro = block_exclusive_scan(cand ? used : 0, s_scan, n_used);
    if (in) t.lm[e] = cand ? n_lm + rl : -1;
    if (cand) {
      const int l = n_lm + rl;
      int o = n_obs + ro;
      a.rho_out[l] = rho;
      a.obs_offset[l] = o;
      a.lm_id[l] = t.id[e];
      a.lm_anchor[l] = anchor;
      a.lm_used[l] = used;
      a.obs_slot[o] = anchor;
      a.obs_idx[o++] = t.idx[anchor * S + e];
      for (int k = 0; k < a.w.n_frames; ++k) {
        const int s = a.w.slot[k];
        if (s != anchor && ((mask >> s) & 1u)) { a.obs_slot[o] = s; a.obs_idx[o++] = t.idx[s * S + e]; }
      }
    }
    n_lm += n_cand;
    n_obs += n_used;
  }
  if (tid == 0) { a.obs_offset[n_lm] = n_obs; a.out[0] = n_lm; a.out[1] = n_obs; }
}

// image factors of the numbered landmarks (trajectory_manager.cpp:206-236, :359-385): one thread per landmark writes its
// (anchor, observation) descriptors at obs_offset[l] - l, in the CSR's window order
__global__ void feature_table_factors_kernel(FeatureTableFactorArgs a) {
  const int l = blockIdx.x * blockDim.x + threadIdx.x;
  if (l >= a.n_landmarks) return;
  const int o0 = a.obs_offset[l], o1 = a.obs_offset[l + 1];
  const int si = a.obs_slot[o0];
  const int ti = si * a.frame_cap + a.obs_idx[o0];
  const int marg = (a.marg_oldest && si == a.oldest_slot && a.rho[l] > 0.0) ? 1 : 0;  // :216-218
  FactorDesc* d = a.out + (o0 - l);
  for (int k = o0 + 1; k < o1; ++k) d[k - o0 - 1] = FactorDesc{ti, a.obs_slot[k] * a.frame_cap + a.obs_idx[k], l, marg};
}

// Map: GetLandmarksInWindow / GetMarginCloud (visual_odometry.cpp:310-372) and the keyframe poses of PublishVioKeyFrame
// over the listed window.  The listed frames' camera poses (GetCameraPose at the frame time, :197-202) are evaluated
// first into shared memory; then the entries, in chunks of kFtThreads: IsLandMarkStable (visual_odometry.h:82-93), a
// block scan, and the stable ones are written compacted, in table order, to mapped host memory.  No atomics.
// kCov: each written point also gets its 3 x 3 covariance at the same row of point_cov9, gathered from the window's
// per-landmark covariances lm_cov9 at the entry's number; NaN for an entry without one (never numbered, or re-anchored
// by the slide, which clears the number).
template <bool kCov>
__global__ void __launch_bounds__(kFtThreads) feature_table_map_kernel(FeatureTableMapArgs a) {
  __shared__ double s_cam[kKeyframeMaxSlots][12];  // by window position: camera R (9) | camera t (3)
  __shared__ int s_scan[32];
  const int tid = threadIdx.x;
  const FeatureTablePtrs& t = a.t;
  constexpr size_t S = kFeatureTableMaxEntries;
  if (tid < a.w.n_frames) {
    M3 Rc;
    V3 tc;
    camera_pose_at(a.st, a.sp, a.R_CI, a.p_CI, a.frame_t[a.w.slot[tid]], Rc, tc);
#pragma unroll
    for (int e = 0; e < 9; ++e) s_cam[tid][e] = Rc.m[e];
    s_cam[tid][9] = tc.x; s_cam[tid][10] = tc.y; s_cam[tid][11] = tc.z;
    const Q4 q = quat_from_matrix(Rc);
    double* c = a.head->cam[tid];
    c[0] = q.x; c[1] = q.y; c[2] = q.z; c[3] = q.w;
    c[4] = tc.x; c[5] = tc.y; c[6] = tc.z;
  }
  __syncthreads();
  const double late = a.window_size * 3.0 / 4.0;
  int n_points = 0;
  for (int c = 0; c < a.n_entries; c += kFtThreads) {
    const int e = c + tid;
    bool stable = false, margin = false;
    MapPoint p;
    [[maybe_unused]] int lm_cov = -1;
    if (e < a.n_entries) {
      const int anchor = t.anchor[e], lm = t.lm[e];
      const uint32_t mask = t.mask[e];
      const int start = a.w.position[anchor];
      const int used = __popc(mask & a.w.listed);
      const bool numbered = lm >= 0 && lm < a.n_rho;
      const double depth = 1.0 / (numbered ? a.rho[lm] : t.rho[e]);  // the next setDepth's value, else the stored one
      // isLandmarkCandidate, start_frame > WINDOW_SIZE * 3 / 4, estimated_depth <= 0 (a NaN depth passes)
      stable = used >= 2 && start < a.window_size - 2 && !(start > late) && !(depth <= 0.0);
      // GetMarginCloud: start_frame == 0, used_num <= 2, solve_flag == SovelSucc (setDepth's !(depth < 0) of a numbered
      // entry, which stable implies; a re-anchored entry carries it in kFeatureSolvedBit)
      margin = stable && start == 0 && used <= 2 && (numbered || (mask & kFeatureSolvedBit));
      if (stable) {
        const FrameFeature f = a.table[size_t(anchor) * a.frame_cap + t.idx[anchor * S + e]];
        const double* w = s_cam[start];
        const V3 pc{f.x * depth, f.y * depth, depth};  // feature_per_frame[0].point * estimated_depth
#pragma unroll
        for (int r = 0; r < 3; ++r) p.xyz[r] = w[3 * r] * pc.x + w[3 * r + 1] * pc.y + w[3 * r + 2] * pc.z + w[9 + r];
        p.id = t.id[e];
        p.in_margin_cloud = margin ? 1 : 0;
        if constexpr (kCov) lm_cov = lm >= 0 && lm < a.n_cov ? lm : -1;
      }
    }
    int total;
    const int r = block_exclusive_scan(stable, s_scan, total);
    if (stable) {
      a.points[n_points + r] = p;
      if constexpr (kCov) {
        double* dst = a.point_cov9 + 9 * size_t(n_points + r);
#pragma unroll
        for (int k = 0; k < 9; ++k) dst[k] = lm_cov >= 0 ? a.lm_cov9[9 * size_t(lm_cov) + k] : NAN;
      }
    }
    n_points += total;
  }
  if (tid == 0) { a.head->n_points = n_points; a.head->pad = 0; }
}

// ---- wire formats -> resident tables ----------------------------------------------------------------

__global__ void unpack_cloud_kernel(UnpackCloudArgs a) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= a.n) return;
  // FeatureMsg2Image: id = int(channels[0] + 0.5); x, y from points[i] (z == 1); p_v = channels[2]
  const int id = int(double(a.ch_id[i]) + 0.5);
  const double x = double(a.points[3 * i]), y = double(a.points[3 * i + 1]);
  FrameFeature f;
  f.x = x; f.y = y;
  f.id = id;
  f.row = int(round(double(a.ch_v[i])));  // std::round(uv(1)) at the Add* call site (trajectory_manager.cpp:366, 374)
  a.out[i] = f;
}

__global__ void unpack_imu_kernel(UnpackImuArgs a) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= a.n) return;
  const unsigned char* rec = a.raw + size_t(i) * a.stride;
  // IMUData: int64 timestamp @0, Vector3d gyro, Vector3d accel (offsets given by the caller)
  const int64_t t = *reinterpret_cast<const int64_t*>(rec);
  const double* g = reinterpret_cast<const double*>(rec + a.off_gyro);
  const double* ac = reinterpret_cast<const double*>(rec + a.off_accel);
  // bias node of the sample (trajectory_manager.cpp:383-403): 0 before kf 0, last at / after the newest kf,
  // else the interval [kf_{i-1}, kf_i) -> i - 1
  int node = 0;
  if (a.n_kf > 0) {
    if (t < a.kf_t[0]) node = 0;
    else if (t >= a.kf_t[a.n_kf - 1]) node = a.n_kf - 1;
    else {
      for (int k = 1; k < a.n_kf; ++k)
        if (t >= a.kf_t[k - 1] && t < a.kf_t[k]) { node = k - 1; break; }
    }
  }
  a.t_node[a.dst0 + i] = make_longlong2(t, node);
  a.ga[3 * size_t(a.dst0 + i)] = make_double2(g[0], g[1]);
  a.ga[3 * size_t(a.dst0 + i) + 1] = make_double2(g[2], ac[0]);
  a.ga[3 * size_t(a.dst0 + i) + 2] = make_double2(ac[1], ac[2]);
}

__global__ void gather_factors_kernel(GatherFactorsArgs a) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= a.n) return;
  const FactorDesc d = a.desc[k];
  const FrameFeature fi = a.table[d.slot_i], fj = a.table[d.slot_j];
  a.t[k] = make_longlong2(a.frame_t[d.slot_i / a.frame_cap], a.frame_t[d.slot_j / a.frame_cap]);
  a.pi[k] = make_double2(fi.x, fi.y);
  a.pj[k] = make_double2(fj.x, fj.y);
  a.meta[k] = make_int4(fi.row, fj.row, d.lm, d.marg);
}

// ---- device-resident window bookkeeping (SURVEY 8f-1): nothing below touches the host ---------------------------
__global__ void extend_knots_kernel(StatePtrs st, int old_n, int new_n) {
  const int k = old_n + blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= new_n) return;
  // trajectory_manager.cpp:114-115: extendKnotsTo(max_time, last_knot)
#pragma unroll
  for (int c = 0; c < 4; ++c) {
    st.q[4 * k + c] = st.q[4 * (old_n - 1) + c];
    st.p[kPStride * k + c] = st.p[kPStride * (old_n - 1) + c];
  }
}
__global__ void slide_copy_kernel(StatePtrs st, int nK, int nB, double* tmp) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < 4 * nK) tmp[i] = st.q[i];
  if (i < kPStride * nK) tmp[4 * nK + i] = st.p[i];
  if (i < 6 * nB) tmp[8 * nK + i] = st.bias[i];
}
__global__ void slide_shift_kernel(StatePtrs st, int nK, int nB, int dk, int db, int new_bias, const double* tmp) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < 4 * (nK - dk)) st.q[i] = tmp[4 * dk + i];
  if (i < kPStride * (nK - dk)) st.p[i] = tmp[4 * nK + kPStride * dk + i];
  const int keepb = nB - db;
  if (i < 6 * (keepb + new_bias)) {
    const int b = i / 6, c = i - 6 * b;
    // kept nodes move down; appended nodes start from the newest estimate (Bgs_[WINDOW_SIZE] after slideWindow)
    const int srcb = b < keepb ? b + db : nB - 1;
    st.bias[i] = nB > 0 ? tmp[8 * nK + 6 * srcb + c] : 0.0;
  }
}
__global__ void remap_rho_kernel(const double* old_rho, const int32_t* old_index, const double* init_rho, int n, double* out) {
  const int l = blockIdx.x * blockDim.x + threadIdx.x;
  if (l >= n) return;
  out[l] = old_index[l] >= 0 ? old_rho[old_index[l]] : init_rho[l];
}
__global__ void shift_imu_copy_kernel(const longlong2* t, const double2* ga, int from, int count, double* tmp) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= count) return;
  longlong2* tt = reinterpret_cast<longlong2*>(tmp);
  double2* tg = reinterpret_cast<double2*>(tmp + 2 * size_t(count));
  tt[k] = t[from + k];
#pragma unroll
  for (int c = 0; c < 3; ++c) tg[3 * k + c] = ga[3 * size_t(from + k) + c];
}
__global__ void shift_imu_back_kernel(longlong2* t, double2* ga, int count, const double* tmp) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= count) return;
  const longlong2* tt = reinterpret_cast<const longlong2*>(tmp);
  const double2* tg = reinterpret_cast<const double2*>(tmp + 2 * size_t(count));
  t[k] = tt[k];
#pragma unroll
  for (int c = 0; c < 3; ++c) ga[3 * size_t(k) + c] = tg[3 * k + c];
}
__global__ void gather_imu_kernel(const int2* src, int n, const longlong2* tab_t, const double2* tab_ga, longlong2* out_t,
                                  double2* out_ga) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n) return;
  const int2 s = src[k];
  out_t[k] = make_longlong2(tab_t[s.x].x, s.y);
#pragma unroll
  for (int c = 0; c < 3; ++c) out_ga[3 * size_t(k) + c] = tab_ga[3 * size_t(s.x) + c];
}
// linearisation point of the kept blocks of a fresh prior (marginalization_factor.cpp:223-236)
__global__ void prior_x0_kernel(StatePtrs st, const int32_t* type, const int32_t* index, int nb, double* x0) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= nb) return;
  const int t = type[b];
  const double* x = block_state(st, t, index[b]);
  const int stored = t == CTVIO_BLK_ROT ? 4 : block_dim(t);  // a rotation keeps its quaternion
  for (int c = 0; c < 4; ++c) x0[4 * b + c] = c < stored ? x[c] : 0.0;
}

}  // namespace

int launch_triangulate(const TriangulateArgs& a, cudaStream_t s) {
  if (a.n_landmarks <= 0) return 0;
  triangulate_kernel<<<(a.n_landmarks + 127) / 128, 128, 0, s>>>(a);
  return 1;
}
int launch_triangulate_window(const TriangulateWindowArgs& a, cudaStream_t s) {
  if (a.n_landmarks <= 0) return 0;
  triangulate_window_kernel<<<(a.n_landmarks + kTriLmPerCta - 1) / kTriLmPerCta, kTriThreads, 0, s>>>(a);
  return 1;
}
int launch_keyframe_parallax(const KeyframeArgs& a, cudaStream_t s) {
  keyframe_parallax_kernel<<<1, kKfThreads, 0, s>>>(a);
  return 1;
}
int launch_feature_table_add(const FeatureTableAddArgs& a, cudaStream_t s) {
  feature_table_add_kernel<<<1, kFtThreads, 0, s>>>(a);
  return 1;
}
int launch_feature_table_slide(const FeatureTableSlideArgs& a, cudaStream_t s) {
  feature_table_slide_kernel<false><<<1, kFtThreads, 0, s>>>(a);
  return 1;
}
int launch_feature_table_slide_reanchor(const FeatureTableSlideArgs& a, cudaStream_t s) {
  feature_table_slide_kernel<true><<<1, kFtThreads, 0, s>>>(a);
  return 1;
}
int launch_feature_table_window(const FeatureTableWindowArgs& a, cudaStream_t s) {
  feature_table_window_kernel<<<1, kFtThreads, 0, s>>>(a);
  return 1;
}
int launch_feature_table_factors(const FeatureTableFactorArgs& a, cudaStream_t s) {
  if (a.n_landmarks <= 0) return 0;
  feature_table_factors_kernel<<<(a.n_landmarks + 127) / 128, 128, 0, s>>>(a);
  return 1;
}
int launch_feature_table_map(const FeatureTableMapArgs& a, cudaStream_t s) {
  feature_table_map_kernel<false><<<1, kFtThreads, 0, s>>>(a);
  return 1;
}
int launch_feature_table_map_cov(const FeatureTableMapArgs& a, cudaStream_t s) {
  feature_table_map_kernel<true><<<1, kFtThreads, 0, s>>>(a);
  return 1;
}
int launch_unpack_cloud(const UnpackCloudArgs& a, cudaStream_t s) {
  if (a.n <= 0) return 0;
  unpack_cloud_kernel<<<(a.n + 127) / 128, 128, 0, s>>>(a);
  return 1;
}
int launch_unpack_imu(const UnpackImuArgs& a, cudaStream_t s) {
  if (a.n <= 0) return 0;
  unpack_imu_kernel<<<(a.n + 127) / 128, 128, 0, s>>>(a);
  return 1;
}
int launch_gather_factors(const GatherFactorsArgs& a, cudaStream_t s) {
  if (a.n <= 0) return 0;
  gather_factors_kernel<<<(a.n + 127) / 128, 128, 0, s>>>(a);
  return 1;
}

int launch_extend_knots(const StatePtrs& st, int old_n, int new_n, cudaStream_t s) {
  if (new_n <= old_n) return 0;
  extend_knots_kernel<<<(new_n - old_n + 63) / 64, 64, 0, s>>>(st, old_n, new_n);
  return 1;
}
int launch_slide_state(const StatePtrs& st, int nK, int nB, int dk, int db, int new_bias, double* tmp, cudaStream_t s) {
  const int work = std::max(8 * nK, 6 * (nB + new_bias)) + 1;
  slide_copy_kernel<<<(work + 127) / 128, 128, 0, s>>>(st, nK, nB, tmp);
  slide_shift_kernel<<<(work + 127) / 128, 128, 0, s>>>(st, nK, nB, dk, db, new_bias, tmp);
  return 2;
}
int launch_remap_rho(const double* old_rho, const int32_t* old_index, const double* init_rho, int n, double* out, cudaStream_t s) {
  if (n <= 0) return 0;
  remap_rho_kernel<<<(n + 127) / 128, 128, 0, s>>>(old_rho, old_index, init_rho, n, out);
  return 1;
}
int launch_shift_imu_table(longlong2* t, double2* ga, int from, int count, double* tmp, cudaStream_t s) {
  if (count <= 0 || from <= 0) return 0;
  shift_imu_copy_kernel<<<(count + 127) / 128, 128, 0, s>>>(t, ga, from, count, tmp);
  shift_imu_back_kernel<<<(count + 127) / 128, 128, 0, s>>>(t, ga, count, tmp);
  return 2;
}
int launch_gather_imu(const int2* src, int n, const longlong2* tab_t, const double2* tab_ga, longlong2* out_t, double2* out_ga,
                      cudaStream_t s) {
  if (n <= 0) return 0;
  gather_imu_kernel<<<(n + 127) / 128, 128, 0, s>>>(src, n, tab_t, tab_ga, out_t, out_ga);
  return 1;
}
int launch_prior_x0(const StatePtrs& st, const int32_t* type, const int32_t* index, int nb, double* x0, cudaStream_t s) {
  if (nb <= 0) return 0;
  prior_x0_kernel<<<(nb + 63) / 64, 64, 0, s>>>(st, type, index, nb, x0);
  return 1;
}

}  // namespace ctvio
