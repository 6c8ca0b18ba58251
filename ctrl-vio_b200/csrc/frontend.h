// Front-end data formats either side of the hot path (frontend.cu): DLT triangulation (from caller poses, and of the
// resident window from the resident spline), the keyframe decision over the resident frame slots, wire-format unpacking,
// device-side construction of the sorted image-factor arrays from the resident per-frame feature tables, and the
// published landmark map of the resident feature table.
#pragma once
#include <cuda_runtime.h>

#include <cstdint>

#include "kernels.h"

namespace ctvio {

struct TriangulateArgs {
  int32_t n_frames;
  const double* Rs;          // [n_frames][9] row-major body rotations
  const double* Ps;          // [n_frames][3]
  M3 ric;                    // camera -> body rotation
  V3 tic;
  int32_t n_landmarks;
  const int32_t* start_frame;  // [n_landmarks]
  const int32_t* obs_offset;   // [n_landmarks + 1] into obs_point; frame of observation k = start_frame + k
  const double* obs_point;     // [total][3]  FeaturePerFrame::point (x, y, 1)
  int32_t window_size;         // WINDOW_SIZE (candidate rule start_frame < WINDOW_SIZE - 2)
  double init_depth;           // INIT_DEPTH
  double* depth;               // [n_landmarks] in/out: > 0 is kept
};
int launch_triangulate(const TriangulateArgs& a, cudaStream_t s);

// one tracked feature of one frame in the resident table (32 B)
struct FrameFeature {
  double x, y;   // undistorted bearing (z == 1)
  int32_t id;    // tracker feature id
  int32_t row;   // rounded pixel row (rolling-shutter line)
  int64_t pad;
};
struct UnpackCloudArgs {
  int32_t n;
  const float* points;  // [n][3] geometry_msgs::Point32
  const float* ch_id;   // channels[0]
  const float* ch_v;    // channels[2]
  FrameFeature* out;    // [n] slice of the frame table
};
int launch_unpack_cloud(const UnpackCloudArgs& a, cudaStream_t s);

struct UnpackImuArgs {
  int32_t n;
  const unsigned char* raw;  // device copy of the IMUData records
  int32_t stride, off_gyro, off_accel;
  const int64_t* kf_t;       // [n_kf] keyframe timestamps (bias-node assignment)
  int32_t n_kf;
  int32_t dst0;              // first destination sample
  longlong2* t_node;
  double2* ga;
};
int launch_unpack_imu(const UnpackImuArgs& a, cudaStream_t s);

// image factor k = (anchor table slot, observation table slot, landmark, marg flag); slot = frame_slot * frame_cap + i
struct FactorDesc {
  int32_t slot_i, slot_j, lm, marg;
};
struct GatherFactorsArgs {
  int32_t n;
  const FactorDesc* desc;     // already in K1's sorted (frame-pair group) order
  const FrameFeature* table;  // [n_slots][frame_cap]
  const int64_t* frame_t;     // [n_slots]
  int32_t frame_cap;
  longlong2* t;
  double2* pi;
  double2* pj;
  int4* meta;
};
int launch_gather_factors(const GatherFactorsArgs& a, cudaStream_t s);

// DLT of the resident window's landmarks: observation k of landmark l (obs_offset[l] <= k < obs_offset[l+1], the first
// one the anchor) is feature obs_idx[k] of frame slot obs_slot[k]; its camera pose is the resident spline at the row
// time frame_t[slot] + row * int64(ld * 1e9) composed with the extrinsic.  Only landmarks with rho_in <= 0 get a new
// value; rho_out receives every landmark (kept ones bitwise).
struct TriangulateWindowArgs {
  int32_t n_landmarks;
  const int32_t* obs_offset;  // [n_landmarks + 1], obs_offset[0] == 0
  const int32_t* obs_slot;    // [total]
  const int32_t* obs_idx;     // [total]
  const FrameFeature* table;  // [n_slots][frame_cap]
  const int64_t* frame_t;     // [n_slots]
  int32_t frame_cap;
  StatePtrs st;               // knots, knot-pair table (valid), line delay
  SplineParams sp;
  M3 R_CI;                    // camera -> IMU rotation
  V3 p_CI;
  double init_depth;          // INIT_DEPTH
  const double* rho_in;       // [n_landmarks]
  double* rho_out;            // [n_landmarks] (must not alias rho_in)
  int32_t* counts;            // [2] zeroed by the caller: {triangulated, fallback}; sign bit of [0] = a time left the spline
};
int launch_triangulate_window(const TriangulateWindowArgs& a, cudaStream_t s);

constexpr int kKeyframeMaxSlots = 16, kKeyframeMaxFeatures = 1024;
// a window listed by the caller as resident frame slots, oldest to newest (each slot at most once)
struct WindowSlots {
  int32_t n_frames;                     // 1 .. kKeyframeMaxSlots
  int32_t slot[kKeyframeMaxSlots];      // frame slot of each window position
  int32_t position[kKeyframeMaxSlots];  // window position of each frame slot (-1: not listed)
  uint32_t listed;                      // mask of the listed slots
};

// Keyframe decision of the new image (addFeatureCheckParallax, feature_manager.cpp:28-87) over resident frame slots:
// w.slot[0 .. n_frames-1] lists the window oldest to newest, the last one the new image.  One CTA of
// kKeyframeMaxFeatures threads; every slot holds at most kKeyframeMaxFeatures features.
struct KeyframeResult {
  int32_t is_keyframe;
  int32_t n_tracked;     // features of the new slot whose id occurs in another listed slot (last_track_num)
  int32_t parallax_num;  // features of slot fc-1 whose id occurs in slot fc-2 (0 when fc < 2)
  int32_t pad;
  double parallax_sum;   // sum of their bearing distances, summed in a fixed order
};
struct KeyframeArgs {
  const FrameFeature* table;  // [n_slots][frame_cap]
  int32_t frame_cap;
  WindowSlots w;
  int32_t count[kKeyframeMaxSlots];  // features ingested in w.slot[k] (<= kKeyframeMaxFeatures)
  double min_parallax;        // MIN_PARALLAX
  KeyframeResult* out;
};
int launch_keyframe_parallax(const KeyframeArgs& a, cudaStream_t s);

// Resident feature table (FeatureManager's feature list): one entry per landmark in creation order, structure of arrays
// over kFeatureTableMaxEntries entries.  idx[s * kFeatureTableMaxEntries + e] is entry e's feature index in frame slot s,
// valid where bit s of mask[e] is set (the anchor slot's bit included).  The live entries' (id, entry) keys are kept
// sorted (kf_key order) in a separate array.  Bit kFeatureSolvedBit of mask[e] carries solve_flag == SovelSucc across a
// re-anchoring slide, which clears the entry's number (only the re-anchoring slide sets it; it is never cleared).
constexpr int kFeatureTableMaxEntries = kKeyframeMaxSlots * kKeyframeMaxFeatures;
constexpr uint32_t kFeatureSolvedBit = 1u << 31;
static_assert(kKeyframeMaxSlots <= 31, "the solved bit sits above the slot bits");
struct FeatureTablePtrs {
  int32_t* id;       // tracker feature id
  int32_t* anchor;   // anchor frame slot
  uint32_t* mask;    // slots holding an observation (bits 0..15), kFeatureSolvedBit
  int32_t* lm;       // number in the last window, -1: not numbered
  double* rho;       // inverse depth (estimated_depth), -1: not initialised
  int32_t* idx;      // [kKeyframeMaxSlots][kFeatureTableMaxEntries]
};
struct FeatureTableAddArgs {
  FeatureTablePtrs t;
  int32_t n_entries;
  const uint64_t* key_in;      // [n_entries] sorted keys of the live entries
  uint64_t* key_out;           // [n_entries + n_new]
  const FrameFeature* cloud;   // the slot's features
  int32_t n_features;          // <= kKeyframeMaxFeatures
  int32_t slot;
  int32_t* out;                // {n_tracked, n_new}
};
struct FeatureTableSlideArgs {
  FeatureTablePtrs t;
  int32_t n_entries;
  const uint64_t* key_in;
  uint64_t* key_out;
  int32_t* new_index;          // [n_entries] scratch
  int32_t slot;                // the leaving slot
  const double* rho;           // resident inverse depths of the last window's numbering
  int32_t n_rho;               // their count (0: no numbering, removeFailures is skipped)
  int32_t* out;                // {n_removed}; the re-anchoring slide: {n_removed, n_reanchored}
  // the re-anchoring slide (feature_table_slide_kernel<true>) only
  WindowSlots w;               // the window before the slide, oldest to newest (w.listed: the held slots)
  int32_t marg_old;            // 1: slot == w.slot[0] (removeBackShiftDepth); 0: slot == w.slot[n_frames-2] (removeFront)
  double init_depth;           // INIT_DEPTH, for a shifted depth that is not > 0
  const FrameFeature* table;   // MARGIN_OLD: the anchor bearings, [n_slots][frame_cap]
  int32_t frame_cap;
  const int64_t* frame_t;      // MARGIN_OLD: w.slot[0] and w.slot[1]'s frame times lie inside the spline (caller checks)
  StatePtrs st;                // MARGIN_OLD: knots, knot-pair table (valid)
  SplineParams sp;
  M3 R_CI;                     // camera -> IMU rotation
  V3 p_CI;
};
struct FeatureTableWindowArgs {
  FeatureTablePtrs t;
  int32_t n_entries;
  WindowSlots w;
  int32_t window_size;
  const double* rho_in;        // resident inverse depths of the last numbering
  int32_t n_rho_in;            // their count (0: no numbering)
  double* rho_out;             // [n_landmarks] the new numbering's inverse depths (must not alias rho_in)
  int32_t* obs_offset;         // [n_landmarks + 1]
  int32_t* obs_slot;           // [n_obs] anchor first, then the listed slots in window order
  int32_t* obs_idx;            // [n_obs]
  int32_t* lm_id;              // [n_landmarks] per-landmark records: feature id, anchor slot, used_num
  int32_t* lm_anchor;
  int32_t* lm_used;
  int32_t* out;                // {n_landmarks, n_obs}
};
struct FeatureTableFactorArgs {
  int32_t n_landmarks;
  const int32_t* obs_offset;
  const int32_t* obs_slot;
  const int32_t* obs_idx;
  const double* rho;           // resident inverse depths (marg flag: rho > 0)
  int32_t oldest_slot;         // slot of window position 0
  int32_t marg_oldest;
  int32_t frame_cap;
  FactorDesc* out;             // [obs_offset[n_landmarks] - n_landmarks], landmark-major
};
// the published landmark map (GetLandmarksInWindow / GetMarginCloud / PublishVioKeyFrame), written by
// feature_table_map_kernel straight into mapped host memory: a header with the listed frames' camera poses, then the
// stable points compacted in table order
struct MapPoint {              // 32 B
  double xyz[3];               // world point
  int32_t id;                  // tracker feature id
  int32_t in_margin_cloud;     // 0 / 1
};
struct MapHeader {
  int32_t n_points;            // stable entries (all of them are written to points)
  int32_t pad;
  double cam[kKeyframeMaxSlots][7];  // camera pose at each listed frame's time: q (x, y, z, w), p
};
struct FeatureTableMapArgs {
  FeatureTablePtrs t;          // read only
  int32_t n_entries;
  WindowSlots w;
  int32_t window_size;
  const FrameFeature* table;   // [n_slots][frame_cap]
  const int64_t* frame_t;      // [n_slots]; every listed frame time lies inside the spline (checked by the caller)
  int32_t frame_cap;
  StatePtrs st;                // knots, knot-pair table (valid)
  SplineParams sp;
  M3 R_CI;                     // camera -> IMU rotation
  V3 p_CI;
  const double* rho;           // resident inverse depths of the last window's numbering
  int32_t n_rho;               // their count (0: no numbering)
  MapHeader* head;             // mapped host memory
  MapPoint* points;            // mapped host memory, [kFeatureTableMaxEntries]
  // feature_table_map_kernel<true> (launch_feature_table_map_cov) only
  const double* lm_cov9;       // [n_cov][9] point covariances in the last window's numbering (entry lm)
  int32_t n_cov;               // their count
  double* point_cov9;          // mapped host memory, [kFeatureTableMaxEntries][9], row k for points[k]
};
int launch_feature_table_add(const FeatureTableAddArgs& a, cudaStream_t s);
int launch_feature_table_slide(const FeatureTableSlideArgs& a, cudaStream_t s);
int launch_feature_table_slide_reanchor(const FeatureTableSlideArgs& a, cudaStream_t s);
int launch_feature_table_window(const FeatureTableWindowArgs& a, cudaStream_t s);
int launch_feature_table_factors(const FeatureTableFactorArgs& a, cudaStream_t s);
int launch_feature_table_map(const FeatureTableMapArgs& a, cudaStream_t s);
int launch_feature_table_map_cov(const FeatureTableMapArgs& a, cudaStream_t s);

// device-resident window bookkeeping (all on the device)
int launch_extend_knots(const StatePtrs& st, int old_n, int new_n, cudaStream_t s);
int launch_slide_state(const StatePtrs& st, int nK, int nB, int dk, int db, int new_bias, double* tmp, cudaStream_t s);
int launch_remap_rho(const double* old_rho, const int32_t* old_index, const double* init_rho, int n, double* out, cudaStream_t s);
int launch_shift_imu_table(longlong2* t, double2* ga, int from, int count, double* tmp, cudaStream_t s);
int launch_gather_imu(const int2* src, int n, const longlong2* tab_t, const double2* tab_ga, longlong2* out_t, double2* out_ga,
                      cudaStream_t s);
int launch_prior_x0(const StatePtrs& st, const int32_t* type, const int32_t* index, int nb, double* x0, cudaStream_t s);

}  // namespace ctvio
