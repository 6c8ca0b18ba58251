// The engine object behind a ctvio_handle and the host helpers engine.cu, resident.cu and solve.cu share.  The
// thread-locals are C++17 inline variables, ONE object each across the library: an error raised in any of the files is
// what ctvio_last_error reports, and every upload is counted.
#pragma once
#include <algorithm>
#include <cmath>
#include <cstring>
#include <string>
#include <vector>

#include "../../include/ctvio.h"
#include "frontend.h"      // + kernels.h
#include "marginalize.h"

namespace ctvio::host {

inline thread_local std::string g_err;  // ctvio_last_error
inline int fail(int code, const std::string& msg) {
  g_err = msg;
  return code;
}

#define CUDA_OK(call)                                                                                   \
  do {                                                                                                  \
    cudaError_t e_ = (call);                                                                            \
    if (e_ != cudaSuccess)                                                                              \
      return fail(CTVIO_ERR_CUDA, std::string(#call) + ": " + cudaGetErrorString(e_));                  \
  } while (0)

// host waits on the device by this thread's C-ABI calls (stream synchronisations and spins on the LM step's published
// scalars), see ctvio_sync_stats
inline thread_local int64_t g_host_waits = 0;
inline cudaError_t stream_sync(cudaStream_t s) {
  ++g_host_waits;
  return cudaStreamSynchronize(s);
}

inline thread_local size_t g_upload_bytes = 0;  // bytes moved by DevBuf::upload (index tables etc.), see ctvio_transfer_stats

// Pinned staging arena of one engine: every host -> device copy of a C-ABI call is staged here and issued as a truly
// asynchronous copy (a cudaMemcpyAsync from pageable memory is a synchronous staged copy, and there are ~20 of them per
// window).  The arena is rewound whenever the engine's stream is found idle at the start of a call (then every copy that
// read from it has completed); a request that does not fit falls back to the pageable copy and grows the arena at the
// next rewind.
struct PinnedArena {
  unsigned char* base = nullptr;
  size_t cap = 0, need = 0;  // need: bytes requested since the last rewind (may exceed cap: those requests fell back)
  ~PinnedArena() { if (base) cudaFreeHost(base); }
  void rewind() {
    if (need > cap) {
      if (base) cudaFreeHost(base);
      base = nullptr;
      cap = 0;
      const size_t n = std::max<size_t>(size_t(1) << 20, need + need / 2);
      if (cudaHostAlloc(reinterpret_cast<void**>(&base), n, cudaHostAllocDefault) == cudaSuccess) cap = n;
      else cudaGetLastError();
    }
    need = 0;
  }
  void* put(const void* src, size_t bytes) {
    const size_t o = (need + 15) & ~size_t(15);
    need = o + bytes;
    if (!base || need > cap) return nullptr;
    std::memcpy(base + o, src, bytes);
    return base + o;
  }
};
inline thread_local PinnedArena* g_arena = nullptr;  // arena of the engine whose C-ABI call is running on this thread

inline cudaError_t staged_h2d(void* dst, const void* src, size_t bytes, cudaStream_t s) {
  if (bytes == 0) return cudaSuccess;
  if (g_arena) {
    if (void* st = g_arena->put(src, bytes)) return cudaMemcpyAsync(dst, st, bytes, cudaMemcpyHostToDevice, s);
  }
  // pageable source: the runtime stages it synchronously, the caller's buffer is free again on return
  return cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, s);
}

template <typename T>
struct DevBuf {
  T* p = nullptr;
  size_t cap = 0;
  ~DevBuf() { if (p) cudaFree(p); }
  cudaError_t reserve(size_t n) {
    if (n <= cap) return cudaSuccess;
    if (p) cudaFree(p);
    p = nullptr;
    cap = 0;
    cudaError_t e = cudaMalloc(&p, std::max<size_t>(n, 1) * sizeof(T));
    if (e == cudaSuccess) cap = n;
    return e;
  }
  // reallocate to at least n elements that start with elements [from, from + count) of the old buffer (count = 0: a plain
  // reallocation); the stream is synchronised before the old buffer is freed, since work in flight may still read it
  cudaError_t grow(size_t n, size_t from, size_t count, cudaStream_t s) {
    DevBuf<T> nb;
    cudaError_t e = nb.reserve(n);
    if (e == cudaSuccess && count) e = cudaMemcpyAsync(nb.p, p + from, count * sizeof(T), cudaMemcpyDeviceToDevice, s);
    if (e == cudaSuccess) e = stream_sync(s);
    if (e == cudaSuccess) swap(*this, nb);
    return e;
  }
  cudaError_t upload(const std::vector<T>& h, cudaStream_t s) {
    cudaError_t e = reserve(h.size());
    if (e != cudaSuccess || h.empty()) return e;
    g_upload_bytes += h.size() * sizeof(T);
    return staged_h2d(p, h.data(), h.size() * sizeof(T), s);
  }
};
template <typename T>
void swap(DevBuf<T>& a, DevBuf<T>& b) { std::swap(a.p, b.p); std::swap(a.cap, b.cap); }

struct DevState {
  DevBuf<double> q, p, bias, rho, ld;
  DevBuf<KnotPair> tab;
  StatePtrs ptrs() { return StatePtrs{q.p, p.p, bias.p, rho.p, ld.p, tab.p}; }
};

struct HostImage { int64_t ti, tj; int32_t rowi, rowj; double pi[2], pj[2]; int32_t lm, marg; };
struct HostImu { int64_t t; double gyro[3], accel[3]; int32_t node, marg; };
struct HostBias { int32_t i, j; double s[6]; int32_t marg; };

// The odometry cycle's covariance publications (ctvio_cycle_covariances).  Host side: pinned + mapped, allocated on
// first use; the kernels and copies of one cycle write it, the host reads it after a synchronisation the cycle makes
// anyway.
struct CycleCovHost {
  LmPublished pub;                                         // the rank test's inputs, written by cov_publish_kernel
  int64_t t[kKeyframeMaxSlots + 1];                        // staging of Cycle::cov_t
  double cov12[144];
  double cov6[(kKeyframeMaxSlots - 1) * 36];
  double map_cov9[size_t(kFeatureTableMaxEntries) * 9];    // written by feature_table_map_kernel<true>
};
// what the last cycle published
struct CycleCovState {
  bool ran = false;         // the last cycle completed (cleared when one starts)
  int32_t requested = 0;    // its options' publications: 1 pose, 2 odometry, 4 map
  int32_t available = 0;    // the same bits for what it published
  int32_t status = CTVIO_OK;
  double rcond = NAN;
  int64_t pose_t = 0;
  int32_t n_frames = 0;     // frames of the solved window: n_frames - 1 pairs
  int64_t frame_t[kKeyframeMaxSlots] = {0};
  int32_t n_lm = 0;         // landmarks of the solved window: rows of the per-landmark covariances
  int32_t n_map = 0, n_map_nan = 0;
  bool pending = false;     // Sigma was enqueued; the rank test has not been read yet
  unsigned long long seq = 0;
  std::string why = "no odometry cycle has run";  // why nothing is available (the getter's error message)
};

}  // namespace ctvio::host

using namespace ctvio;
using namespace ctvio::host;

struct ctvio_engine {
  ctvio_config cfg;
  ctvio_options opt;
  cudaStream_t stream = nullptr, stream2 = nullptr, stream3 = nullptr;  // stream2 / stream3: IMU and bias / prior factors run
                                                                         // beside the visual kernel
  cudaEvent_t ev_join3 = nullptr;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr, ev_fork = nullptr, ev_join = nullptr;
  bool masks_dirty = true;
  SplineParams sp;
  RigParams rig;
  bool deterministic = false;   // ctvio_set_deterministic: ordered flushes, single stream (kernels.h)
  DevBuf<int32_t> d_ticket;     // [0] kernel flush ticket, [1] scalar flush ticket

  // sizes
  int nK = 0, nB = 0, nL = 0;
  bool have_knots = false, have_bias = false, have_rho = false;

  // state: two buffers (current / candidate) + snapshot
  DevState x[2], snap;
  DevState xs;                 // third state buffer of the pipelined LM driver (swapped into x[] when it ends up current)
  DevBuf<LmDecision> d_dec;    // device-side step decision (accept, next radius) read by the speculated linear solve
  DevState& state(int i) { return i < 2 ? x[i] : xs; }
  int cur = 0;
  bool table_valid = false;

  // factors (host copies in caller order)
  std::vector<HostImage> img;
  std::vector<HostImu> imu;
  std::vector<HostBias> biasf;
  bool structure_dirty = true;
  // image factors whose descriptors live on the device (caller order): set as soon as ctvio_add_image_features_from_table
  // adds to the factor set; slot-named factors of the same set are uploaded next to them.  No host record exists for
  // these factors, and their structure is built by structure.cu.
  DevBuf<ctvio::FactorDesc> d_img_in;
  int n_img_dev = 0;
  size_t n_img() const { return img.size() + size_t(n_img_dev); }

  // device factor arrays
  DevBuf<longlong2> d_img_t;
  DevBuf<double2> d_img_pi, d_img_pj;
  DevBuf<int4> d_img_meta;
  DevBuf<int32_t> d_img_orig;
  DevBuf<VisualItem> d_items;
  int n_items = 0;
  std::vector<int32_t> img_order;  // sorted position -> original index
  std::vector<int32_t> imu_order;
  DevBuf<longlong2> d_imu_t;
  DevBuf<double2> d_imu_ga;
  DevBuf<ImuItem> d_imu_items;
  DevBuf<int32_t> d_imu_orig;
  int n_imu_items = 0;
  DevBuf<int2> d_bf_ij;
  DevBuf<double> d_bf_s;
  // the first n_bf_dev bias factors of the set take their sqrt_info6 rows from bf_s_dev (device memory, row k for factor
  // k) instead of their host record: the odometry cycle's weights never leave the device
  const double* bf_s_dev = nullptr;
  int n_bf_dev = 0;

  // landmark layout / schur batches
  std::vector<int32_t> h_lo, h_hi;
  std::vector<int64_t> h_woff;
  DevBuf<int32_t> d_lo, d_hi;
  DevBuf<SchurEntry> d_schur_list;
  DevBuf<int64_t> d_woff;
  DevBuf<SchurTileItem> d_schur_items;
  int n_schur_items = 0, n_schur_entries = 0;
  int64_t w_len = 0;                        // length of the compact W array (woff[nL])
  DevBuf<uint8_t> d_cmask, d_active;
  std::vector<uint8_t> h_cmask, h_active;  // h_active: camera part, then the host build's landmark part
  // device structure build (structure.cu): scratch, its count block; either build's knot bitmask of the factors' windows
  DevBuf<uint64_t> sb_key;
  DevBuf<int32_t> sb_idx;
  DevBuf<uint32_t> sb_counts;
  std::vector<uint32_t> h_struct_counts, img_knots;

  // normal equations (two buffers, each one slab: A | gc | hl | gl | wld | W)
  DevBuf<double> ne_slab[2];
  size_t ne_slab_len = 0;
  size_t off_gc = 0, off_hl = 0, off_gl = 0, off_wld = 0, off_W = 0;
  // linear system
  DevBuf<double> d_M, d_Linv, d_y, d_sc, d_sl, d_hh, d_dc, d_dl, d_rho_sync, d_chol_part;
  DevBuf<int32_t> d_chol_flags, d_m_flags;  // tile flags of K5 and of K4 (reduced_system_kernel)
  DevBuf<uint8_t> d_owned;
  DevBuf<double> d_shard_pack, d_shard_scal;  // sharded mode: packed all-reduce buffer, scalar all-gather buffer
  int npad = 0, linv_npad = -1;
  unsigned chol_seq = 0;  // tile-DAG launches so far (packet buffer parity)
  DevBuf<LmScalars> d_scal;
  LmScalars* h_scal = nullptr;  // pinned
  LmPublished* h_pub = nullptr; // pinned + mapped: written by the last kernel of an LM step
  unsigned long long pub_seq = 0;
  cudaEvent_t ev_zero = nullptr;
  bool slab_zeroed[2] = {false, false};  // the normal-equation buffer was cleared ahead of time on stream2

  // prior
  ctvio::PriorHost prior, new_prior;
  DevBuf<double> d_prior_J, d_prior_r, d_prior_JtJ, d_prior_x0, d_prior_dx, d_prior_res;
  DevBuf<int32_t> d_prior_type, d_prior_index, d_prior_col, d_prior_col2g;
  bool prior_dirty = true;
  bool prior_enabled = true;      // ctvio_enable_prior: estimators without the prior (InitTrajectory) keep it resident
  bool prior_on_device = false;   // the active prior's J / r / x0 / J'J were adopted device-to-device (host vectors empty)
  bool new_prior_on_host = false; // ctvio_get_prior has fetched the freshly marginalized prior's J / r / x0
  DevBuf<double> d_newprior_x0;
  // wire-format ingestion (resident.cu, frontend.cu): resident per-frame feature tables, resident IMU table
  static constexpr int kFrameSlots = ctvio::kKeyframeMaxSlots, kFrameCap = ctvio::kKeyframeMaxFeatures;  // 16, 1024
  DevBuf<ctvio::FrameFeature> d_frames;   // [kFrameSlots][kFrameCap]
  DevBuf<int64_t> d_frame_t;              // [kFrameSlots]
  DevBuf<float> d_cloud_stage;            // staging for one message (5 floats per point... points 3 + id + v)
  int64_t h_frame_t[16] = {0};
  int32_t h_frame_n[16] = {0};
  std::vector<ctvio::FactorDesc> img_desc;  // parallel to img when the factors are slot-named (host-built set)
  DevBuf<ctvio::FactorDesc> d_img_desc;
  DevBuf<longlong2> d_imu_tab_t;           // resident IMU table {t, 0}
  DevBuf<double2> d_imu_tab_ga;            // [cap][3]
  DevBuf<unsigned char> d_imu_raw;
  std::vector<int64_t> h_imu_tab_t;        // host mirror: timestamps only
  std::vector<int32_t> imu_src;            // parallel to imu when the samples came from the resident table (table index)
  DevBuf<int2> d_imu_src;
  PinnedArena arena;
  // pinned host mirror of the state, refreshed by the calls that end with a stream synchronisation anyway (solve,
  // re-alignment): the getters then cost a memcpy instead of a device copy + synchronise each
  double* h_mirror = nullptr;
  size_t h_mirror_cap = 0;
  bool mirror_valid = false;
  size_t h2d_bytes = 0, d2h_bytes = 0;     // bytes moved by the C-ABI calls since ctvio_transfer_stats(reset)

  DevBuf<double> d_tmp;  // scratch (gauge inputs, probe outputs)
  DevBuf<int32_t> d_tri_idx;  // index uploads: ctvio_triangulate, ctvio_remap_landmarks, ctvio_triangulate_window
  DevBuf<int32_t> d_tri_cnt;  // ctvio_triangulate_window: {triangulated, fallback}
  DevBuf<ctvio::KeyframeResult> d_kf_result;  // ctvio_check_keyframe
  uint32_t h_frame_ingested = 0;  // frame slots holding a cloud from ctvio_ingest_feature_cloud (cleared when the table slides it)
  // resident feature table (ctvio_feature_table_*), allocated at full size on first use
  struct FeatureTable {
    DevBuf<int32_t> id, anchor, lm, idx, new_index;
    DevBuf<uint32_t> mask;
    DevBuf<double> rho;
    DevBuf<uint64_t> key[2];  // sorted (id, entry) keys, ping-pong
    int cur_key = 0;
    DevBuf<int32_t> obs_offset, obs_slot, obs_idx, lm_id, lm_anchor, lm_used, result;
    DevBuf<ctvio::FactorDesc> desc;
    int n_entries = 0;
    uint32_t held = 0;            // frame slots whose cloud the table holds
    int n_lm = -1;                // landmarks of the last window (-1: none yet); the resident inverse depths follow it
    int n_obs = 0;
    bool window_current = false;  // the CSR and records describe the table as it is (no add / slide since the window)
    int32_t oldest_slot = 0;
    // ctvio_feature_table_map's output, written by its kernel: pinned + mapped, allocated on first use
    ctvio::MapHeader* h_map_head = nullptr;
    ctvio::MapPoint* h_map_points = nullptr;
    ctvio::FeatureTablePtrs ptrs() { return ctvio::FeatureTablePtrs{id.p, anchor.p, mask.p, lm.p, rho.p, idx.p}; }
  } ft;
  // marginalization workspace (K7), kept across windows: allocation / free costs more than the kernels
  struct MargWs {
    DevBuf<int32_t> pos_cam, pos_lm, prior_pos, marg_img, marg_imu, new_type, new_index;
    DevBuf<int2> bij;
    DevBuf<double> eig_scratch, Jrow, bs, A, b, Amm, V, ev, Vs, Ainv, T, Ap, bp, Ap2, V2, ev2, vb, J, r;
  } mws;
  // ctvio_covariance workspace (covariance.cu): Jacobi scales, mask, L^-1, pivots, outputs, the saved scalar block;
  // ctvio_pose_covariance's query times and 12 x 12 outputs; ctvio_point_covariance's landmarks, times (t) and
  // [outputs 9 n | bearings 2 n] (pose); ctvio_relative_pose_covariance's [t_a | t_b] (t) and [cov6 | cross6] (pose)
  struct CovWs {
    DevBuf<double> sc, sl, X, piv, cov, var, pose;
    DevBuf<uint8_t> cmask;
    DevBuf<LmScalars> scal;
    DevBuf<int64_t> t;
    DevBuf<int32_t> lm;
  } cws;
  // the per-image odometry cycle (odometry.cu): the window's frames and the bookkeeping a caller of the separate entry
  // points keeps itself
  struct Cycle {
    bool started = false;
    ctvio_cycle_options opt{};
    int32_t slot[16] = {0};        // window position -> frame slot, oldest to newest
    int64_t t[16] = {0};           // window position -> frame time
    int n_frames = 0;
    int64_t next_frame = 0;        // number of frames the cycle has taken in (the allocator's f)
    DevBuf<double> bias_w;         // [n_frames - 1][6] bias random-walk weights of the current window
    DevBuf<double> imu_carry;      // {prefix of dt^2 at the last sample ingested, its time (int64 bits), valid}
    DevBuf<double> snap;           // local knot 0 before the main solve: q (4), p (3), then R0 / t0 (12)
    // the covariance publications: workspace that lives from the re-alignment to the map (not cws, which every
    // covariance call reuses), and what the last cycle published
    DevBuf<int64_t> cov_t;         // the TF time, then the solved window's frame times
    DevBuf<double> cov_out;        // cov12 (144) | cov6 [n_frames - 1][36] | cov9 [n_landmarks][9]
    CycleCovHost* cov_host = nullptr;
    CycleCovState cov;
  } cyc;
  // ctvio_odometry_checkpoint / ctvio_odometry_restore (checkpoint.cu): the blob's device and pinned staging, the
  // checksum's per-CTA partial sums and ticket, and the restore's verdict (pinned + mapped).  Scratch only: a restore
  // writes the engine's run only after the verdict passed.
  struct CkptWs {
    DevBuf<unsigned char> stage;
    DevBuf<unsigned long long> partial;
    DevBuf<int32_t> ticket;        // zeroed once; the last CTA of every launch resets it
    unsigned char* h_stage = nullptr;
    size_t h_cap = 0;
    int32_t* h_verdict = nullptr;
  } ckpt;
  int n_marg_img = -1;  // marginalized image factors of the last ctvio_marginalize (-1: pos_cam / pos_lm / marg_img not built)

  // multi-GPU
  void* nccl_comm = nullptr;
  int rank = 0, world = 1;
  bool shard_checked = false;  // landmark ownership verified for the current factor set

  int64_t launches = 0;

  ProblemDims dims() const {
    ProblemDims d;
    d.nK = nK; d.nB = nB; d.nL = nL;
    d.idx_bias0 = 6 * nK;
    d.idx_ld = 6 * nK + 6 * nB;
    d.np = d.idx_ld + 1;
    return d;
  }
  NormalEqPtrs ne(int b) {
    double* s = ne_slab[b].p;
    return NormalEqPtrs{s, s + off_gc, s + off_hl, s + off_gl, s + off_wld, s + off_W, &d_scal.p->cost_eval};
  }
  LandmarkLayout lml() { return LandmarkLayout{d_lo.p, d_hi.p, d_woff.p}; }
};

namespace ctvio::host {

// RAII: route this thread's uploads through the engine's arena for the duration of one C-ABI call
struct ArenaScope {
  PinnedArena* prev;
  explicit ArenaScope(ctvio_engine* e) : prev(g_arena) {
    if (e->stream && cudaStreamQuery(e->stream) == cudaSuccess) e->arena.rewind();  // idle: nothing reads the arena any more
    else cudaGetLastError();
    g_arena = &e->arena;
  }
  ~ArenaScope() { g_arena = prev; }
};

// n elements from the device to the host on the engine stream, counted in d2h_bytes; no synchronisation
template <class T>
int copy_to_host(ctvio_engine* e, T* dst, const T* src, size_t n = 1) {
  CUDA_OK(cudaMemcpyAsync(dst, src, n * sizeof(T), cudaMemcpyDeviceToHost, e->stream));
  e->d2h_bytes += n * sizeof(T);
  return CTVIO_OK;
}

// n elements of a kernel's small result, back to the host at the end of the call
template <class T>
int read_result(ctvio_engine* e, T* dst, const T* src, size_t n = 1) {
  if (const int rc = copy_to_host(e, dst, src, n)) return rc;
  CUDA_OK(stream_sync(e->stream));
  return CTVIO_OK;
}

inline int ensure_table(ctvio_engine* e) {
  if (!e->table_valid) {
    e->launches += launch_knot_table(e->x[e->cur].ptrs(), e->nK, e->stream);
    e->table_valid = true;
  }
  return CTVIO_OK;
}

// resident.cu: the resident feature table's arrays, at full size, on first use
int ensure_feature_table(ctvio_engine* e);
// odometry.cu: ctvio_odometry_start's option checks (also applied to a checkpoint's options by ctvio_odometry_restore)
int check_cycle_options(const ctvio_cycle_options* o);

// structure.cu: the structure build of the image-factor set, on the device or on the host (T: tiles per side of the
// reduced system).  structure_build_device reads back the one count block; schur_lists_device fills the K4 lists it sized.
int structure_build_device(ctvio_engine* e, int T);
int schur_lists_device(ctvio_engine* e, int T);
int structure_build_host(ctvio_engine* e);
int schur_lists_host(ctvio_engine* e, int T);
// ctvio_marginalize's image part: knot bitmask, counts, marg_img and the landmarks' ranks (pos_lm, -1: none), the last
// two in e->mws (device; offset_pos_lm_device adds the base) or in the host vectors
int marg_discover_device(ctvio_engine* e, std::vector<uint32_t>& knots, int& n_marg, int& n_rho);
int offset_pos_lm_device(ctvio_engine* e, int base);
int marg_discover_host(ctvio_engine* e, std::vector<uint32_t>& knots, int& n_marg, int& n_rho,
                       std::vector<int32_t>& marg_img, std::vector<int32_t>& pos_lm);
// sharded mode: per-landmark owned flags (hi > 0 of the built structure) into either buffer (may be null)
int owned_flags_device(ctvio_engine* e, double* as_double, uint8_t* as_byte);

// prior.cu: prepare()'s prior stage, and the active prior as the factor kernels see it
int prepare_prior(ctvio_engine* e);
PriorPtrs prior_ptrs(ctvio_engine* e);

// engine.cu, used by the LM driver in solve.cu
int prepare(ctvio_engine* e);  // structures of the factor set, built by structure.cu and the stages of engine.cu
// first knot of the spline segment of an evaluation time; its padded window [first, last] (false: outside the spline)
int knot_window_first(const ctvio_engine* e, int64_t t);
bool knot_window(const ctvio_engine* e, int64_t t, int& first, int& last);
void evaluate(ctvio_engine* e, int xb, int nb, bool full, bool reset_cost = true);
int read_scalars(ctvio_engine* e, bool published = false);
LinearLaunch linear_launch(ctvio_engine* e, int nb);
int refresh_mirror(ctvio_engine* e);
int alloc_state(ctvio_engine* e, DevState& s);
// bodies of entry points the odometry cycle (odometry.cu) runs without their trailing stream synchronisation
int add_bias_factors_device(ctvio_engine* e, int n, const int32_t* ni, const int32_t* nj, const double* d_sqrt_info6,
                            const int32_t* marg);
int adopt_prior_body(ctvio_engine* e, bool keep_new_prior);
int ingest_feature_cloud_body(ctvio_engine* e, int32_t slot, int64_t t_ns, int32_t n, const float* points, const float* ch_id,
                              const float* ch_v, bool sync);
int ingest_imu_body(ctvio_engine* e, int32_t n, const void* records, int32_t stride, int32_t off_gyro, int32_t off_accel,
                    int64_t drop_before_ns, bool sync, int* first_new);
// ctvio_feature_table_map; with point_cov9 (mapped host memory) the kernel also writes each point's covariance there,
// gathered from lm_cov9 [n_cov][9] by the entry's number (feature_table_map_kernel<true>)
int feature_table_map_body(ctvio_engine* e, int32_t n_frames, const int32_t* frame_slots, int32_t window_size,
                           int32_t capacity, double* xyz_world, int32_t* feature_id, uint8_t* in_margin_cloud,
                           int32_t* n_points, double* cam_q_xyzw, double* cam_p_xyz, const double* lm_cov9, int32_t n_cov,
                           double* point_cov9);
// covariance.cu, for the odometry cycle: Sigma with the knots <= gauge_knot held constant and its projections enqueued
// on the engine stream without a host wait, the rank test's inputs published to e->cyc.cov_host->pub (the cycle reads
// them after its next synchronisation, rank_test).  pose / rel / points: the TF pose at e->cyc.cov.pose_t, the
// consecutive frame pairs of e->cyc.cov.frame_t, the window's landmarks.
int cycle_covariance_enqueue(ctvio_engine* e, int gauge_knot, bool pose, bool rel, bool points);
const double* cycle_point_covariances(ctvio_engine* e);  // [n_lm][9] in the solved window's numbering, on the device
// the rank test of a published block, after a synchronisation: CTVIO_OK, or the error the covariance calls return for
// the same inputs (the evaluation's, or CTVIO_ERR_STATE "<who>: rank deficient"; message in *why)
int rank_test(const LmPublished& pub, const char* who, std::string* why);
// the ranges the covariance calls check (the range ctvio_query_trajectory accepts): the times t[0 .. n) lie inside the
// spline; every frame time of a slot the feature table holds (the anchors of its landmarks) lies inside the spline
bool times_inside(const SplineParams& sp, int n, const int64_t* t);
bool held_frames_inside(ctvio_engine* e);

}  // namespace ctvio::host
