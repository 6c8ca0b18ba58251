// Host side of the CUDA engine: C-ABI of include/ctvio.h, problem preprocessing (frame-pair groups,
// landmark ranges, Schur batches), device-resident window state and the LM trust-region driver.
//
// The driver restates Ceres 1.14's TrustRegionMinimizer / LevenbergMarquardtStrategy semantics that
// the reference gets from ceres::Solve (trajectory_estimator.cpp:367-408; SURVEY.md Appendix B):
// Jacobi scaling fixed at iteration 0, D^2 = clamp(diag)/mu, rho = dcost/dmodel accepted above 1e-3,
// mu <- mu / max(1/3, 1-(2rho-1)^3) on success, mu <- mu/f, f <- 2f on failure, function / parameter
// tolerances, Armijo projected line search when the line delay has bounds.
// GPU-first differences from a port: every candidate point is evaluated with full Jacobians into a
// second normal-equation buffer (an accepted step costs no re-linearisation pass), all per-step
// quantities are reduced on the device, and the host reads back ONE 96-byte scalar block per step.
#include <cuda_runtime.h>

#include <algorithm>
#include <atomic>
#include <chrono>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <string>
#include <vector>

#include "../../include/ctvio.h"
#include "frontend.h"
#include "kernels.h"
#include "marginalize.h"
#include "poly_min.h"

using namespace ctvio;

namespace {

thread_local std::string g_err;
int fail(int code, const std::string& msg) {
  g_err = msg;
  return code;
}

#define CUDA_OK(call)                                                                                   \
  do {                                                                                                  \
    cudaError_t e_ = (call);                                                                            \
    if (e_ != cudaSuccess)                                                                              \
      return fail(CTVIO_ERR_CUDA, std::string(#call) + ": " + cudaGetErrorString(e_));                  \
  } while (0)

thread_local size_t g_upload_bytes = 0;  // bytes moved by DevBuf::upload (index tables etc.), see ctvio_transfer_stats

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
thread_local PinnedArena* g_arena = nullptr;  // arena of the engine whose C-ABI call is running on this thread

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
  cudaError_t upload(const std::vector<T>& h, cudaStream_t s) {
    cudaError_t e = reserve(h.size());
    if (e != cudaSuccess || h.empty()) return e;
    g_upload_bytes += h.size() * sizeof(T);
    return staged_h2d(p, h.data(), h.size() * sizeof(T), s);
  }
};

struct DevState {
  DevBuf<double> q, p, bias, rho, ld;
  DevBuf<KnotPair> tab;
  StatePtrs ptrs() { return StatePtrs{q.p, p.p, bias.p, rho.p, ld.p, tab.p}; }
};

struct HostImage { int64_t ti, tj; int32_t rowi, rowj; double pi[2], pj[2]; int32_t lm, marg; };
struct HostImu { int64_t t; double gyro[3], accel[3]; int32_t node, marg; };
struct HostBias { int32_t i, j; double s[6]; int32_t marg; };

}  // namespace

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
  bool use_tma = true;
  bool deterministic = false;   // ctvio_set_deterministic: ordered flushes, single stream (kernels.h)
  DevBuf<int32_t> d_ticket;     // [0] kernel flush ticket, [1] scalar flush ticket

  // sizes
  int nK = 0, nB = 0, nL = 0;
  bool have_knots = false, have_bias = false, have_rho = false;

  // state: two buffers (current / candidate) + snapshot
  DevState x[2], snap;
  DevState xs;                 // third state buffer of the pipelined LM driver (swapped into x[] when it ends up current)
  DevBuf<LmPublished> d_pubstage;  // device staging copy of the published block (forwarded to h_pub from stream2)
  DevBuf<LmDecision> d_dec;    // device-side step decision (accept, next radius) read by the speculated linear solve
  cudaEvent_t ev_iter = nullptr;  // recorded behind the last kernel of every LM step (before anything speculative)
  bool speculate = true;       // CTVIO_NO_SPECULATION=1 switches the pipelined driver off
  bool staged_publish = false; // CTVIO_STAGED_PUBLISH=1: the scalar block reaches the host through a device staging copy
                               // forwarded from stream2 (measured: no gain - off by default)
  DevState& state(int i) { return i < 2 ? x[i] : xs; }
  int cur = 0;
  bool table_valid = false;

  // factors (host copies in caller order)
  std::vector<HostImage> img;
  std::vector<HostImu> imu;
  std::vector<HostBias> biasf;
  bool structure_dirty = true;

  // device factor arrays
  DevBuf<longlong2> d_img_t;
  DevBuf<double2> d_img_pi, d_img_pj;
  DevBuf<int4> d_img_meta;
  DevBuf<int32_t> d_img_orig;
  DevBuf<VisualItem> d_items;
  int n_items = 0;
  std::vector<int32_t> img_order;  // sorted position -> original index
  std::vector<int32_t> img_li, img_lj;    // ... and the last knot of those windows
  std::vector<int32_t> img_wi0, img_wj0;  // first knot of the padded anchor / observation window per factor (caller order)
  std::vector<VisualItem> h_items;        // K1 work items (one per chunk of a frame-pair group)
  std::vector<int32_t> imu_order;
  DevBuf<longlong2> d_imu_t;
  DevBuf<double2> d_imu_ga;
  DevBuf<ImuItem> d_imu_items;
  DevBuf<int32_t> d_imu_orig;
  int n_imu_items = 0;
  DevBuf<int2> d_bf_ij;
  DevBuf<double> d_bf_s;

  // landmark layout / schur batches
  std::vector<int32_t> h_lo, h_hi;
  std::vector<int64_t> h_woff;
  DevBuf<int32_t> d_lo, d_hi;
  DevBuf<SchurEntry> d_schur_list;
  DevBuf<int64_t> d_woff;
  DevBuf<SchurTileItem> d_schur_items;
  DevBuf<double> d_lis, d_lc;
  int n_schur_items = 0;
  DevBuf<uint8_t> d_cmask, d_active;
  std::vector<uint8_t> h_cmask, h_active;

  // normal equations (two buffers, each one slab: A | gc | hl | gl | wld | W)
  DevBuf<double> ne_slab[2];
  size_t ne_slab_len = 0;
  size_t off_gc = 0, off_hl = 0, off_gl = 0, off_wld = 0, off_W = 0;
  // linear system
  DevBuf<double> d_M, d_Linv, d_y, d_sc, d_sl, d_hh, d_dc, d_dl, d_rho_sync, d_chol_part;
  DevBuf<int32_t> d_chol_flags;
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
  // wire-format ingestion (frontend.cu): resident per-frame feature tables, resident IMU table
  static constexpr int kFrameSlots = 16, kFrameCap = 1024;
  DevBuf<ctvio::FrameFeature> d_frames;   // [kFrameSlots][kFrameCap]
  DevBuf<int64_t> d_frame_t;              // [kFrameSlots]
  DevBuf<float> d_cloud_stage;            // staging for one message (5 floats per point... points 3 + id + v)
  int64_t h_frame_t[16] = {0};
  int32_t h_frame_n[16] = {0};
  std::vector<ctvio::FactorDesc> img_desc;  // parallel to img when the factors came from the resident tables
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
  DevBuf<int32_t> d_tri_idx;  // ctvio_triangulate: start frames | observation offsets
  // marginalization workspace (K7), kept across windows: allocation / free costs more than the kernels
  struct MargWs {
    DevBuf<int32_t> pos_cam, pos_lm, prior_pos, marg_img, marg_imu;
    DevBuf<int2> bij;
    DevBuf<double> eig_scratch, Jrow, bs, A, b, Amm, V, ev, Vs, Ainv, T, Ap, bp, Ap2, V2, ev2, vb, J, r;
  } mws;

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

namespace {

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

// enqueue the device -> pinned-host copies of the whole state (the caller synchronises the stream afterwards)
int refresh_mirror(ctvio_engine* e, cudaStream_t on = nullptr) {
  const size_t need = 4 * size_t(e->nK) + kPStride * size_t(e->nK) + 6 * size_t(std::max(e->nB, 1)) + size_t(std::max(e->nL, 1)) + 8;
  if (need > e->h_mirror_cap) {
    if (e->h_mirror) cudaFreeHost(e->h_mirror);
    e->h_mirror = nullptr;
    e->h_mirror_cap = 0;
    if (cudaHostAlloc(reinterpret_cast<void**>(&e->h_mirror), (2 * need) * sizeof(double), cudaHostAllocDefault) != cudaSuccess) {
      cudaGetLastError();
      e->mirror_valid = false;
      return CTVIO_OK;  // the getters fall back to direct copies
    }
    e->h_mirror_cap = 2 * need;
  }
  DevState& x = e->x[e->cur];
  double* m = e->h_mirror;
  cudaStream_t st = on ? on : e->stream;
  CUDA_OK(cudaMemcpyAsync(m, x.q.p, 4 * size_t(e->nK) * sizeof(double), cudaMemcpyDeviceToHost, st));
  m += 4 * size_t(e->nK);
  CUDA_OK(cudaMemcpyAsync(m, x.p.p, kPStride * size_t(e->nK) * sizeof(double), cudaMemcpyDeviceToHost, st));
  m += kPStride * size_t(e->nK);
  if (e->nB) CUDA_OK(cudaMemcpyAsync(m, x.bias.p, 6 * size_t(e->nB) * sizeof(double), cudaMemcpyDeviceToHost, st));
  m += 6 * size_t(std::max(e->nB, 1));
  if (e->nL) CUDA_OK(cudaMemcpyAsync(m, x.rho.p, size_t(e->nL) * sizeof(double), cudaMemcpyDeviceToHost, st));
  m += size_t(std::max(e->nL, 1));
  CUDA_OK(cudaMemcpyAsync(m, x.ld.p, sizeof(double), cudaMemcpyDeviceToHost, st));
  e->mirror_valid = true;  // valid once the caller has synchronised
  return CTVIO_OK;
}

int knot_window_first(const ctvio_engine* e, int64_t t) {
  int64_t s = (t - e->cfg.t0_ns) / e->cfg.dt_ns;
  return int(s);
}

// padded window [first, last] of an evaluation time (se3_spline.h:463-503), clamped to the spline
bool knot_window(const ctvio_engine* e, int64_t t, int& first, int& last) {
  const int64_t maxt = e->cfg.t0_ns + int64_t(e->nK - 3) * e->cfg.dt_ns;
  if (t < e->cfg.t0_ns || t >= maxt) return false;
  const int smax = e->nK - 4;
  const int s1 = knot_window_first(e, t);
  int64_t t2 = t + e->cfg.rs_padding_ns;
  int s2 = (t2 >= maxt) ? smax : int((t2 - e->cfg.t0_ns) / e->cfg.dt_ns);
  if (s2 > s1 + 1) return false;  // padding wider than one knot interval is not supported by the 5-knot window
  first = s1;
  last = std::min(s2 + 3, e->nK - 1);
  return true;
}

int prepare_prior(ctvio_engine* e);
int fetch_new_prior(ctvio_engine* e);

// Build every host-side structure that depends on the factor set / sizes and upload it.
int prepare(ctvio_engine* e) {
  if (!e->have_knots) return fail(CTVIO_ERR_STATE, "knots have not been set");
  ArenaScope arena(e);
  static const bool prep_timing = std::getenv("CTVIO_PREP_TIMING") != nullptr;
  auto tp0 = std::chrono::steady_clock::now();
  auto lap = [&](const char* what) {
    if (!prep_timing) return;
    auto t = std::chrono::steady_clock::now();
    std::fprintf(stderr, "[prepare] %-22s %7.1f us\n", what, std::chrono::duration<double, std::micro>(t - tp0).count());
    tp0 = t;
  };
  if (e->nK < 4) return fail(CTVIO_ERR_STATE, "need at least 4 knots");
  if (!e->have_bias) { e->nB = 0; }
  cudaStream_t st = e->stream;
  const ProblemDims d = e->dims();
  if (e->structure_dirty) {
    e->shard_checked = false;
    // ---- image factors: frame-pair groups ----
    const int n = int(e->img.size());
    std::vector<int32_t>&wi0 = e->img_wi0, &wj0 = e->img_wj0;
    wi0.resize(n); wj0.resize(n);
    e->img_li.resize(n); e->img_lj.resize(n);
    e->h_lo.assign(e->nL, INT32_MAX);
    e->h_hi.assign(e->nL, 0);
    // the image factors of a window carry a dozen distinct frame times: the padded knot window of a time (two 64-bit
    // divisions) is looked up in a small direct-mapped cache
    struct WinCache { int64_t t = INT64_MIN; int f = 0, l = 0; bool ok = false; } wc[64];
    auto window_of = [&](int64_t t, int& f, int& l) {
      WinCache& c = wc[size_t(uint64_t(t) * 0x9E3779B97F4A7C15ull >> 58)];
      if (c.t != t) { c.t = t; c.ok = knot_window(e, t, c.f, c.l); }
      f = c.f; l = c.l;
      return c.ok;
    };
    for (int k = 0; k < n; ++k) {
      const HostImage& o = e->img[k];
      int f0, l0, f1, l1;
      if (!window_of(o.ti, f0, l0) || !window_of(o.tj, f1, l1))
        return fail(CTVIO_ERR_TIME_RANGE, "image factor time (+ rolling-shutter padding) outside the spline");
      if (o.lm < 0 || o.lm >= e->nL) return fail(CTVIO_ERR_INVALID, "landmark index out of range");
      wi0[k] = f0; wj0[k] = f1;
      e->img_li[k] = l0; e->img_lj[k] = l1;
      e->h_lo[o.lm] = std::min(e->h_lo[o.lm], 6 * std::min(f0, f1));
      e->h_hi[o.lm] = std::max(e->h_hi[o.lm], 6 * (std::max(l0, l1) + 1));
    }
    e->img_order.resize(n);
    {
      // order: (frame-pair group, landmark, position).  The reference's feature loop hands the factors over landmark by
      // landmark (trajectory_manager.cpp:360-385), so they usually arrive sorted by landmark already: then a STABLE
      // counting sort by group is the whole job (O(n), this runs once per window inside the end-to-end time); any other
      // input order takes the general key sort.
      bool lm_sorted = true;
      for (int k = 1; k < n && lm_sorted; ++k) lm_sorted = e->img[k - 1].lm <= e->img[k].lm;
      const size_t nKk = size_t(e->nK) + 1;
      if (lm_sorted && nKk * nKk <= (size_t(1) << 22)) {
        std::vector<int32_t> start(nKk * nKk + 1, 0);
        for (int k = 0; k < n; ++k) ++start[size_t(wi0[k]) * nKk + size_t(wj0[k]) + 1];
        for (size_t g = 1; g < start.size(); ++g) start[g] += start[g - 1];
        for (int k = 0; k < n; ++k) e->img_order[start[size_t(wi0[k]) * nKk + size_t(wj0[k])]++] = k;
      } else {
        std::vector<uint64_t> key(n);
        const uint64_t nLl = uint64_t(std::max(e->nL, 1));
        if (uint64_t(nKk) * nKk * nLl < (uint64_t(1) << 40) && uint64_t(n) < (uint64_t(1) << 24)) {
          for (int k = 0; k < n; ++k)
            key[k] = (((uint64_t(wi0[k]) * nKk + uint64_t(wj0[k])) * nLl + uint64_t(e->img[k].lm)) << 24) | uint64_t(k);
          std::sort(key.begin(), key.end());
          for (int k = 0; k < n; ++k) e->img_order[k] = int32_t(key[k] & 0xffffffu);
        } else {
          for (int k = 0; k < n; ++k) e->img_order[k] = k;
          std::stable_sort(e->img_order.begin(), e->img_order.end(), [&](int a, int b) {
            if (wi0[a] != wi0[b]) return wi0[a] < wi0[b];
            if (wj0[a] != wj0[b]) return wj0[a] < wj0[b];
            return e->img[a].lm < e->img[b].lm;
          });
        }
      }
    }
    std::vector<longlong2> ht(n);
    std::vector<double2> hpi(n), hpj(n);
    std::vector<int4> hm(n);
    for (int k = 0; k < n; ++k) {
      const HostImage& o = e->img[e->img_order[k]];
      ht[k] = make_longlong2(o.ti, o.tj);
      hpi[k] = make_double2(o.pi[0], o.pi[1]);
      hpj[k] = make_double2(o.pj[0], o.pj[1]);
      hm[k] = make_int4(o.rowi, o.rowj, o.lm, o.marg);
    }
    lap("image windows + sort");
    // work items: chunks of one group; chunk size adapts so that small problems still spread over the SMs
    // (a group is split into equal chunks of at most `cap` observations, cap a multiple of the 128-observation round)
    // one evaluation round (<= 128 observations, a lane pair each) per CTA: the round is latency bound whatever its
    // fill, so a group is cut into EQUAL chunks of at most one round (263 observations -> 3 x 88, not 128 + 128 + 7)
    // and every chunk gets its own CTA; CTVIO_VIS_CAP overrides (multiples of 128) for experiments
    int cap = kVisObsPerRound;
    if (const char* env = std::getenv("CTVIO_VIS_CAP")) cap = std::max(kVisObsPerRound, std::atoi(env) / kVisObsPerRound * kVisObsPerRound);
    std::vector<VisualItem>& items = e->h_items;
    items.clear();
    for (int k = 0; k < n;) {
      const int a = e->img_order[k];
      int end = k;
      while (end < n && wi0[e->img_order[end]] == wi0[a] && wj0[e->img_order[end]] == wj0[a]) ++end;
      const int cnt = end - k;
      // a few stragglers beyond a full round are cheaper as their own small item than as an extra round
      const int nchunks = (cnt + cap - 1) / cap;
      const int per = (cnt + nchunks - 1) / nchunks;
      for (int s = k; s < end; s += per) items.push_back(VisualItem{s, std::min(per, end - s), wi0[a], wj0[a]});
      k = end;
    }
    e->n_items = int(items.size());
    if (!e->img_desc.empty()) {
      // factors added from the resident frame tables: only the sorted 16-byte descriptors go up, the SoA payload is
      // gathered on the device
      std::vector<ctvio::FactorDesc> sd(n);
      for (int k = 0; k < n; ++k) sd[k] = e->img_desc[e->img_order[k]];
      CUDA_OK(e->d_img_desc.upload(sd, st));
      CUDA_OK(e->d_img_t.reserve(n)); CUDA_OK(e->d_img_pi.reserve(n)); CUDA_OK(e->d_img_pj.reserve(n)); CUDA_OK(e->d_img_meta.reserve(n));
      ctvio::GatherFactorsArgs ga;
      ga.n = n; ga.desc = e->d_img_desc.p; ga.table = e->d_frames.p; ga.frame_t = e->d_frame_t.p;
      ga.frame_cap = ctvio_engine::kFrameCap;
      ga.t = e->d_img_t.p; ga.pi = e->d_img_pi.p; ga.pj = e->d_img_pj.p; ga.meta = e->d_img_meta.p;
      e->launches += ctvio::launch_gather_factors(ga, st);
    } else {
      CUDA_OK(e->d_img_t.upload(ht, st));
      CUDA_OK(e->d_img_pi.upload(hpi, st));
      CUDA_OK(e->d_img_pj.upload(hpj, st));
      CUDA_OK(e->d_img_meta.upload(hm, st));
    }
    CUDA_OK(e->d_img_orig.upload(e->img_order, st));
    CUDA_OK(e->d_items.upload(items, st));

    lap("image arrays + upload");
    // ---- landmark layout ----
    e->h_woff.assign(e->nL + 1, 0);
    for (int l = 0; l < e->nL; ++l) {
      if (e->h_hi[l] == 0) e->h_lo[l] = 0;
      e->h_woff[l + 1] = e->h_woff[l] + (e->h_hi[l] - e->h_lo[l]);
    }
    CUDA_OK(e->d_lo.upload(e->h_lo, st));
    CUDA_OK(e->d_hi.upload(e->h_hi, st));
    CUDA_OK(e->d_woff.upload(e->h_woff, st));
    lap("landmark layout");
    // ---- imu / bias factors ----
    const int ni = int(e->imu.size());
    std::vector<longlong2> it(ni);
    std::vector<double2> iga(3 * size_t(ni));
    const int64_t maxt = e->cfg.t0_ns + int64_t(e->nK - 3) * e->cfg.dt_ns;
    std::vector<int32_t>& imu_order = e->imu_order;
    imu_order.assign(ni, 0);
    std::vector<int32_t> imu_s(ni);
    for (int k = 0; k < ni; ++k) {
      const HostImu& o = e->imu[k];
      if (o.t < e->cfg.t0_ns || o.t >= maxt) return fail(CTVIO_ERR_TIME_RANGE, "imu time outside the spline");
      if (o.node < 0 || o.node >= e->nB) return fail(CTVIO_ERR_INVALID, "bias node out of range");
      imu_order[k] = k;
      imu_s[k] = knot_window_first(e, o.t);
    }
    // runs of samples sharing (start knot, bias node) -> one CTA each
    std::stable_sort(imu_order.begin(), imu_order.end(), [&](int a, int b) {
      if (imu_s[a] != imu_s[b]) return imu_s[a] < imu_s[b];
      return e->imu[a].node < e->imu[b].node;
    });
    std::vector<ImuItem> imu_items;
    for (int k = 0; k < ni; ++k) {
      const HostImu& o = e->imu[imu_order[k]];
      it[k] = make_longlong2(o.t, o.node);
      iga[3 * k] = make_double2(o.gyro[0], o.gyro[1]);
      iga[3 * k + 1] = make_double2(o.gyro[2], o.accel[0]);
      iga[3 * k + 2] = make_double2(o.accel[1], o.accel[2]);
      const int s = imu_s[imu_order[k]];
      if (imu_items.empty() || imu_items.back().s != s || imu_items.back().node != o.node ||
          imu_items.back().count >= kImuMaxPerItem)
        imu_items.push_back(ImuItem{k, 0, s, o.node});
      imu_items.back().count++;
    }
    e->n_imu_items = int(imu_items.size());
    CUDA_OK(e->d_imu_items.upload(imu_items, st));
    CUDA_OK(e->d_imu_orig.upload(imu_order, st));
    if (!e->imu_src.empty()) {
      // samples taken from the resident IMU table: (table index, bias node) pairs go up, the payload is gathered
      std::vector<int2> src(ni);
      for (int k = 0; k < ni; ++k) src[k] = make_int2(e->imu_src[imu_order[k]], e->imu[imu_order[k]].node);
      CUDA_OK(e->d_imu_src.upload(src, st));
      CUDA_OK(e->d_imu_t.reserve(ni)); CUDA_OK(e->d_imu_ga.reserve(3 * size_t(ni)));
      e->launches += ctvio::launch_gather_imu(e->d_imu_src.p, ni, e->d_imu_tab_t.p, e->d_imu_tab_ga.p, e->d_imu_t.p, e->d_imu_ga.p, st);
    } else {
      CUDA_OK(e->d_imu_t.upload(it, st));
      CUDA_OK(e->d_imu_ga.upload(iga, st));
    }
    const int nb = int(e->biasf.size());
    std::vector<int2> bij(nb);
    std::vector<double> bs(6 * size_t(nb));
    for (int k = 0; k < nb; ++k) {
      const HostBias& o = e->biasf[k];
      if (o.i < 0 || o.i >= e->nB || o.j < 0 || o.j >= e->nB) return fail(CTVIO_ERR_INVALID, "bias node out of range");
      bij[k] = make_int2(o.i, o.j);
      for (int c = 0; c < 6; ++c) bs[6 * k + c] = o.s[c];
    }
    CUDA_OK(e->d_bf_ij.upload(bij, st));
    CUDA_OK(e->d_bf_s.upload(bs, st));

    lap("imu / bias");
    // ---- buffers ----
    const size_t np = size_t(d.np);
    e->off_gc = np * np;
    e->off_hl = e->off_gc + np;
    e->off_gl = e->off_hl + e->nL;
    e->off_wld = e->off_gl + e->nL;
    e->off_W = e->off_wld + e->nL;
    e->ne_slab_len = e->off_W + size_t(e->h_woff[e->nL]);
    for (int b = 0; b < 2; ++b) CUDA_OK(e->ne_slab[b].reserve(e->ne_slab_len));
    e->npad = ((d.np + kCholNB - 1) / kCholNB) * kCholNB;
    CUDA_OK(e->d_M.reserve(size_t(e->npad) * e->npad + 3 * size_t(e->npad)));  // M | rhs | diagA | yf (all-reduce slab)
    if (chol_dag_lpub_len(e->npad) > e->d_Linv.cap || chol_dag_part_len(e->npad) > e->d_chol_part.cap || e->linv_npad != e->npad) {
      CUDA_OK(e->d_Linv.reserve(chol_dag_lpub_len(e->npad)));
      CUDA_OK(e->d_chol_part.reserve(chol_dag_part_len(e->npad)));
      e->launches += launch_chol_dag_init(e->d_Linv.p, e->d_chol_part.p, e->npad, e->stream);  // message words start as sentinels
      e->linv_npad = e->npad;
      e->chol_seq = 0;
    }
    lap("buffers");
    {
      // ---- K4 work items: per 64x64 tile (ti >= tj) of the reduced system the landmarks whose knot-dim range
      // [lo, hi) touches both blocks, cut into parts of `part` landmarks so that about two waves of CTAs exist
      // whatever the window size (the line-delay row / column is a matrix-vector product done by the diagonal tiles) ----
      const int T = e->npad / kCholNB;
      std::vector<std::vector<int32_t>> lists(size_t(T) * (T + 1) / 2);
      std::vector<int32_t> order;
      for (int l = 0; l < e->nL; ++l)
        if (e->h_hi[l] > 0) order.push_back(l);
      std::stable_sort(order.begin(), order.end(), [&](int a, int b) {
        if (e->h_lo[a] != e->h_lo[b]) return e->h_lo[a] < e->h_lo[b];
        return e->h_hi[a] < e->h_hi[b];
      });
      size_t total = 0;
      for (int l : order) {
        int blocks[64], nbk = 0;
        const int b0 = e->h_lo[l] / kCholNB, b1 = (e->h_hi[l] - 1) / kCholNB;
        for (int b = b0; b <= b1 && nbk < 63; ++b) blocks[nbk++] = b;
        for (int x = 0; x < nbk; ++x)
          for (int y = 0; y <= x; ++y) {
            lists[size_t(blocks[x]) * (blocks[x] + 1) / 2 + blocks[y]].push_back(l);
            ++total;
          }
      }
      const int n_sm = device_sm_count();
      const int part = std::max(32, int((total / size_t(2 * n_sm) + 31) / 32) * 32);
      std::vector<SchurTileItem> items;
      std::vector<SchurEntry> flat;
      flat.reserve(total);
      for (int ti = 0; ti < T; ++ti)
        for (int tj = 0; tj <= ti; ++tj) {
          const std::vector<int32_t>& v = lists[size_t(ti) * (ti + 1) / 2 + tj];
          for (size_t s0 = 0; s0 < v.size(); s0 += part)
            items.push_back(SchurTileItem{ti, tj, int32_t(flat.size() + s0), int32_t(std::min(v.size() - s0, size_t(part)))});
          for (int32_t l : v) flat.push_back(SchurEntry{l, e->h_lo[l], e->h_hi[l], 0, e->h_woff[l]});
        }
      e->n_schur_items = int(items.size());
      CUDA_OK(e->d_schur_list.upload(flat, st));
      CUDA_OK(e->d_schur_items.upload(items, st));
      CUDA_OK(e->d_lis.reserve(e->nL));
      CUDA_OK(e->d_lc.reserve(e->nL));
    }
    lap("schur lists");
    if (chol_dag_flags_len(e->npad) > e->d_chol_flags.cap) {
      CUDA_OK(e->d_chol_flags.reserve(chol_dag_flags_len(e->npad)));
      CUDA_OK(cudaMemsetAsync(e->d_chol_flags.p, 0, e->d_chol_flags.cap * sizeof(int32_t), e->stream));
    }
    CUDA_OK(e->d_y.reserve(e->npad));
    CUDA_OK(e->d_sc.reserve(np));
    CUDA_OK(e->d_sl.reserve(e->nL));
    CUDA_OK(e->d_hh.reserve(e->nL));
    CUDA_OK(e->d_dc.reserve(np));
    CUDA_OK(e->d_dl.reserve(e->nL));
    if (e->nL > 0) CUDA_OK(cudaMemsetAsync(e->d_hh.p, 0, sizeof(double) * e->nL, st));
    e->prior_dirty = true;
  }
  lap("reserves");
  // ---- masks (depend on options + structure) ----
  if (e->structure_dirty || e->masks_dirty) {
    e->h_cmask.assign(d.np, 0);
    for (int k = 0; k < e->nK; ++k)
      if (e->opt.lock_traj || (e->opt.fixed_knot_index >= 0 && k <= e->opt.fixed_knot_index))
        for (int c = 0; c < 6; ++c) e->h_cmask[6 * k + c] = 1;  // trajectory_estimator.cpp:134-138
    for (int b = 0; b < e->nB; ++b)
      for (int c = 0; c < 3; ++c) {
        if (e->opt.lock_wb) e->h_cmask[d.idx_bias0 + 6 * b + c] = 1;
        if (e->opt.lock_ab) e->h_cmask[d.idx_bias0 + 6 * b + 3 + c] = 1;
      }
    if (e->opt.fix_ld) e->h_cmask[d.idx_ld] = 1;
    std::vector<uint8_t> touched(d.np + e->nL, 0);
    auto mark = [&](int f, int l) {
      for (int k = f; k <= l; ++k)
        for (int c = 0; c < 6; ++c) touched[6 * k + c] = 1;
    };
    // image factors: a window of a dozen frames has a few dozen distinct padded knot windows [first, last]; each is
    // marked once (the windows were computed by the structure pass above)
    {
      std::vector<uint8_t> seen(size_t(e->nK) * 8, 0);
      auto mark_once = [&](int f, int l) {
        uint8_t& sflag = seen[size_t(f) * 8 + size_t(l - f)];
        if (!sflag) { sflag = 1; mark(f, l); }
      };
      const size_t n = e->img.size();
      for (size_t k = 0; k < n; ++k) {
        mark_once(e->img_wi0[k], e->img_li[k]);
        mark_once(e->img_wj0[k], e->img_lj[k]);
        touched[d.np + e->img[k].lm] = 1;
      }
      if (n) touched[d.idx_ld] = 1;
    }
    for (const HostImu& o : e->imu) {
      const int s = knot_window_first(e, o.t);
      mark(s, s + 3);
      for (int c = 0; c < 6; ++c) touched[d.idx_bias0 + 6 * o.node + c] = 1;
    }
    for (const HostBias& o : e->biasf)
      for (int c = 0; c < 6; ++c) touched[d.idx_bias0 + 6 * o.i + c] = touched[d.idx_bias0 + 6 * o.j + c] = 1;
    if (e->prior.n > 0 && e->prior_enabled)
      for (size_t b = 0; b < e->prior.type.size(); ++b) {
        const int g = ctvio::prior_block_base(e->prior.type[b], e->prior.index[b], d.nK, d.nB);
        const int ls = (e->prior.type[b] == CTVIO_BLK_LD || e->prior.type[b] == CTVIO_BLK_RHO) ? 1 : 3;
        if (g >= 0) for (int c = 0; c < ls; ++c) touched[g + c] = 1;
      }
    e->h_active.assign(d.np + e->nL, 0);
    for (int i = 0; i < d.np; ++i) e->h_active[i] = touched[i] && !e->h_cmask[i];
    for (int l = 0; l < e->nL; ++l) e->h_active[d.np + l] = touched[d.np + l];
    CUDA_OK(e->d_cmask.upload(e->h_cmask, st));
    CUDA_OK(e->d_active.upload(e->h_active, st));
    e->masks_dirty = false;
  }
  lap("masks");
  e->structure_dirty = false;
  if (e->prior_dirty) {
    const int rc = prepare_prior(e);
    if (rc != CTVIO_OK) return rc;
  }
  return CTVIO_OK;
}

int prepare_prior(ctvio_engine* e) {
  const ProblemDims d = e->dims();
  const ctvio::PriorHost& pr = e->prior;
  e->prior_dirty = false;
  if (pr.n <= 0) return CTVIO_OK;
  cudaStream_t st = e->stream;
  std::vector<int32_t> col2g(pr.n, -1);
  for (size_t b = 0; b < pr.type.size(); ++b) {
    const int g = ctvio::prior_block_base(pr.type[b], pr.index[b], d.nK, d.nB);
    if (pr.type[b] == CTVIO_BLK_RHO) return fail(CTVIO_ERR_INVALID, "inverse-depth blocks cannot be part of a prior");
    if (g < 0) return fail(CTVIO_ERR_INVALID, "prior block index out of range");
    const int ls = pr.type[b] == CTVIO_BLK_LD ? 1 : 3;
    for (int c = 0; c < ls; ++c)
      if (!e->h_cmask[g + c]) col2g[pr.col[b] + c] = g + c;
  }
  if (!e->prior_on_device) {
    CUDA_OK(e->d_prior_J.upload(pr.J, st));
    CUDA_OK(e->d_prior_r.upload(pr.r, st));
    CUDA_OK(e->d_prior_x0.upload(pr.x0, st));
  }
  CUDA_OK(e->d_prior_type.upload(pr.type, st));
  CUDA_OK(e->d_prior_index.upload(pr.index, st));
  CUDA_OK(e->d_prior_col.upload(pr.col, st));
  CUDA_OK(e->d_prior_col2g.upload(col2g, st));
  CUDA_OK(e->d_prior_JtJ.reserve(size_t(pr.n) * pr.n));
  CUDA_OK(e->d_prior_dx.reserve(pr.n));
  CUDA_OK(e->d_prior_res.reserve(pr.n));
  CUDA_OK(cudaMemsetAsync(e->d_prior_dx.p, 0, size_t(pr.n) * sizeof(double), st));
  e->launches += ctvio::launch_gram(e->d_prior_J.p, pr.n, pr.n, e->d_prior_JtJ.p, st);
  return CTVIO_OK;
}

// make sure the host copy of the freshly marginalized prior exists (ctvio_get_prior; the device-to-device hand-over of
// ctvio_adopt_prior never needs it)
int fetch_new_prior(ctvio_engine* e) {
  ctvio::PriorHost& np_ = e->new_prior;
  if (e->new_prior_on_host || np_.n <= 0) return CTVIO_OK;
  np_.J.resize(size_t(np_.n) * np_.n);
  np_.r.resize(np_.n);
  np_.x0.resize(4 * np_.type.size());
  CUDA_OK(cudaMemcpyAsync(np_.J.data(), e->mws.J.p, np_.J.size() * sizeof(double), cudaMemcpyDeviceToHost, e->stream));
  CUDA_OK(cudaMemcpyAsync(np_.r.data(), e->mws.r.p, np_.r.size() * sizeof(double), cudaMemcpyDeviceToHost, e->stream));
  CUDA_OK(cudaMemcpyAsync(np_.x0.data(), e->d_newprior_x0.p, np_.x0.size() * sizeof(double), cudaMemcpyDeviceToHost, e->stream));
  CUDA_OK(cudaStreamSynchronize(e->stream));
  e->d2h_bytes += (np_.J.size() + np_.r.size() + np_.x0.size()) * sizeof(double);
  e->new_prior_on_host = true;
  return CTVIO_OK;
}

PriorPtrs prior_ptrs(ctvio_engine* e) {
  PriorPtrs p;
  std::memset(&p, 0, sizeof(p));
  p.n = e->prior_enabled ? e->prior.n : 0;
  if (p.n <= 0) return p;
  p.n_blocks = int(e->prior.type.size());
  p.J = e->d_prior_J.p; p.r = e->d_prior_r.p; p.JtJ = e->d_prior_JtJ.p;
  p.type = e->d_prior_type.p; p.index = e->d_prior_index.p; p.col = e->d_prior_col.p;
  p.x0 = e->d_prior_x0.p; p.col2g = e->d_prior_col2g.p;
  p.dx = e->d_prior_dx.p; p.res = e->d_prior_res.p;
  return p;
}

VisualLaunch visual_launch(ctvio_engine* e, int xb, int nb, double cauchy) {
  VisualLaunch v;
  v.obs = ImageObsPtrs{e->d_img_t.p, e->d_img_pi.p, e->d_img_pj.p, e->d_img_meta.p, int32_t(e->img.size())};
  v.items = e->d_items.p;
  v.n_items = e->n_items;
  v.st = e->state(xb).ptrs();
  v.ne = e->ne(nb);
  v.lm = e->lml();
  v.dims = e->dims();
  v.sp = e->sp;
  v.rig = e->rig;
  v.cauchy = cauchy;
  v.cmask = e->d_cmask.p;
  v.scal = e->d_scal.p;
  v.use_tma = e->use_tma;
  v.det_ticket = e->deterministic ? e->d_ticket.p : nullptr;
  return v;
}
ImuLaunch imu_launch(ctvio_engine* e, int xb, int nb) {
  ImuLaunch v;
  v.obs = ImuObsPtrs{e->d_imu_t.p, e->d_imu_ga.p, int32_t(e->imu.size())};
  v.items = e->d_imu_items.p;
  v.n_items = e->n_imu_items;
  v.st = e->state(xb).ptrs();
  v.ne = e->ne(nb);
  v.dims = e->dims();
  v.sp = e->sp;
  v.rig = e->rig;
  v.cmask = e->d_cmask.p;
  v.scal = e->d_scal.p;
  v.det_ticket = e->deterministic ? e->d_ticket.p : nullptr;
  return v;
}
SmallFactorsLaunch small_launch(ctvio_engine* e, int xb, int nb) {
  SmallFactorsLaunch v;
  v.bf = BiasFactorPtrs{e->d_bf_ij.p, e->d_bf_s.p, int32_t(e->biasf.size())};
  v.prior = prior_ptrs(e);
  v.st = e->state(xb).ptrs();
  v.ne = e->ne(nb);
  v.dims = e->dims();
  v.cmask = e->d_cmask.p;
  v.scal = e->d_scal.p;
  v.deterministic = e->deterministic ? 1 : 0;
  return v;
}
LinearLaunch linear_launch(ctvio_engine* e, int nb) {
  LinearLaunch a;
  a.dims = e->dims();
  a.ne = e->ne(nb);
  a.lm = e->lml();
  a.schur_list = e->d_schur_list.p;
  a.schur_items = e->d_schur_items.p;
  a.n_schur_items = e->n_schur_items;
  a.lis = e->d_lis.p; a.lc = e->d_lc.p;
  a.cmask = e->d_cmask.p;
  a.active = e->d_active.p;
  a.sc = e->d_sc.p; a.sl = e->d_sl.p;
  a.M = e->d_M.p; a.Linv = e->d_Linv.p; a.y = e->d_y.p;
  a.rhs = e->d_M.p + size_t(e->npad) * e->npad;
  a.diagA = a.rhs + e->npad;
  a.yf = a.diagA + e->npad;
  a.chol_part = e->d_chol_part.p; a.chol_flags = e->d_chol_flags.p; a.chol_seq = &e->chol_seq;
  a.sharded = e->world > 1 ? 1 : 0;
  a.hh = e->d_hh.p; a.dc = e->d_dc.p; a.dl = e->d_dl.p;
  a.npad = e->npad;
  a.scal = e->d_scal.p;
  a.go = nullptr;
  a.det_ticket = e->deterministic ? e->d_ticket.p : nullptr;
  return a;
}

// sharded mode: ONE all-gather of every rank's 8 scalars (sums AND maxima travel together), reduced in a fixed rank
// order by a one-thread kernel that also publishes the common block to mapped host memory (no copy + stream synchronise)
int allreduce_scalars(ctvio_engine* e, bool publish = false) {
  if (e->world <= 1) return CTVIO_OK;
  CUDA_OK(e->d_shard_scal.reserve(8 + 8 * size_t(e->world)));
  e->launches += ctvio::launch_shard_scalars_pack(e->d_scal.p, e->d_shard_scal.p, e->stream);
  std::string err;
  if (!ctvio::comm_allgather(e->nccl_comm, e->d_shard_scal.p, e->d_shard_scal.p + 8, 8, e->stream, &err))
    return fail(CTVIO_ERR_NCCL, err);
  e->launches += ctvio::launch_shard_scalars_reduce(e->d_shard_scal.p + 8, e->world, e->d_scal.p, publish ? e->h_pub : nullptr,
                                                    publish ? ++e->pub_seq : 0, e->stream);
  return CTVIO_OK;
}

// sharded mode: every rank must enter (or skip) the collectives of a solve together.  Sums a per-rank error flag; returns
// CTVIO_OK only if every rank reported local_rc == 0 (a failing rank keeps its own message).
int shard_consensus(ctvio_engine* e, int local_rc) {
  if (e->world <= 1) return local_rc;
  const std::string local_msg = g_err;
  cudaStream_t st = e->stream;
  CUDA_OK(e->d_tmp.reserve(16));
  const double flag = local_rc ? 1.0 : 0.0;
  double total = 0.0;
  CUDA_OK(cudaMemcpyAsync(e->d_tmp.p, &flag, sizeof(double), cudaMemcpyHostToDevice, st));
  std::string err;
  if (!ctvio::comm_allreduce_sum(e->nccl_comm, e->d_tmp.p, 1, st, &err)) return fail(CTVIO_ERR_NCCL, err);
  CUDA_OK(cudaMemcpyAsync(&total, e->d_tmp.p, sizeof(double), cudaMemcpyDeviceToHost, st));
  CUDA_OK(cudaStreamSynchronize(st));
  if (local_rc) return fail(local_rc, local_msg);
  if (total != 0.0) return fail(CTVIO_ERR_STATE, "another rank of the sharded solve failed before the first collective");
  return CTVIO_OK;
}

// sharded mode: the landmark prologue (hh, lis, lc) and the per-landmark Schur terms are formed from rank-local sums, so
// all observations of one landmark must live on ONE rank.  Checked once per structure change with one all-reduce of the
// per-landmark owner counts.
int shard_check_ownership(ctvio_engine* e) {
  if (e->world <= 1 || e->shard_checked) return CTVIO_OK;
  cudaStream_t st = e->stream;
  std::vector<double> owned(size_t(std::max(e->nL, 1)), 0.0);
  for (const HostImage& o : e->img) owned[o.lm] = 1.0;
  CUDA_OK(e->d_rho_sync.reserve(2 * size_t(std::max(e->nL, 1))));
  CUDA_OK(cudaMemcpyAsync(e->d_rho_sync.p, owned.data(), owned.size() * sizeof(double), cudaMemcpyHostToDevice, st));
  std::string err;
  if (!ctvio::comm_allreduce_sum(e->nccl_comm, e->d_rho_sync.p, owned.size(), st, &err)) return fail(CTVIO_ERR_NCCL, err);
  CUDA_OK(cudaMemcpyAsync(owned.data(), e->d_rho_sync.p, owned.size() * sizeof(double), cudaMemcpyDeviceToHost, st));
  CUDA_OK(cudaStreamSynchronize(st));
  for (int l = 0; l < e->nL; ++l)
    if (owned[l] > 1.0)
      return fail(CTVIO_ERR_INVALID, "sharded solve: landmark " + std::to_string(l) + " has observations on " +
                                         std::to_string(int(owned[l])) + " ranks (shard image factors by landmark)");
  e->shard_checked = true;
  return CTVIO_OK;
}

// the LM step: reduced system (+ all-reduce of [M | rhs | diagA] over NVLink in sharded mode), factor, solve
int lm_step(ctvio_engine* e, int nb, double radius, const ApplyLaunch* fused_apply = nullptr, const double* radius_dev = nullptr,
            const int32_t* go = nullptr) {
  LinearLaunch lin = linear_launch(e, nb);
  lin.go = go;
  cudaStream_t st = e->stream;
  if (e->deterministic) cudaMemsetAsync(e->d_ticket.p, 0, 2 * sizeof(int32_t), st);
  e->launches += launch_reduced_system(lin, radius, st, radius_dev);
  if (e->world > 1) {
    // one all-reduce of the lower-triangular tiles + rhs + diagonal (half the bytes of the dense slab), damping after it
    std::string err;
    const size_t count = ctvio::shard_pack_len(e->npad);
    CUDA_OK(e->d_shard_pack.reserve(count));
    e->launches += ctvio::launch_shard_pack(lin, e->d_shard_pack.p, st);
    if (!ctvio::comm_allreduce_sum(e->nccl_comm, e->d_shard_pack.p, count, st, &err)) return fail(CTVIO_ERR_NCCL, err);
    e->launches += ctvio::launch_shard_unpack(lin, e->d_shard_pack.p, radius, st);
  }
  e->launches += launch_factor_solve(lin, st);
  if (fused_apply) e->launches += launch_step_and_apply(lin, *fused_apply, st);
  else e->launches += launch_step_vectors(lin, st);
  return CTVIO_OK;
}

// one pass over all residual blocks at state buffer xb into normal-equation buffer nb
// reset_cost = false: cost_eval was already zeroed by scale_copy_kernel of the same LM step
void evaluate(ctvio_engine* e, int xb, int nb, bool full, bool reset_cost = true) {
  cudaStream_t st = e->stream;
  if (full) {
    if (e->slab_zeroed[nb]) {
      cudaStreamWaitEvent(st, e->ev_zero, 0);  // cleared on stream2 while the linear solve was running
      e->slab_zeroed[nb] = false;
    } else {
      cudaMemsetAsync(e->ne_slab[nb].p, 0, e->ne_slab_len * sizeof(double), st);
    }
  }
  if (reset_cost) cudaMemsetAsync(&e->d_scal.p->cost_eval, 0, sizeof(double), st);
  // fork: the (latency-bound) IMU + bias + prior kernels overlap the visual kernel on a second stream
  // sharded mode: IMU / bias / prior factors live on rank 0 only (every rank holds its own landmark shard)
  const bool fork = (e->rank == 0) && (!e->imu.empty() || !e->biasf.empty() || (e->prior.n > 0 && e->prior_enabled));
  if (e->deterministic) {
    // one stream, one kernel at a time, every kernel flushing in block order: every sum has ONE accumulation order
    cudaMemsetAsync(e->d_ticket.p, 0, 2 * sizeof(int32_t), st);
    e->launches += launch_visual(visual_launch(e, xb, nb, e->cfg.cauchy_solve), full, st);
    if (fork) {
      cudaMemsetAsync(e->d_ticket.p, 0, 2 * sizeof(int32_t), st);
      e->launches += launch_imu(imu_launch(e, xb, nb), full, st);
      e->launches += launch_small_factors(small_launch(e, xb, nb), full, st);
    }
    return;
  }
  // (streaming windows: K2 + K3 one after the other take longer than K1 - they get a stream each)
  const bool split = fork && !e->imu.empty() && (!e->biasf.empty() || (e->prior.n > 0 && e->prior_enabled));
  if (fork) {
    cudaEventRecord(e->ev_fork, st);
    cudaStreamWaitEvent(e->stream2, e->ev_fork, 0);
    e->launches += launch_imu(imu_launch(e, xb, nb), full, e->stream2);
    if (split) {
      cudaStreamWaitEvent(e->stream3, e->ev_fork, 0);
      e->launches += launch_small_factors(small_launch(e, xb, nb), full, e->stream3);
      cudaEventRecord(e->ev_join3, e->stream3);
    } else {
      e->launches += launch_small_factors(small_launch(e, xb, nb), full, e->stream2);
    }
    cudaEventRecord(e->ev_join, e->stream2);
  }
  e->launches += launch_visual(visual_launch(e, xb, nb, e->cfg.cauchy_solve), full, st);
  if (fork) cudaStreamWaitEvent(st, e->ev_join, 0);
  if (split) cudaStreamWaitEvent(st, e->ev_join3, 0);
}

// zero the normal-equation buffer the NEXT evaluation will accumulate into, on the second stream, so that it overlaps
// the linear solve of this step (only valid when everything enqueued earlier has completed: call right after a read-back)
void prezero_slab(ctvio_engine* e, int nb) {
  cudaMemsetAsync(e->ne_slab[nb].p, 0, e->ne_slab_len * sizeof(double), e->stream2);
  cudaEventRecord(e->ev_zero, e->stream2);
  e->slab_zeroed[nb] = true;
}

// published = true: the last kernel of the step (gradient_norm_kernel) has been asked to write the scalar block to
// mapped host memory with sequence number e->pub_seq: spin on it instead of copy + stream synchronise
int read_scalars(ctvio_engine* e, bool published = false) {
  if (published) {
    volatile unsigned long long* seq = &e->h_pub->seq;
    unsigned spins = 0;
    while (*seq != e->pub_seq) {
      if ((++spins & 0xfffu) == 0 && cudaStreamQuery(e->stream) != cudaErrorNotReady) {
        if (*seq == e->pub_seq) break;
        CUDA_OK(cudaStreamSynchronize(e->stream));
        CUDA_OK(cudaStreamSynchronize(e->stream2));  // (pipelined driver: the publication is forwarded from stream2)
        if (*seq != e->pub_seq) return fail(CTVIO_ERR_CUDA, "LM step finished without publishing its scalars");
      }
    }
    std::atomic_thread_fence(std::memory_order_acquire);
    *e->h_scal = const_cast<const LmPublished*>(e->h_pub)->s;
  } else {
    CUDA_OK(cudaMemcpyAsync(e->h_scal, e->d_scal.p, sizeof(LmScalars), cudaMemcpyDeviceToHost, e->stream));
    CUDA_OK(cudaStreamSynchronize(e->stream));
  }
  if ((e->h_scal->error_flags & 1) || (e->world > 1 && e->h_scal->err_sum > 0.0)) {
    cudaMemsetAsync(&e->d_scal.p->error_flags, 0, sizeof(int32_t), e->stream);
    return fail(CTVIO_ERR_TIME_RANGE, "a factor time left its knot window / the spline (line delay too large?)");
  }
  return CTVIO_OK;
}

int ensure_table(ctvio_engine* e) {
  if (!e->table_valid) {
    e->launches += launch_knot_table(e->x[e->cur].ptrs(), e->nK, e->stream);
    e->table_valid = true;
  }
  return CTVIO_OK;
}

int alloc_state(ctvio_engine* e, DevState& s) {
  CUDA_OK(s.q.reserve(4 * size_t(e->nK)));
  CUDA_OK(s.p.reserve(kPStride * size_t(e->nK)));
  CUDA_OK(s.tab.reserve(size_t(std::max(e->nK - 1, 1))));
  CUDA_OK(s.bias.reserve(6 * size_t(std::max(e->nB, 1))));
  CUDA_OK(s.rho.reserve(size_t(std::max(e->nL, 1))));
  CUDA_OK(s.ld.reserve(1));
  return CTVIO_OK;
}

}  // namespace

// =================================================================================================
extern "C" {

const char* ctvio_last_error(void) { return g_err.c_str(); }
int ctvio_abi_version(void) { return CTVIO_ABI_VERSION; }

int ctvio_create(const ctvio_config* cfg, ctvio_handle* out) {
  if (!cfg || !out) return fail(CTVIO_ERR_INVALID, "null argument");
  if (cfg->dt_ns <= 0) return fail(CTVIO_ERR_INVALID, "dt_ns must be positive");
  if (cfg->rs_padding_ns < 0 || cfg->rs_padding_ns > cfg->dt_ns)
    return fail(CTVIO_ERR_INVALID, "rs_padding_ns must lie in [0, dt_ns]: the staged knot window holds 5 knots "
                                   "(4 + one interval of rolling-shutter padding, se3_spline.h:463-503 with 39 ms / 50 ms)");
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0)
    return fail(CTVIO_ERR_NO_DEVICE, "no CUDA device visible: the ctvio engine has no CPU fallback");
  if (cfg->device < 0 || cfg->device >= ndev) return fail(CTVIO_ERR_NO_DEVICE, "device ordinal out of range");
  CUDA_OK(cudaSetDevice(cfg->device));
  cudaDeviceProp prop;
  CUDA_OK(cudaGetDeviceProperties(&prop, cfg->device));
  // sm_90a code runs on compute capability 9.0 only (arch-specific features: no forward compatibility)
  if (prop.major != 9 || prop.minor != 0)
    return fail(CTVIO_ERR_NO_DEVICE, "libctvio_b200 is built for sm_90a (H100) only");
  ctvio_engine* e = new ctvio_engine();
  e->cfg = *cfg;
  std::memset(&e->opt, 0, sizeof(e->opt));
  e->opt.fixed_knot_index = -1;
  e->opt.fix_ld = 1;
  e->sp = SplineParams{cfg->t0_ns, cfg->dt_ns, 0, 1e9 / double(cfg->dt_ns)};
  e->rig.R_CI = so3_matrix(Q4{cfg->q_CtoI[0], cfg->q_CtoI[1], cfg->q_CtoI[2], cfg->q_CtoI[3]});
  e->rig.p_CI = V3{cfg->p_CinI[0], cfg->p_CinI[1], cfg->p_CinI[2]};
  e->rig.w_img = cfg->image_weight;
  e->rig.gravity = V3{cfg->gravity[0], cfg->gravity[1], cfg->gravity[2]};
  for (int k = 0; k < 6; ++k) e->rig.imu_info[k] = cfg->imu_info[k];
  if (const char* det = std::getenv("CTVIO_DETERMINISTIC")) e->deterministic = det[0] == '1';
  if (const char* ns = std::getenv("CTVIO_NO_SPECULATION")) e->speculate = ns[0] != '1';
  if (const char* dp = std::getenv("CTVIO_STAGED_PUBLISH")) e->staged_publish = dp[0] == '1';
  const char* no_tma = std::getenv("CTVIO_NO_TMA");
  e->use_tma = !(no_tma && no_tma[0] == '1');
  if (cudaStreamCreateWithFlags(&e->stream, cudaStreamNonBlocking) != cudaSuccess ||
      cudaStreamCreateWithFlags(&e->stream2, cudaStreamNonBlocking) != cudaSuccess ||
      cudaStreamCreateWithFlags(&e->stream3, cudaStreamNonBlocking) != cudaSuccess ||
      cudaEventCreateWithFlags(&e->ev_join3, cudaEventDisableTiming) != cudaSuccess ||
      cudaEventCreate(&e->ev0) != cudaSuccess || cudaEventCreate(&e->ev1) != cudaSuccess ||
      cudaEventCreateWithFlags(&e->ev_fork, cudaEventDisableTiming) != cudaSuccess ||
      cudaEventCreateWithFlags(&e->ev_join, cudaEventDisableTiming) != cudaSuccess ||
      cudaEventCreateWithFlags(&e->ev_zero, cudaEventDisableTiming) != cudaSuccess ||
      cudaEventCreate(&e->ev_iter) != cudaSuccess || e->d_dec.reserve(1) != cudaSuccess || e->d_pubstage.reserve(1) != cudaSuccess ||
      cudaHostAlloc(&e->h_pub, sizeof(LmPublished), cudaHostAllocMapped) != cudaSuccess ||
      cudaMallocHost(&e->h_scal, sizeof(LmScalars)) != cudaSuccess || e->d_scal.reserve(1) != cudaSuccess ||
      e->d_ticket.reserve(4) != cudaSuccess) {
    delete e;
    return fail(CTVIO_ERR_CUDA, "could not create stream / events / scalar block");
  }
  cudaMemsetAsync(e->d_scal.p, 0, sizeof(LmScalars), e->stream);
  std::memset(e->h_pub, 0, sizeof(LmPublished));
  *out = e;
  return CTVIO_OK;
}

int ctvio_destroy(ctvio_handle e) {
  if (!e) return CTVIO_OK;
  cudaSetDevice(e->cfg.device);
  cudaStreamSynchronize(e->stream);
  ctvio::comm_destroy(e->nccl_comm);
  if (e->h_scal) cudaFreeHost(e->h_scal);
  if (e->h_pub) cudaFreeHost(e->h_pub);
  if (e->h_mirror) cudaFreeHost(e->h_mirror);
  if (e->ev_zero) cudaEventDestroy(e->ev_zero);
  cudaEventDestroy(e->ev0);
  cudaEventDestroy(e->ev1);
  cudaEventDestroy(e->ev_fork);
  cudaEventDestroy(e->ev_join);
  cudaStreamDestroy(e->stream2);
  if (e->stream3) cudaStreamDestroy(e->stream3);
  if (e->ev_join3) cudaEventDestroy(e->ev_join3);
  cudaStreamDestroy(e->stream);
  delete e;
  return CTVIO_OK;
}

int ctvio_set_options(ctvio_handle e, const ctvio_options* o) {
  if (!e || !o) return fail(CTVIO_ERR_INVALID, "null argument");
  e->opt = *o;
  e->masks_dirty = true;
  e->prior_dirty = true;  // col2g depends on the constant mask
  return CTVIO_OK;
}

int ctvio_set_knots(ctvio_handle e, int32_t n, const double* q, const double* p) {
  if (!e || !q || !p || n < 4) return fail(CTVIO_ERR_INVALID, "need >= 4 knots");
  cudaSetDevice(e->cfg.device);
  if (n != e->nK) e->structure_dirty = true;
  e->nK = n;
  e->sp.n_knots = n;
  for (int b = 0; b < 2; ++b) { const int rc = alloc_state(e, e->x[b]); if (rc) return rc; }
  ArenaScope arena(e);
  std::vector<double> p4(kPStride * size_t(n), 0.0);
  for (int k = 0; k < n; ++k) for (int c = 0; c < 3; ++c) p4[kPStride * k + c] = p[3 * k + c];
  CUDA_OK(staged_h2d(e->x[e->cur].q.p, q, 4 * size_t(n) * sizeof(double), e->stream));
  CUDA_OK(staged_h2d(e->x[e->cur].p.p, p4.data(), p4.size() * sizeof(double), e->stream));  // staged: p4 may go away
  e->mirror_valid = false;
  e->h2d_bytes += size_t(n) * 56;
  e->have_knots = true;
  e->table_valid = false;
  return CTVIO_OK;
}

int ctvio_set_biases(ctvio_handle e, int32_t n, const double* b) {
  if (!e || (n > 0 && !b) || n < 0) return fail(CTVIO_ERR_INVALID, "bad bias array");
  cudaSetDevice(e->cfg.device);
  if (n != e->nB) e->structure_dirty = true;
  e->nB = n;
  for (int k = 0; k < 2; ++k) CUDA_OK(e->x[k].bias.reserve(6 * size_t(std::max(n, 1))));
  ArenaScope arena(e);
  if (n > 0) CUDA_OK(staged_h2d(e->x[e->cur].bias.p, b, 6 * size_t(n) * sizeof(double), e->stream));
  e->mirror_valid = false;
  e->h2d_bytes += size_t(n) * 48;
  e->have_bias = true;
  return CTVIO_OK;
}

int ctvio_set_inv_depths(ctvio_handle e, int32_t n, const double* r) {
  if (!e || (n > 0 && !r) || n < 0) return fail(CTVIO_ERR_INVALID, "bad inverse-depth array");
  cudaSetDevice(e->cfg.device);
  if (n != e->nL) e->structure_dirty = true;
  e->nL = n;
  for (int k = 0; k < 2; ++k) CUDA_OK(e->x[k].rho.reserve(size_t(std::max(n, 1))));
  ArenaScope arena(e);
  if (n > 0) CUDA_OK(staged_h2d(e->x[e->cur].rho.p, r, size_t(n) * sizeof(double), e->stream));
  e->mirror_valid = false;
  e->h2d_bytes += size_t(n) * 8;
  e->have_rho = true;
  return CTVIO_OK;
}

int ctvio_set_time_origin(ctvio_handle e, int64_t t0_ns) {
  if (!e) return fail(CTVIO_ERR_INVALID, "null handle");
  if ((t0_ns - e->cfg.t0_ns) % e->cfg.dt_ns != 0) return fail(CTVIO_ERR_INVALID, "time origin off the knot grid");
  e->cfg.t0_ns = t0_ns;
  e->sp.t0_ns = t0_ns;
  e->structure_dirty = true;
  e->table_valid = false;
  return CTVIO_OK;
}

int ctvio_set_line_delay(ctvio_handle e, double ld) {
  if (!e) return fail(CTVIO_ERR_INVALID, "null handle");
  cudaSetDevice(e->cfg.device);
  for (int k = 0; k < 2; ++k) CUDA_OK(e->x[k].ld.reserve(1));
  ArenaScope arena(e);
  CUDA_OK(staged_h2d(e->x[e->cur].ld.p, &ld, sizeof(double), e->stream));
  e->mirror_valid = false;
  return CTVIO_OK;
}

int ctvio_get_knots(ctvio_handle e, double* q, double* p) {
  if (!e || !e->have_knots) return fail(CTVIO_ERR_STATE, "knots have not been set");
  cudaSetDevice(e->cfg.device);
  e->d2h_bytes += size_t(e->nK) * ((q ? 32 : 0) + (p ? 32 : 0));
  if (e->mirror_valid) {  // refreshed by the last solve / re-alignment: no device round trip
    const double* mq = e->h_mirror;
    const double* mp = mq + 4 * size_t(e->nK);
    if (q) std::memcpy(q, mq, 4 * size_t(e->nK) * sizeof(double));
    if (p) for (int k = 0; k < e->nK; ++k) for (int c = 0; c < 3; ++c) p[3 * k + c] = mp[kPStride * k + c];
    return CTVIO_OK;
  }
  if (q) CUDA_OK(cudaMemcpyAsync(q, e->x[e->cur].q.p, 4 * size_t(e->nK) * sizeof(double), cudaMemcpyDeviceToHost, e->stream));
  std::vector<double> p4;
  if (p) {
    p4.resize(kPStride * size_t(e->nK));
    CUDA_OK(cudaMemcpyAsync(p4.data(), e->x[e->cur].p.p, p4.size() * sizeof(double), cudaMemcpyDeviceToHost, e->stream));
  }
  CUDA_OK(cudaStreamSynchronize(e->stream));
  if (p) for (int k = 0; k < e->nK; ++k) for (int c = 0; c < 3; ++c) p[3 * k + c] = p4[kPStride * k + c];
  return CTVIO_OK;
}
int ctvio_get_biases(ctvio_handle e, double* b) {
  if (!e || !b) return fail(CTVIO_ERR_INVALID, "null argument");
  cudaSetDevice(e->cfg.device);
  e->d2h_bytes += size_t(e->nB) * 48;
  if (e->mirror_valid) {
    std::memcpy(b, e->h_mirror + (4 + kPStride) * size_t(e->nK), 6 * size_t(e->nB) * sizeof(double));
    return CTVIO_OK;
  }
  if (e->nB > 0) CUDA_OK(cudaMemcpyAsync(b, e->x[e->cur].bias.p, 6 * size_t(e->nB) * sizeof(double), cudaMemcpyDeviceToHost, e->stream));
  CUDA_OK(cudaStreamSynchronize(e->stream));
  return CTVIO_OK;
}
int ctvio_get_inv_depths(ctvio_handle e, double* r) {
  if (!e || !r) return fail(CTVIO_ERR_INVALID, "null argument");
  cudaSetDevice(e->cfg.device);
  e->d2h_bytes += size_t(e->nL) * 8;
  if (e->mirror_valid) {
    std::memcpy(r, e->h_mirror + (4 + kPStride) * size_t(e->nK) + 6 * size_t(std::max(e->nB, 1)), size_t(e->nL) * sizeof(double));
    return CTVIO_OK;
  }
  if (e->nL > 0) CUDA_OK(cudaMemcpyAsync(r, e->x[e->cur].rho.p, size_t(e->nL) * sizeof(double), cudaMemcpyDeviceToHost, e->stream));
  CUDA_OK(cudaStreamSynchronize(e->stream));
  return CTVIO_OK;
}
int ctvio_get_line_delay(ctvio_handle e, double* ld) {
  if (!e || !ld) return fail(CTVIO_ERR_INVALID, "null argument");
  cudaSetDevice(e->cfg.device);
  if (e->mirror_valid) {
    *ld = e->h_mirror[(4 + kPStride) * size_t(e->nK) + 6 * size_t(std::max(e->nB, 1)) + size_t(std::max(e->nL, 1))];
    return CTVIO_OK;
  }
  CUDA_OK(cudaMemcpyAsync(ld, e->x[e->cur].ld.p, sizeof(double), cudaMemcpyDeviceToHost, e->stream));
  CUDA_OK(cudaStreamSynchronize(e->stream));
  return CTVIO_OK;
}

int ctvio_clear_factors(ctvio_handle e) {
  if (!e) return fail(CTVIO_ERR_INVALID, "null handle");
  e->img.clear(); e->imu.clear(); e->biasf.clear();
  e->img_desc.clear(); e->imu_src.clear();
  e->structure_dirty = true;
  return CTVIO_OK;
}

int ctvio_add_image_features(ctvio_handle e, int32_t n, const int64_t* ti, const int32_t* rowi, const double* pi,
                             const int64_t* tj, const int32_t* rowj, const double* pj, const int32_t* lm,
                             const int32_t* marg) {
  if (!e || n < 0 || (n > 0 && (!ti || !rowi || !pi || !tj || !rowj || !pj || !lm)))
    return fail(CTVIO_ERR_INVALID, "null argument");
  if (!e->img_desc.empty()) return fail(CTVIO_ERR_STATE, "image factors from the resident tables are already present");
  e->img.reserve(e->img.size() + n);
  for (int k = 0; k < n; ++k) {
    HostImage o{ti[k], tj[k], rowi[k], rowj[k], {pi[2 * k], pi[2 * k + 1]}, {pj[2 * k], pj[2 * k + 1]}, lm[k],
                marg ? marg[k] : 0};
    e->img.push_back(o);
  }
  e->structure_dirty = true;
  return CTVIO_OK;
}
int ctvio_add_imu_measurements(ctvio_handle e, int32_t n, const int64_t* t, const double* gyro, const double* accel,
                               const int32_t* node, const int32_t* marg) {
  if (!e || n < 0 || (n > 0 && (!t || !gyro || !accel || !node))) return fail(CTVIO_ERR_INVALID, "null argument");
  if (!e->imu_src.empty()) return fail(CTVIO_ERR_STATE, "IMU factors from the resident table are already present");
  for (int k = 0; k < n; ++k) {
    HostImu o{t[k], {gyro[3 * k], gyro[3 * k + 1], gyro[3 * k + 2]}, {accel[3 * k], accel[3 * k + 1], accel[3 * k + 2]},
              node[k], marg ? marg[k] : 0};
    e->imu.push_back(o);
  }
  e->structure_dirty = true;
  return CTVIO_OK;
}
int ctvio_add_bias_factors(ctvio_handle e, int32_t n, const int32_t* ni, const int32_t* nj, const double* s,
                           const int32_t* marg) {
  if (!e || n < 0 || (n > 0 && (!ni || !nj || !s))) return fail(CTVIO_ERR_INVALID, "null argument");
  for (int k = 0; k < n; ++k) {
    HostBias o{ni[k], nj[k], {s[6 * k], s[6 * k + 1], s[6 * k + 2], s[6 * k + 3], s[6 * k + 4], s[6 * k + 5]},
               marg ? marg[k] : 0};
    e->biasf.push_back(o);
  }
  e->structure_dirty = true;
  return CTVIO_OK;
}

int ctvio_set_prior(ctvio_handle e, int32_t n, const double* J, const double* r, int32_t nb, const int32_t* type,
                    const int32_t* index, const int32_t* col, const double* x0) {
  if (!e) return fail(CTVIO_ERR_INVALID, "null handle");
  e->prior = ctvio::PriorHost();
  e->prior_dirty = true;
  e->prior_on_device = false;
  e->masks_dirty = true;  // the prior's blocks count as touched parameters
  if (n <= 0) return CTVIO_OK;
  if (!J || !r || nb <= 0 || !type || !index || !col || !x0) return fail(CTVIO_ERR_INVALID, "null argument");
  {
    // the blocks must tile the n columns exactly: col[b] + c indexes host tables and device scratch (dx, col2g)
    std::vector<uint8_t> covered(size_t(n), 0);
    for (int b = 0; b < nb; ++b) {
      if (type[b] < CTVIO_BLK_ROT || type[b] > CTVIO_BLK_RHO) return fail(CTVIO_ERR_INVALID, "prior block type out of range");
      const int ls = (type[b] == CTVIO_BLK_LD || type[b] == CTVIO_BLK_RHO) ? 1 : 3;
      if (col[b] < 0 || col[b] + ls > n) return fail(CTVIO_ERR_INVALID, "prior block column outside [0, n)");
      for (int c = 0; c < ls; ++c) {
        if (covered[col[b] + c]) return fail(CTVIO_ERR_INVALID, "prior blocks overlap");
        covered[col[b] + c] = 1;
      }
    }
    for (int c = 0; c < n; ++c)
      if (!covered[c]) return fail(CTVIO_ERR_INVALID, "prior blocks do not cover all n columns");
  }
  e->prior.n = n;
  e->prior.J.assign(J, J + size_t(n) * n);
  e->prior.r.assign(r, r + n);
  e->prior.type.assign(type, type + nb);
  e->prior.index.assign(index, index + nb);
  e->prior.col.assign(col, col + nb);
  e->prior.x0.assign(x0, x0 + 4 * size_t(nb));
  return CTVIO_OK;
}

// -------------------------------------------------------------------------------------------------
int ctvio_solve(ctvio_handle e, int32_t max_iterations, ctvio_summary* out) {
  if (!e) return fail(CTVIO_ERR_INVALID, "null handle");
  cudaSetDevice(e->cfg.device);
  int rc = prepare(e);
  rc = shard_consensus(e, rc);  // every rank leaves here together, or none enters the collectives below
  if (rc) return rc;
  rc = shard_check_ownership(e);
  if (rc) return rc;  // the all-reduced counts are identical on every rank: all of them return
  cudaStream_t st = e->stream;
  const ProblemDims d = e->dims();
  // Ceres 1.14 Solver::Options defaults
  const double initial_radius = 1e4, max_radius = 1e16, min_radius = 1e-32, min_relative_decrease = 1e-3;
  const double function_tolerance = 1e-6, gradient_tolerance = 1e-10, parameter_tolerance = 1e-8;
  const int max_consecutive_invalid = 5;
  const double ls_sufficient_decrease = 1e-4, ls_max_contraction = 1e-3, ls_min_contraction = 0.6, ls_min_step = 1e-9;
  const int ls_max_iterations = 20;

  ctvio_summary sum;
  std::memset(&sum, 0, sizeof(sum));
  const int64_t launches0 = e->launches;
  cudaEventRecord(e->ev0, st);

  const bool is_constrained = !e->opt.fix_ld && (e->world > 1 || e->h_active[d.idx_ld]);
  if (is_constrained) {  // IterationZero: x = Plus(x, 0) projects the line delay into its bounds
    double ld;
    CUDA_OK(cudaMemcpyAsync(&ld, e->x[e->cur].ld.p, sizeof(double), cudaMemcpyDeviceToHost, st));
    CUDA_OK(cudaStreamSynchronize(st));
    const double c = std::min(std::max(ld, e->opt.ld_lower), e->opt.ld_upper);
    if (c != ld) CUDA_OK(cudaMemcpyAsync(e->x[e->cur].ld.p, &c, sizeof(double), cudaMemcpyHostToDevice, st));
  }
  ensure_table(e);
  const bool sharded = e->world > 1;
  int cur = e->cur;  // state buffer and normal-equation buffer flip together
  evaluate(e, cur, cur, true);
  sum.num_jacobian_evals++;
  LinearLaunch lin = linear_launch(e, cur);
  if (sharded) {
    // Jacobi scaling needs the diagonal of the WHOLE camera block: all-reduce it once
    e->launches += launch_extract_diag(lin, st);
    std::string err;
    if (!ctvio::comm_allreduce_sum(e->nccl_comm, lin.diagA, size_t(e->npad), st, &err)) return fail(CTVIO_ERR_NCCL, err);
    e->launches += launch_jacobi_scale_from_diag(lin, st);
  } else {
    e->launches += launch_jacobi_scale(lin, st);
  }
  if (sharded) {
    e->launches += launch_gradient_norm(lin, e->x[cur].ptrs(), e->opt.fix_ld, e->opt.ld_lower, e->opt.ld_upper, st);
    rc = allreduce_scalars(e);
    if (rc) return rc;
    rc = read_scalars(e);
  } else {
    // (published through mapped memory like every later step: no copy + stream synchronisation)
    e->launches += launch_gradient_norm(lin, e->x[cur].ptrs(), e->opt.fix_ld, e->opt.ld_lower, e->opt.ld_upper, st, true, e->h_pub,
                                        ++e->pub_seq);
    rc = read_scalars(e, true);
  }
  if (rc) return rc;
  double x_cost = e->h_scal->cost_eval;
  double gmax = e->h_scal->gmax;  // sharded: the all-gathered maximum
  sum.initial_cost = x_cost;
  sum.num_successful_steps = 1;

  double radius = initial_radius, decrease_factor = 2.0;
  int num_invalid = 0;
  bool last_ok = true;
  int iter = 0;
  int term = CTVIO_TERM_NO_CONVERGENCE;

  auto make_apply = [&](int from, int to, double alpha) {
    ApplyLaunch ap;
    ap.dims = d;
    ap.x = e->state(from).ptrs();
    ap.xc = e->state(to).ptrs();
    ap.dc = e->d_dc.p; ap.dl = e->d_dl.p;
    ap.alpha = alpha;
    ap.active = e->d_active.p;
    ap.count_camera = e->rank == 0 ? 1 : 0;
    ap.clamp_ld = e->opt.fix_ld ? 0 : 1;
    ap.ld_lower = e->opt.ld_lower; ap.ld_upper = e->opt.ld_upper;
    ap.scal = e->d_scal.p;
    ap.det_ticket = e->deterministic ? e->d_ticket.p : nullptr;
    return ap;
  };
  auto apply = [&](int from, int to, double alpha, bool reset = true) {
    if (e->deterministic) cudaMemsetAsync(e->d_ticket.p, 0, 2 * sizeof(int32_t), st);
    e->launches += launch_apply_step(make_apply(from, to, alpha), st, reset);
  };

  // ---- pipelined driver (single GPU, no bounds, default flush mode) --------------------------------------------
  // The host round trip between two LM steps (publish -> host decision -> launch: a noticeable part of a step at C2) is
  // taken off the critical path: gradient_norm_kernel also takes the accept / radius decision on the device, and the
  // linear solve of step i+1 is enqueued BEFORE the host has seen step i, assuming acceptance (the common case),
  // reading its radius from device memory and writing its candidate into a third state buffer.  When the host then
  // finds step i rejected / invalid / terminating, the speculated kernels' results are simply never used (they touch
  // only the step vectors, the free state buffer and per-step scalars that the next real step resets).
  // It pays at C2 / C5 sizes but was measured slower per LM step at 100 k observations and more, with identical kernels
  // and a host that is provably ahead (CTVIO_LM_TRACE) - cause not found; the round trip it hides is a small part of
  // such a step anyway.  CTVIO_SPECULATION=always / never overrides the size test.
  bool spec_size_ok = e->img.size() <= 20000;
  if (const char* sp = std::getenv("CTVIO_SPECULATION")) {
    if (std::strcmp(sp, "always") == 0) spec_size_ok = true;
    if (std::strcmp(sp, "never") == 0) spec_size_ok = false;
  }
  const bool pipelined = e->speculate && spec_size_ok && !sharded && !is_constrained && !e->deterministic;
  int cur_ne = cur;  // normal-equation buffer of the current point (state and normal equations flip separately here)
  if (pipelined) {
    rc = alloc_state(e, e->xs);
    if (rc) return rc;
    bool spec_ready = false;     // a speculated linear solve from (cur, cur_ne) into state `spec_out` is in flight
    bool spec_in_flight = false; // speculated kernels that read ne_slab[cur_ne ^ 1] may still be running
    int spec_out = -1;
    unsigned spec_chol_seq0 = e->chol_seq;
    double host_spec_us = 0, host_wait_us = 0;
    static const bool lm_trace = std::getenv("CTVIO_LM_TRACE") != nullptr;  // host-side timing of the driver
    cudaEventRecord(e->ev_iter, st);
    while (true) {
      if (iter >= max_iterations) { term = CTVIO_TERM_NO_CONVERGENCE; break; }
      if (last_ok && gmax <= gradient_tolerance) { term = CTVIO_TERM_GRADIENT; break; }
      if (radius < min_radius) { term = CTVIO_TERM_MIN_RADIUS; break; }
      ++iter;
      const int cand_ne = cur_ne ^ 1;
      int cand;
      if (spec_ready) {
        cand = spec_out;  // the linear solve of this step already ran (or is running) behind the previous step
        // ne_slab[cand_ne] was the current point's buffer of the previous step: its last reader finished before that
        // step's scalars were published, and the speculated kernels read ne_slab[cur_ne] only
        prezero_slab(e, cand_ne);
      } else {
        cand = 0;
        while (cand == cur) ++cand;
        if (!spec_in_flight) prezero_slab(e, cand_ne);  // else: cleared in stream order by evaluate()
        const ApplyLaunch full_step = make_apply(cur, cand, 1.0);
        rc = lm_step(e, cur_ne, radius, &full_step);
        if (rc) return rc;
      }
      sum.num_linear_solves++;
      evaluate(e, cand, cand_ne, true, false);
      sum.num_jacobian_evals++;
      const LmDecideArgs da{e->d_dec.p, x_cost, radius, min_relative_decrease, max_radius,
                            parameter_tolerance, function_tolerance, gradient_tolerance, min_radius};
      e->launches += launch_gradient_norm(linear_launch(e, cand_ne), e->state(cand).ptrs(), e->opt.fix_ld, e->opt.ld_lower,
                                          e->opt.ld_upper, st, false, e->staged_publish ? e->d_pubstage.p : e->h_pub, ++e->pub_seq,
                                          &da);
      cudaEventRecord(e->ev_iter, st);
      if (e->staged_publish) {
        // the block goes to the host from the second stream: its PCIe round trip overlaps the speculated linear solve
        cudaStreamWaitEvent(e->stream2, e->ev_iter, 0);
        e->launches += launch_publish(e->d_pubstage.p, e->h_pub, e->stream2);
      }
      // ---- speculate: step iter + 1 from (cand, cand_ne), radius from the device-side decision ----
      spec_ready = false;
      if (iter < max_iterations) {
        spec_out = 0;
        while (spec_out == cur || spec_out == cand) ++spec_out;
        const ApplyLaunch spec_step = make_apply(cand, spec_out, 1.0);
        spec_chol_seq0 = e->chol_seq;
        const auto th0 = std::chrono::steady_clock::now();
        rc = lm_step(e, cand_ne, 0.0, &spec_step, &e->d_dec.p->radius_next, &e->d_dec.p->go);
        if (rc) return rc;
        spec_ready = true;
        spec_in_flight = true;
        host_spec_us += std::chrono::duration<double, std::micro>(std::chrono::steady_clock::now() - th0).count();
      }
      const auto th1 = std::chrono::steady_clock::now();
      rc = read_scalars(e, true);
      host_wait_us += std::chrono::duration<double, std::micro>(std::chrono::steady_clock::now() - th1).count();
      if (rc) return rc;
      const LmScalars sc = *e->h_scal;
      const LmDecision dec = const_cast<const LmPublished*>(e->h_pub)->dec;
      if (spec_ready && !dec.go) {
        // the device has cancelled the speculated step (its expensive kernels return at once): it does not count as a
        // launch of the tile-DAG solver (message buffer parity), and this driver will not use it
        e->chol_seq = spec_chol_seq0;
        spec_ready = false;
      }
      if (!dec.valid) {
        spec_ready = false;
        ++sum.num_unsuccessful_steps;
        last_ok = false;
        if (++num_invalid >= max_consecutive_invalid) { term = CTVIO_TERM_FAILURE; break; }
        radius /= decrease_factor;
        decrease_factor *= 2.0;
        continue;
      }
      num_invalid = 0;
      const double step_norm = std::sqrt(sc.step_norm2), x_norm = std::sqrt(sc.x_norm2);
      if (step_norm <= parameter_tolerance * (x_norm + parameter_tolerance)) { term = CTVIO_TERM_PARAMETER; break; }
      const double cost_change = x_cost - sc.cost_eval;
      if (std::fabs(cost_change) <= function_tolerance * x_cost) { term = CTVIO_TERM_FUNCTION; break; }
      if (dec.accept) {
        cur = cand;
        cur_ne = cand_ne;
        x_cost = sc.cost_eval;
        gmax = sc.gmax;
        radius = dec.radius_next;
        decrease_factor = 2.0;
        last_ok = true;
        ++sum.num_successful_steps;
        if (!spec_ready) spec_in_flight = false;
      } else {
        spec_ready = false;
        radius /= decrease_factor;
        decrease_factor *= 2.0;
        last_ok = false;
        ++sum.num_unsuccessful_steps;
      }
    }
    // the current state must live in x[0] / x[1] outside this function: exchange buffer names (kernels in flight hold
    // raw pointers and only touch buffers that are free under either name)
    if (cur == 2) {
      const int f = 0;  // any of the two: neither is current
      DevState &a = e->xs, &b = e->x[f];
      std::swap(a.q.p, b.q.p); std::swap(a.q.cap, b.q.cap);
      std::swap(a.p.p, b.p.p); std::swap(a.p.cap, b.p.cap);
      std::swap(a.bias.p, b.bias.p); std::swap(a.bias.cap, b.bias.cap);
      std::swap(a.rho.p, b.rho.p); std::swap(a.rho.cap, b.rho.cap);
      std::swap(a.ld.p, b.ld.p); std::swap(a.ld.cap, b.ld.cap);
      std::swap(a.tab.p, b.tab.p); std::swap(a.tab.cap, b.tab.cap);
      cur = f;
    }
    e->cur = cur;
    e->table_valid = true;
    e->slab_zeroed[0] = e->slab_zeroed[1] = false;  // (a pending clear is ordered by ev_zero only inside this loop)
    // results: wait for the last REAL kernel only (ev_iter); speculated leftovers keep running behind it and are
    // ordered before anything the next call enqueues on the engine stream
    CUDA_OK(cudaStreamWaitEvent(e->stream2, e->ev_iter, 0));
    {
      const int rcm = refresh_mirror(e, e->stream2);
      if (rcm) return rcm;
    }
    CUDA_OK(cudaStreamSynchronize(e->stream2));
    float ms = 0;
    cudaEventElapsedTime(&ms, e->ev0, e->ev_iter);
    if (lm_trace) std::fprintf(stderr, "[lm] iters %d device %.3f ms host: spec enqueue %.1f us/iter, wait %.1f us/iter\n", iter, ms, host_spec_us / std::max(iter, 1), host_wait_us / std::max(iter, 1));
    sum.iterations = iter;
    sum.termination = term;
    sum.final_cost = x_cost;
    sum.final_radius = radius;
    sum.device_ms = ms;
    sum.kernel_launches = e->launches - launches0;
    if (out) *out = sum;
    return CTVIO_OK;
  }

  while (true) {
    if (iter >= max_iterations) { term = CTVIO_TERM_NO_CONVERGENCE; break; }
    if (last_ok && gmax <= gradient_tolerance) { term = CTVIO_TERM_GRADIENT; break; }
    if (radius < min_radius) { term = CTVIO_TERM_MIN_RADIUS; break; }
    ++iter;
    const int cand = cur ^ 1;
    // ---- trust-region step + speculative full evaluation of the candidate ----
    prezero_slab(e, cand);  // everything enqueued so far has completed (scalars were read back): overlaps lm_step
    // (scale_copy_kernel of lm_step zeroes step_norm2 / x_norm2 / cost_eval / gmax: no memsets on the stream; the full
    //  step is applied by the same launch that forms the step vectors)
    const ApplyLaunch full_step = make_apply(cur, cand, 1.0);
    rc = lm_step(e, cur, radius, &full_step);
    if (rc) return rc;
    sum.num_linear_solves++;
    evaluate(e, cand, cand, true, false);
    sum.num_jacobian_evals++;
    LinearLaunch linc = linear_launch(e, cand);
    // single GPU: the gradient-norm kernel publishes the block; sharded: the reduction kernel behind the all-gather does
    if (!sharded) {
      e->launches += launch_gradient_norm(linc, e->x[cand].ptrs(), e->opt.fix_ld, e->opt.ld_lower, e->opt.ld_upper, st, false,
                                          e->h_pub, ++e->pub_seq);
    } else {
      e->launches += launch_gradient_norm(linc, e->x[cand].ptrs(), e->opt.fix_ld, e->opt.ld_lower, e->opt.ld_upper, st, false,
                                          nullptr, 0);
      rc = allreduce_scalars(e, true);
      if (rc) return rc;
    }
    rc = read_scalars(e, true);
    if (rc) return rc;
    LmScalars sc = *e->h_scal;
    const double model_cost_change = -sc.gd - 0.5 * sc.dHd;
    const bool valid = !sc.chol_fail && std::isfinite(model_cost_change) && model_cost_change > 0.0;
    if (!valid) {
      ++sum.num_unsuccessful_steps;
      last_ok = false;
      if (++num_invalid >= max_consecutive_invalid) { term = CTVIO_TERM_FAILURE; break; }
      radius /= decrease_factor;
      decrease_factor *= 2.0;
      continue;
    }
    num_invalid = 0;
    double cand_cost = sc.cost_eval, cand_gmax = sc.gmax, step_norm2 = sc.step_norm2, x_norm2 = sc.x_norm2;
    // ---- Armijo projected line search (bounds-constrained problems only; Ceres line_search.cc) ----
    if (is_constrained) {
      const double g0 = sc.gd;  // gradient . delta at x
      struct Sample { double x, value, gradient; bool value_ok, grad_ok; };
      Sample initial{0.0, x_cost, g0, true, true}, previous{0, 0, 0, false, false};
      Sample current{1.0, cand_cost, 0.0, std::isfinite(cand_cost), false};
      bool have_grad = false;
      int ls_iters = 0;
      bool success = true;
      while (!current.value_ok || current.value > x_cost + ls_sufficient_decrease * g0 * current.x) {
        ++ls_iters;
        if (ls_iters >= ls_max_iterations) { success = false; break; }
        if (current.value_ok && !have_grad) {
          // directional derivative at the trial point: g(x + a d) . d from the candidate buffers
          e->launches += ctvio::launch_dot_gradient(linear_launch(e, cand), st);
          rc = allreduce_scalars(e);
          if (rc) return rc;
          rc = read_scalars(e);
          if (rc) return rc;
          current.gradient = e->h_scal->gd;
          current.grad_ok = std::isfinite(current.gradient);
        }
        const double smin = ls_max_contraction * current.x, smax = ls_min_contraction * current.x;
        double step;
        if (!current.value_ok) {
          step = std::min(std::max(current.x * 0.5, smin), smax);
        } else {
          std::vector<ctvio::PolySample> samples;
          samples.push_back({initial.x, initial.value, initial.gradient, true, true});
          samples.push_back({current.x, current.value, current.gradient, true, current.grad_ok});
          if (previous.value_ok) samples.push_back({previous.x, previous.value, previous.gradient, true, previous.grad_ok});
          step = ctvio::minimize_interpolating_polynomial(samples, smin, smax);
        }
        if (step * sc.dir_max < ls_min_step) { success = false; break; }
        previous = current;
        apply(cur, cand, step);
        evaluate(e, cand, cand, true);
        sum.num_jacobian_evals++;
        e->launches += launch_gradient_norm(linear_launch(e, cand), e->x[cand].ptrs(), e->opt.fix_ld, e->opt.ld_lower,
                                            e->opt.ld_upper, st);
        rc = allreduce_scalars(e);
        if (rc) return rc;
        rc = read_scalars(e);
        if (rc) return rc;
        current = Sample{step, e->h_scal->cost_eval, 0.0, std::isfinite(e->h_scal->cost_eval), false};
        have_grad = false;
      }
      sum.num_line_search_steps += ls_iters;
      if (!success && current.x != 1.0) {
        // Ceres keeps the full step when the search fails: rebuild the alpha = 1 candidate
        apply(cur, cand, 1.0);
        evaluate(e, cand, cand, true);
        sum.num_jacobian_evals++;
        e->launches += launch_gradient_norm(linear_launch(e, cand), e->x[cand].ptrs(), e->opt.fix_ld, e->opt.ld_lower,
                                            e->opt.ld_upper, st);
        rc = allreduce_scalars(e);
        if (rc) return rc;
        rc = read_scalars(e);
        if (rc) return rc;
      }
      cand_cost = e->h_scal->cost_eval;
      cand_gmax = e->h_scal->gmax;
      step_norm2 = e->h_scal->step_norm2;
      x_norm2 = e->h_scal->x_norm2;
    }
    // ---- tolerances, step acceptance ----
    const double step_norm = std::sqrt(step_norm2), x_norm = std::sqrt(x_norm2);
    if (step_norm <= parameter_tolerance * (x_norm + parameter_tolerance)) { term = CTVIO_TERM_PARAMETER; break; }
    const double cost_change = x_cost - cand_cost;
    if (std::fabs(cost_change) <= function_tolerance * x_cost) { term = CTVIO_TERM_FUNCTION; break; }
    const double rho = cost_change / model_cost_change;
    if (rho > min_relative_decrease) {
      cur = cand;  // candidate state AND its normal equations become current: no re-linearisation pass
      x_cost = cand_cost;
      gmax = cand_gmax;
      radius = radius / std::max(1.0 / 3.0, 1.0 - std::pow(2.0 * rho - 1.0, 3));
      radius = std::min(max_radius, radius);
      decrease_factor = 2.0;
      last_ok = true;
      ++sum.num_successful_steps;
    } else {
      radius /= decrease_factor;
      decrease_factor *= 2.0;
      last_ok = false;
      ++sum.num_unsuccessful_steps;
    }
  }
  e->cur = cur;
  e->table_valid = true;
  if (sharded && e->nL > 0) {
    // every rank updated only the inverse depths of its own landmark shard: make them consistent everywhere
    CUDA_OK(e->d_rho_sync.reserve(2 * size_t(e->nL)));
    std::vector<uint8_t> owned(e->nL, 0);
    for (const HostImage& o : e->img) owned[o.lm] = 1;
    CUDA_OK(e->d_owned.upload(owned, st));
    e->launches += ctvio::launch_rho_pack(e->x[cur].rho.p, e->d_owned.p, e->d_rho_sync.p, e->nL, st);
    std::string err;
    if (!ctvio::comm_allreduce_sum(e->nccl_comm, e->d_rho_sync.p, 2 * size_t(e->nL), st, &err)) return fail(CTVIO_ERR_NCCL, err);
    e->launches += ctvio::launch_rho_unpack(e->x[cur].rho.p, e->d_rho_sync.p, e->nL, st);
  }
  cudaEventRecord(e->ev1, st);  // (the timed region of summary.device_ms ends here)
  {
    const int rcm = refresh_mirror(e);  // state -> pinned host mirror, rides on the synchronisation below
    if (rcm) return rcm;
  }
  CUDA_OK(cudaStreamSynchronize(st));
  float ms = 0;
  cudaEventElapsedTime(&ms, e->ev0, e->ev1);
  sum.iterations = iter;
  sum.termination = term;
  sum.final_cost = x_cost;
  sum.final_radius = radius;
  sum.device_ms = ms;
  sum.kernel_launches = e->launches - launches0;
  if (out) *out = sum;
  return CTVIO_OK;
}

int ctvio_gauge_realign(ctvio_handle e, int32_t min_idx, const double* R0, const double* t0) {
  if (!e || !R0 || !t0 || min_idx < 0 || min_idx >= e->nK) return fail(CTVIO_ERR_INVALID, "bad argument");
  cudaSetDevice(e->cfg.device);
  CUDA_OK(e->d_tmp.reserve(12));
  double h[12];
  for (int k = 0; k < 9; ++k) h[k] = R0[k];
  for (int k = 0; k < 3; ++k) h[9 + k] = t0[k];
  CUDA_OK(cudaMemcpyAsync(e->d_tmp.p, h, sizeof(h), cudaMemcpyHostToDevice, e->stream));  // (stack source: staged by the runtime)
  e->launches += launch_gauge_realign(e->x[e->cur].ptrs(), e->nK, min_idx, e->d_tmp.p, e->stream);
  {
    const int rcm = refresh_mirror(e);
    if (rcm) return rcm;
  }
  CUDA_OK(cudaStreamSynchronize(e->stream));
  e->table_valid = true;
  return CTVIO_OK;
}

int ctvio_save_state(ctvio_handle e) {
  if (!e || !e->have_knots) return fail(CTVIO_ERR_STATE, "state not set");
  cudaSetDevice(e->cfg.device);
  int rc = alloc_state(e, e->snap);
  if (rc) return rc;
  DevState& s = e->x[e->cur];
  cudaStream_t st = e->stream;
  CUDA_OK(cudaMemcpyAsync(e->snap.q.p, s.q.p, 4 * size_t(e->nK) * sizeof(double), cudaMemcpyDeviceToDevice, st));
  CUDA_OK(cudaMemcpyAsync(e->snap.p.p, s.p.p, kPStride * size_t(e->nK) * sizeof(double), cudaMemcpyDeviceToDevice, st));
  if (e->nB) CUDA_OK(cudaMemcpyAsync(e->snap.bias.p, s.bias.p, 6 * size_t(e->nB) * sizeof(double), cudaMemcpyDeviceToDevice, st));
  if (e->nL) CUDA_OK(cudaMemcpyAsync(e->snap.rho.p, s.rho.p, size_t(e->nL) * sizeof(double), cudaMemcpyDeviceToDevice, st));
  CUDA_OK(cudaMemcpyAsync(e->snap.ld.p, s.ld.p, sizeof(double), cudaMemcpyDeviceToDevice, st));
  return CTVIO_OK;
}
int ctvio_restore_state(ctvio_handle e) {
  if (!e || !e->snap.q.p) return fail(CTVIO_ERR_STATE, "no snapshot");
  cudaSetDevice(e->cfg.device);
  DevState& s = e->x[e->cur];
  cudaStream_t st = e->stream;
  CUDA_OK(cudaMemcpyAsync(s.q.p, e->snap.q.p, 4 * size_t(e->nK) * sizeof(double), cudaMemcpyDeviceToDevice, st));
  CUDA_OK(cudaMemcpyAsync(s.p.p, e->snap.p.p, kPStride * size_t(e->nK) * sizeof(double), cudaMemcpyDeviceToDevice, st));
  if (e->nB) CUDA_OK(cudaMemcpyAsync(s.bias.p, e->snap.bias.p, 6 * size_t(e->nB) * sizeof(double), cudaMemcpyDeviceToDevice, st));
  if (e->nL) CUDA_OK(cudaMemcpyAsync(s.rho.p, e->snap.rho.p, size_t(e->nL) * sizeof(double), cudaMemcpyDeviceToDevice, st));
  CUDA_OK(cudaMemcpyAsync(s.ld.p, e->snap.ld.p, sizeof(double), cudaMemcpyDeviceToDevice, st));
  e->table_valid = false;
  e->mirror_valid = false;
  return CTVIO_OK;
}

// ---- probes --------------------------------------------------------------------------------------
int ctvio_eval_image_factors(ctvio_handle e, int32_t want_jac, double cauchy, double* r, int32_t* s, double* J,
                             double* cost) {
  if (!e) return fail(CTVIO_ERR_INVALID, "null handle");
  cudaSetDevice(e->cfg.device);
  int rc = prepare(e);
  if (rc) return rc;
  ensure_table(e);
  const size_t n = e->img.size();
  DevBuf<double> dr, dJ;
  DevBuf<int32_t> ds;
  CUDA_OK(dr.reserve(2 * n));
  CUDA_OK(ds.reserve(2 * n));
  if (want_jac) CUDA_OK(dJ.reserve(100 * n));
  cudaStream_t st = e->stream;
  cudaMemsetAsync(&e->d_scal.p->cost_eval, 0, sizeof(double), st);
  e->launches += launch_probe_image(visual_launch(e, e->cur, e->cur, cauchy), e->d_img_orig.p, want_jac != 0, dr.p, ds.p,
                                    want_jac ? dJ.p : nullptr, st);
  rc = read_scalars(e);
  if (rc) return rc;
  if (r && n) CUDA_OK(cudaMemcpy(r, dr.p, 2 * n * sizeof(double), cudaMemcpyDeviceToHost));
  if (s && n) CUDA_OK(cudaMemcpy(s, ds.p, 2 * n * sizeof(int32_t), cudaMemcpyDeviceToHost));
  if (J && want_jac && n) CUDA_OK(cudaMemcpy(J, dJ.p, 100 * n * sizeof(double), cudaMemcpyDeviceToHost));
  if (cost) *cost = e->h_scal->cost_eval;
  return CTVIO_OK;
}

int ctvio_eval_imu_factors(ctvio_handle e, int32_t want_jac, double* r, int32_t* s, double* J, double* cost) {
  if (!e) return fail(CTVIO_ERR_INVALID, "null handle");
  cudaSetDevice(e->cfg.device);
  int rc = prepare(e);
  if (rc) return rc;
  ensure_table(e);
  const size_t n = e->imu.size();
  DevBuf<double> dr, dJ;
  DevBuf<int32_t> ds;
  CUDA_OK(dr.reserve(6 * n));
  CUDA_OK(ds.reserve(n));
  if (want_jac) CUDA_OK(dJ.reserve(156 * n));
  cudaStream_t st = e->stream;
  cudaMemsetAsync(&e->d_scal.p->cost_eval, 0, sizeof(double), st);
  e->launches += launch_probe_imu(imu_launch(e, e->cur, e->cur), e->d_imu_orig.p, want_jac != 0, dr.p, ds.p,
                                  want_jac ? dJ.p : nullptr, st);
  rc = read_scalars(e);
  if (rc) return rc;
  if (r && n) CUDA_OK(cudaMemcpy(r, dr.p, 6 * n * sizeof(double), cudaMemcpyDeviceToHost));
  if (s && n) CUDA_OK(cudaMemcpy(s, ds.p, n * sizeof(int32_t), cudaMemcpyDeviceToHost));
  if (J && want_jac && n) CUDA_OK(cudaMemcpy(J, dJ.p, 156 * n * sizeof(double), cudaMemcpyDeviceToHost));
  if (cost) *cost = e->h_scal->cost_eval;
  return CTVIO_OK;
}

int ctvio_residual_summary(ctvio_handle e, int32_t* counts, double* sums, double* prior_sum) {
  if (!e || !counts || !sums) return fail(CTVIO_ERR_INVALID, "null argument");
  cudaSetDevice(e->cfg.device);
  int rc = prepare(e);
  if (rc) return rc;
  ensure_table(e);
  cudaStream_t st = e->stream;
  const size_t ni = e->img.size(), nm = e->imu.size(), nb = e->biasf.size();
  const int np_ = e->prior_enabled ? e->prior.n : 0;
  DevBuf<double> dr, dout;
  DevBuf<int32_t> ds;
  CUDA_OK(dr.reserve(2 * ni + 6 * nm + 8));
  CUDA_OK(ds.reserve(2 * ni + nm + 8));
  CUDA_OK(dout.reserve(18));
  CUDA_OK(cudaMemsetAsync(dout.p, 0, 18 * sizeof(double), st));
  // residuals without the loss (cauchy scale 0 = no corrector), original factor order does not matter for the sums
  if (ni) e->launches += launch_probe_image(visual_launch(e, e->cur, e->cur, 0.0), e->d_img_orig.p, false, dr.p, ds.p, nullptr, st);
  if (nm) e->launches += launch_probe_imu(imu_launch(e, e->cur, e->cur), e->d_imu_orig.p, false, dr.p + 2 * ni, ds.p + 2 * ni, nullptr, st);
  e->launches += ctvio::launch_abs_column_sums(dr.p, int(ni), 2, dout.p, st);
  e->launches += ctvio::launch_abs_column_sums(dr.p + 2 * ni, int(nm), 6, dout.p + 2, st);
  e->launches += ctvio::launch_bias_abs_sums(e->d_bf_ij.p, e->d_bf_s.p, int(nb), e->x[e->cur].bias.p, dout.p + 8, st);
  if (np_ > 0) {
    e->launches += launch_small_factors(small_launch(e, e->cur, e->cur), false, st);  // leaves r + J dx in prior.res
  }
  rc = read_scalars(e);
  if (rc) return rc;
  CUDA_OK(cudaMemcpy(sums, dout.p, 18 * sizeof(double), cudaMemcpyDeviceToHost));
  counts[0] = int32_t(ni); counts[1] = int32_t(nm); counts[2] = int32_t(nb); counts[3] = np_ > 0 ? 1 : 0;
  if (prior_sum && np_ > 0) {
    CUDA_OK(cudaMemcpy(prior_sum, e->d_prior_res.p, size_t(np_) * sizeof(double), cudaMemcpyDeviceToHost));
    for (int i = 0; i < np_; ++i) prior_sum[i] = std::fabs(prior_sum[i]);
  }
  return CTVIO_OK;
}

int ctvio_eval_cost(ctvio_handle e, double* cost) {
  if (!e || !cost) return fail(CTVIO_ERR_INVALID, "null argument");
  cudaSetDevice(e->cfg.device);
  int rc = prepare(e);
  if (rc) return rc;
  ensure_table(e);
  evaluate(e, e->cur, e->cur, false);
  rc = read_scalars(e);
  if (rc) return rc;
  *cost = e->h_scal->cost_eval;
  return CTVIO_OK;
}

int ctvio_normal_equations(ctvio_handle e, double* Hcc, double* gc, double* hl, double* gl, double* cost) {
  if (!e) return fail(CTVIO_ERR_INVALID, "null handle");
  cudaSetDevice(e->cfg.device);
  int rc = prepare(e);
  if (rc) return rc;
  ensure_table(e);
  evaluate(e, e->cur, e->cur, true);
  rc = read_scalars(e);
  if (rc) return rc;
  const ProblemDims d = e->dims();
  const size_t np = d.np;
  NormalEqPtrs ne = e->ne(e->cur);
  if (Hcc) {
    std::vector<double> up(np * np);
    CUDA_OK(cudaMemcpy(up.data(), ne.A, np * np * sizeof(double), cudaMemcpyDeviceToHost));
    for (size_t i = 0; i < np; ++i)
      for (size_t j = i; j < np; ++j) Hcc[i * np + j] = Hcc[j * np + i] = up[i * np + j];
  }
  if (gc) CUDA_OK(cudaMemcpy(gc, ne.gc, np * sizeof(double), cudaMemcpyDeviceToHost));
  if (hl && e->nL) CUDA_OK(cudaMemcpy(hl, ne.hl, e->nL * sizeof(double), cudaMemcpyDeviceToHost));
  if (gl && e->nL) CUDA_OK(cudaMemcpy(gl, ne.gl, e->nL * sizeof(double), cudaMemcpyDeviceToHost));
  if (cost) *cost = e->h_scal->cost_eval;
  return CTVIO_OK;
}

int ctvio_query_trajectory(ctvio_handle e, int32_t n, const int64_t* t, double* q, double* p, double* omega,
                           double* vel, double* acc) {
  if (!e || n < 0 || (n > 0 && !t)) return fail(CTVIO_ERR_INVALID, "bad argument");
  if (!e->have_knots) return fail(CTVIO_ERR_STATE, "knots have not been set");
  cudaSetDevice(e->cfg.device);
  ensure_table(e);
  if (n == 0) return CTVIO_OK;
  DevBuf<int64_t> dt;
  DevBuf<double> out;
  CUDA_OK(dt.reserve(n));
  CUDA_OK(out.reserve(16 * size_t(n)));
  cudaStream_t st = e->stream;
  CUDA_OK(cudaMemcpyAsync(dt.p, t, size_t(n) * sizeof(int64_t), cudaMemcpyHostToDevice, st));
  QueryLaunch a;
  a.st = e->x[e->cur].ptrs();
  a.sp = e->sp;
  a.n = n;
  a.t = dt.p;
  a.q = out.p; a.p = out.p + 4 * size_t(n); a.omega = out.p + 7 * size_t(n); a.vel = out.p + 10 * size_t(n);
  a.acc = out.p + 13 * size_t(n);
  a.scal = e->d_scal.p;
  e->launches += launch_query(a, st);
  int rc = read_scalars(e);
  if (rc) return rc;
  if (q) CUDA_OK(cudaMemcpy(q, a.q, 4 * size_t(n) * sizeof(double), cudaMemcpyDeviceToHost));
  if (p) CUDA_OK(cudaMemcpy(p, a.p, 3 * size_t(n) * sizeof(double), cudaMemcpyDeviceToHost));
  if (omega) CUDA_OK(cudaMemcpy(omega, a.omega, 3 * size_t(n) * sizeof(double), cudaMemcpyDeviceToHost));
  if (vel) CUDA_OK(cudaMemcpy(vel, a.vel, 3 * size_t(n) * sizeof(double), cudaMemcpyDeviceToHost));
  if (acc) CUDA_OK(cudaMemcpy(acc, a.acc, 3 * size_t(n) * sizeof(double), cudaMemcpyDeviceToHost));
  return CTVIO_OK;
}

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
  CUDA_OK(cudaStreamSynchronize(st));
  return CTVIO_OK;
}

int ctvio_profile_kernels(ctvio_handle e, int32_t reps, int32_t flush_l2, double* out) {
  if (!e || !out || reps == 0) return fail(CTVIO_ERR_INVALID, "bad argument");
  const bool visual_only = reps < 0;  // reps < 0: only out_ms[0] (K1) - usable on a sharded engine (no collectives)
  if (visual_only) reps = -reps;
  cudaSetDevice(e->cfg.device);
  int rc = prepare(e);
  if (rc) return rc;
  ensure_table(e);
  cudaStream_t st = e->stream;
  const int cur = e->cur, cand = cur ^ 1;
  DevBuf<unsigned char> flush;
  const size_t flush_bytes = size_t(256) << 20;
  if (flush_l2) CUDA_OK(flush.reserve(flush_bytes));
  if (visual_only) {
    for (int k = 0; k < 8; ++k) out[k] = 0.0;
    double total = 0;
    for (int it = -3; it < reps; ++it) {
      if (flush_l2) cudaMemsetAsync(flush.p, it & 0xff, flush_bytes, st);
      cudaMemsetAsync(e->ne_slab[cur].p, 0, e->ne_slab_len * sizeof(double), st);
      cudaEventRecord(e->ev0, st);
      launch_visual(visual_launch(e, cur, cur, e->cfg.cauchy_solve), true, st);
      cudaEventRecord(e->ev1, st);
      if (cudaEventSynchronize(e->ev1) != cudaSuccess) return fail(CTVIO_ERR_CUDA, "kernel failed while profiling");
      float ms = 0;
      cudaEventElapsedTime(&ms, e->ev0, e->ev1);
      if (it >= 0) total += ms;
    }
    out[0] = total / reps;
    cudaMemsetAsync(&e->d_scal.p->error_flags, 0, sizeof(int32_t), st);
    CUDA_OK(cudaStreamSynchronize(st));
    return CTVIO_OK;
  }
  // a valid linearisation + step so that every stage has meaningful inputs
  evaluate(e, cur, cur, true);
  LinearLaunch lin = linear_launch(e, cur);
  launch_jacobi_scale(lin, st);
  launch_lm_step(lin, 1e4, st);
  rc = read_scalars(e);
  if (rc) return rc;
  ApplyLaunch ap;
  ap.dims = e->dims();
  ap.x = e->x[cur].ptrs(); ap.xc = e->x[cand].ptrs();
  ap.dc = e->d_dc.p; ap.dl = e->d_dl.p; ap.alpha = 1.0; ap.active = e->d_active.p;
  ap.count_camera = 1;
  ap.clamp_ld = e->opt.fix_ld ? 0 : 1; ap.ld_lower = e->opt.ld_lower; ap.ld_upper = e->opt.ld_upper;
  ap.scal = e->d_scal.p;
  auto time_stage = [&](int stage, double* ms_out) -> int {
    double total = 0;
    for (int it = -3; it < reps; ++it) {
      if (flush_l2) cudaMemsetAsync(flush.p, it & 0xff, flush_bytes, st);
      if (stage == 0 || stage == 1 || stage == 2)
        cudaMemsetAsync(e->ne_slab[cur].p, 0, e->ne_slab_len * sizeof(double), st);
      cudaEventRecord(e->ev0, st);
      switch (stage) {
        case 0: launch_visual(visual_launch(e, cur, cur, e->cfg.cauchy_solve), true, st); break;
        case 1: launch_imu(imu_launch(e, cur, cur), true, st); break;
        case 2: launch_small_factors(small_launch(e, cur, cur), true, st); break;
        case 3: launch_reduced_system(lin, 1e4, st); break;
        case 4: launch_factor_solve(lin, st); break;
        case 5: launch_step_vectors(lin, st); break;
        case 6: launch_apply_step(ap, st); break;
        default: launch_visual(visual_launch(e, cur, cur, e->cfg.cauchy_solve), false, st); break;
      }
      cudaEventRecord(e->ev1, st);
      if (cudaEventSynchronize(e->ev1) != cudaSuccess) return fail(CTVIO_ERR_CUDA, "kernel failed while profiling");
      float ms = 0;
      cudaEventElapsedTime(&ms, e->ev0, e->ev1);
      if (it >= 0) total += ms;
    }
    *ms_out = total / reps;
    return CTVIO_OK;
  };
  // stage order keeps inputs valid: 3 (reduced system) must precede 4 (it is factored in place)
  for (int stage : {0, 1, 2, 7}) { rc = time_stage(stage, &out[stage]); if (rc) return rc; }
  evaluate(e, cur, cur, true);  // restore a complete set of normal equations
  {
    double total3 = 0, total4 = 0, total5 = 0;
    for (int it = -3; it < reps; ++it) {
      float ms;
      if (flush_l2) cudaMemsetAsync(flush.p, it & 0xff, flush_bytes, st);
      cudaEventRecord(e->ev0, st); launch_reduced_system(lin, 1e4, st); cudaEventRecord(e->ev1, st);
      cudaEventSynchronize(e->ev1); cudaEventElapsedTime(&ms, e->ev0, e->ev1); if (it >= 0) total3 += ms;
      if (flush_l2) cudaMemsetAsync(flush.p, it & 0xff, flush_bytes, st);
      cudaEventRecord(e->ev0, st); launch_factor_solve(lin, st); cudaEventRecord(e->ev1, st);
      cudaEventSynchronize(e->ev1); cudaEventElapsedTime(&ms, e->ev0, e->ev1); if (it >= 0) total4 += ms;
      if (flush_l2) cudaMemsetAsync(flush.p, it & 0xff, flush_bytes, st);
      cudaEventRecord(e->ev0, st); launch_step_vectors(lin, st); cudaEventRecord(e->ev1, st);
      cudaEventSynchronize(e->ev1); cudaEventElapsedTime(&ms, e->ev0, e->ev1); if (it >= 0) total5 += ms;
    }
    out[3] = total3 / reps; out[4] = total4 / reps; out[5] = total5 / reps;
  }
  rc = time_stage(6, &out[6]);
  if (rc) return rc;
  cudaMemsetAsync(&e->d_scal.p->error_flags, 0, sizeof(int32_t), st);
  CUDA_OK(cudaStreamSynchronize(st));
  return CTVIO_OK;
}

int ctvio_selfcheck_solver(ctvio_handle e, int32_t reps, int32_t* mismatches, double* rel_residual) {
  if (!e || !mismatches || !rel_residual || reps <= 0) return fail(CTVIO_ERR_INVALID, "bad argument");
  cudaSetDevice(e->cfg.device);
  int rc = prepare(e);
  if (rc) return rc;
  ensure_table(e);
  cudaStream_t st = e->stream;
  const int cur = e->cur;
  evaluate(e, cur, cur, true);
  LinearLaunch lin = linear_launch(e, cur);
  launch_jacobi_scale(lin, st);
  launch_reduced_system(lin, 1e4, st);
  const size_t n = size_t(e->npad), len = n * n + n;  // M | rhs are contiguous
  DevBuf<double> backup;
  CUDA_OK(backup.reserve(len));
  CUDA_OK(cudaMemcpyAsync(backup.p, lin.M, len * sizeof(double), cudaMemcpyDeviceToDevice, st));
  std::vector<double> hM(len), x0(n), x(n);
  CUDA_OK(cudaMemcpyAsync(hM.data(), lin.M, len * sizeof(double), cudaMemcpyDeviceToHost, st));
  *mismatches = 0;
  for (int r = 0; r < reps; ++r) {
    if (r > 0) CUDA_OK(cudaMemcpyAsync(lin.M, backup.p, len * sizeof(double), cudaMemcpyDeviceToDevice, st));
    launch_factor_solve(lin, st);
    CUDA_OK(cudaMemcpyAsync((r == 0 ? x0 : x).data(), lin.y, n * sizeof(double), cudaMemcpyDeviceToHost, st));
    CUDA_OK(cudaStreamSynchronize(st));
    if (r > 0 && std::memcmp(x.data(), x0.data(), n * sizeof(double)) != 0) ++*mismatches;
  }
  // residual of the first solve against the host copy (only the lower triangle of M is maintained by K4)
  for (size_t i = 0; i < n; ++i)
    for (size_t j = i + 1; j < n; ++j) hM[i * n + j] = hM[j * n + i];
  const double* rhs = hM.data() + n * n;
  double rmax = 0, bmax = 0;
  for (size_t i = 0; i < n; ++i) {
    double s = -rhs[i];
    for (size_t j = 0; j < n; ++j) s += hM[i * n + j] * x0[j];
    rmax = std::max(rmax, std::fabs(s));
    bmax = std::max(bmax, std::fabs(rhs[i]));
  }
  *rel_residual = bmax > 0 ? rmax / bmax : rmax;
  cudaMemsetAsync(&e->d_scal.p->error_flags, 0, sizeof(int32_t), st);
  CUDA_OK(cudaStreamSynchronize(st));
  return CTVIO_OK;
}

int ctvio_measure_fp64_tflops(ctvio_handle e, double* tflops) {
  if (!e || !tflops) return fail(CTVIO_ERR_INVALID, "null argument");
  cudaSetDevice(e->cfg.device);
  const double v = ctvio::measure_fp64_tflops(e->stream);
  if (v < 0) return fail(CTVIO_ERR_CUDA, "fp64 micro-benchmark failed");
  *tflops = v;
  return CTVIO_OK;
}

int ctvio_measure_fp64_tensor_tflops(ctvio_handle e, double* tflops) {
  if (!e || !tflops) return fail(CTVIO_ERR_INVALID, "null argument");
  cudaSetDevice(e->cfg.device);
  const double v = ctvio::measure_fp64_tensor_tflops(e->stream);
  if (v < 0) return fail(CTVIO_ERR_CUDA, "fp64 tensor-core micro-benchmark failed");
  *tflops = v;
  return CTVIO_OK;
}

// ---- marginalization (K7), see marginalize.cu ---------------------------------------------------
int ctvio_marginalize(ctvio_handle e, int32_t* n_out, int32_t* nb_out) {
  if (!e || !n_out || !nb_out) return fail(CTVIO_ERR_INVALID, "null argument");
  *n_out = 0;
  *nb_out = 0;
  cudaSetDevice(e->cfg.device);
  e->new_prior = ctvio::PriorHost();
  if (!e->opt.is_marg_state) return CTVIO_OK;
  ArenaScope arena(e);
  int rc = prepare(e);
  if (rc) return rc;
  ensure_table(e);
  cudaStream_t st = e->stream;
  const ProblemDims d = e->dims();
  const int later = e->opt.ctrl_to_be_opt_later, nowk = e->opt.ctrl_to_be_opt_now;
  const bool drop_knots = later > nowk;  // trajectory_estimator.cpp:161

  // ---- which parameter blocks the recorded factors touch, and which of them are dropped ----
  // block key order == position order: knots (rot, pos per knot), bias nodes (bg, ba), line delay, inverse depths
  struct Key {
    int type, index;
    bool operator<(const Key& o) const {
      auto rank = [](const Key& k) {
        switch (k.type) {
          case CTVIO_BLK_ROT: return std::make_pair(0, 2 * k.index);
          case CTVIO_BLK_POS: return std::make_pair(0, 2 * k.index + 1);
          case CTVIO_BLK_BG: return std::make_pair(1, 2 * k.index);
          case CTVIO_BLK_BA: return std::make_pair(1, 2 * k.index + 1);
          case CTVIO_BLK_LD: return std::make_pair(2, 0);
          default: return std::make_pair(3, k.index);
        }
      };
      return rank(*this) < rank(o);
    }
  };
  struct Info { bool dropped = false; int pos = -1; };
  std::map<Key, Info> blocks;
  auto touch = [&](int type, int index, bool drop) { Info& b = blocks[Key{type, index}]; b.dropped = b.dropped || drop; };
  bool use_prior = false;
  if (e->prior.n > 0) {  // [1] old prior (trajectory_manager.cpp:166-203)
    auto is_drop = [&](size_t b) {
      const int t = e->prior.type[b], i = e->prior.index[b];
      const bool isknot = t == CTVIO_BLK_ROT || t == CTVIO_BLK_POS;
      return (isknot && i >= nowk && i < later) || ((t == CTVIO_BLK_BG || t == CTVIO_BLK_BA) && i == 0);
    };
    for (size_t b = 0; b < e->prior.type.size(); ++b) use_prior = use_prior || is_drop(b);
    if (use_prior)
      for (size_t b = 0; b < e->prior.type.size(); ++b) touch(e->prior.type[b], e->prior.index[b], is_drop(b));
  }
  std::vector<int32_t> marg_img, marg_imu;
  for (size_t k = 0; k < e->img_order.size(); ++k) {  // [2] image factors (trajectory_estimator.cpp:325-331)
    const HostImage& o = e->img[e->img_order[k]];
    if (!o.marg) continue;
    marg_img.push_back(int32_t(k));
    int f0, l0, f1, l1;
    knot_window(e, o.ti, f0, l0);
    knot_window(e, o.tj, f1, l1);
    for (int side = 0; side < 2; ++side)
      for (int kk = (side ? f1 : f0); kk <= (side ? l1 : l0); ++kk) {
        touch(CTVIO_BLK_ROT, kk, drop_knots && kk < later);
        touch(CTVIO_BLK_POS, kk, drop_knots && kk < later);
      }
    touch(CTVIO_BLK_RHO, o.lm, true);
    touch(CTVIO_BLK_LD, 0, false);
  }
  for (size_t k = 0; k < e->imu_order.size(); ++k) {  // [3] IMU factors (:249-257)
    const HostImu& o = e->imu[e->imu_order[k]];
    if (!o.marg) continue;
    marg_imu.push_back(int32_t(k));
    const int s = knot_window_first(e, o.t);
    for (int kk = s; kk <= s + 3; ++kk) {
      touch(CTVIO_BLK_ROT, kk, drop_knots && kk < later);
      touch(CTVIO_BLK_POS, kk, drop_knots && kk < later);
    }
    touch(CTVIO_BLK_BG, o.node, true);
    touch(CTVIO_BLK_BA, o.node, true);
  }
  std::vector<int2> bij;
  std::vector<double> bs;
  for (const HostBias& o : e->biasf) {  // [4] bias factors (:280-285), drop {bg_i, ba_i}
    if (!o.marg) continue;
    bij.push_back(make_int2(o.i, o.j));
    for (int c = 0; c < 6; ++c) bs.push_back(o.s[c]);
    touch(CTVIO_BLK_BG, o.i, true); touch(CTVIO_BLK_BG, o.j, false);
    touch(CTVIO_BLK_BA, o.i, true); touch(CTVIO_BLK_BA, o.j, false);
  }
  if (blocks.empty()) return CTVIO_OK;
  auto local_size = [](int t) { return (t == CTVIO_BLK_LD || t == CTVIO_BLK_RHO) ? 1 : 3; };
  int pos = 0;
  for (auto& kv : blocks) if (kv.second.dropped) { kv.second.pos = pos; pos += local_size(kv.first.type); }
  const int m = pos;
  for (auto& kv : blocks) if (!kv.second.dropped) { kv.second.pos = pos; pos += local_size(kv.first.type); }
  const int n = pos - m, P = pos;
  if (n <= 0) return CTVIO_OK;  // the reference hands back nullptr (trajectory_estimator.cpp:198-201)

  std::vector<int32_t> pos_cam(d.np, -1), pos_lm(std::max(e->nL, 1), -1), prior_pos(std::max(e->prior.n, 1), -1);
  for (const auto& kv : blocks) {
    if (kv.first.type == CTVIO_BLK_RHO) { pos_lm[kv.first.index] = kv.second.pos; continue; }
    const int g = ctvio::prior_block_base(kv.first.type, kv.first.index, d.nK, d.nB);
    if (g < 0) return fail(CTVIO_ERR_INVALID, "marginalization block index out of range");
    for (int c = 0; c < local_size(kv.first.type); ++c) pos_cam[g + c] = kv.second.pos + c;
  }
  if (use_prior)
    for (size_t b = 0; b < e->prior.type.size(); ++b) {
      const int p0 = blocks[Key{e->prior.type[b], e->prior.index[b]}].pos;
      for (int c = 0; c < local_size(e->prior.type[b]); ++c) prior_pos[e->prior.col[b] + c] = p0 + c;
    }

  // ---- A, b on the device ----
  ctvio_engine::MargWs& ws = e->mws;
  DevBuf<int32_t>&d_pos_cam = ws.pos_cam, &d_pos_lm = ws.pos_lm, &d_prior_pos = ws.prior_pos, &d_marg_img = ws.marg_img,
      &d_marg_imu = ws.marg_imu;
  DevBuf<int2>& d_bij = ws.bij;
  DevBuf<double>&d_bs = ws.bs, &d_A = ws.A, &d_b = ws.b;
  CUDA_OK(d_pos_cam.upload(pos_cam, st));
  CUDA_OK(d_pos_lm.upload(pos_lm, st));
  CUDA_OK(d_prior_pos.upload(prior_pos, st));
  CUDA_OK(d_marg_img.upload(marg_img, st));
  CUDA_OK(d_marg_imu.upload(marg_imu, st));
  CUDA_OK(d_bij.upload(bij, st));
  CUDA_OK(d_bs.upload(bs, st));
  CUDA_OK(d_A.reserve(size_t(P) * P));
  CUDA_OK(d_b.reserve(P));
  {
    // row-compressed Jacobian of every recorded factor, then [A | b] = Jrow' Jrow in a fixed summation order
    const int n_old = use_prior ? e->prior.n : 0;
    const int row_img = 0, row_imu = 2 * int(marg_img.size()), row_bias = row_imu + 6 * int(marg_imu.size());
    const int row_prior = row_bias + 6 * int(bij.size());
    const int R = row_prior + n_old;
    const int ldj = (P + 2) & ~1;
    CUDA_OK(ws.Jrow.reserve(size_t(std::max(R, 1)) * ldj));
    CUDA_OK(cudaMemsetAsync(ws.Jrow.p, 0, size_t(std::max(R, 1)) * ldj * sizeof(double), st));
    ctvio::MargImageArgs a;
    a.obs = ImageObsPtrs{e->d_img_t.p, e->d_img_pi.p, e->d_img_pj.p, e->d_img_meta.p, int32_t(e->img.size())};
    a.marg_index = d_marg_img.p; a.n_marg = int32_t(marg_img.size());
    a.st = e->x[e->cur].ptrs(); a.sp = e->sp; a.rig = e->rig; a.cauchy = e->cfg.cauchy_marg;
    a.pos_cam = d_pos_cam.p; a.pos_lm = d_pos_lm.p; a.idx_ld = d.idx_ld;
    a.Jrow = ws.Jrow.p; a.ldj = ldj; a.row0 = row_img; a.P = P; a.scal = e->d_scal.p;
    // the three row kernels write disjoint row ranges of Jrow: one stream each, joined before the SYRK
    cudaEventRecord(e->ev_fork, st);
    e->launches += ctvio::launch_marg_image(a, st);
    ctvio::MargImuArgs b;
    b.obs = ImuObsPtrs{e->d_imu_t.p, e->d_imu_ga.p, int32_t(e->imu.size())};
    b.marg_index = d_marg_imu.p; b.n_marg = int32_t(marg_imu.size());
    b.st = a.st; b.sp = e->sp; b.rig = e->rig; b.pos_cam = d_pos_cam.p; b.idx_bias0 = d.idx_bias0;
    b.Jrow = ws.Jrow.p; b.ldj = ldj; b.row0 = row_imu; b.P = P; b.scal = e->d_scal.p;
    cudaStreamWaitEvent(e->stream2, e->ev_fork, 0);
    e->launches += ctvio::launch_marg_imu(b, e->stream2);
    cudaEventRecord(e->ev_join, e->stream2);
    ctvio::MargSmallArgs c;
    c.bf_ij = d_bij.p; c.bf_s = d_bs.p; c.n_bias = int32_t(bij.size());
    c.prior = prior_ptrs(e); c.use_prior = use_prior ? 1 : 0; c.prior_pos = d_prior_pos.p;
    c.st = a.st; c.pos_cam = d_pos_cam.p; c.idx_bias0 = d.idx_bias0;
    c.Jrow = ws.Jrow.p; c.ldj = ldj; c.row0_bias = row_bias; c.row0_prior = row_prior; c.P = P;
    cudaStreamWaitEvent(e->stream3, e->ev_fork, 0);
    e->launches += ctvio::launch_marg_small(c, e->stream3);
    cudaEventRecord(e->ev_join3, e->stream3);
    cudaStreamWaitEvent(st, e->ev_join, 0);
    cudaStreamWaitEvent(st, e->ev_join3, 0);
    e->launches += ctvio::launch_marg_syrk(ws.Jrow.p, R, ldj, P, d_A.p, d_b.p, st);
  }
  // ---- dense Schur complement through eigen-decompositions (marginalization_factor.cpp:240-263) ----
  const double eps = 1e-30;
  DevBuf<double>&d_Amm = ws.Amm, &d_V = ws.V, &d_ev = ws.ev, &d_Vs = ws.Vs, &d_Ainv = ws.Ainv, &d_T = ws.T, &d_Ap = ws.Ap,
      &d_bp = ws.bp, &d_Ap2 = ws.Ap2, &d_V2 = ws.V2, &d_ev2 = ws.ev2, &d_vb = ws.vb, &d_J = ws.J, &d_r = ws.r;
  CUDA_OK(d_Ap.reserve(size_t(n) * n));
  CUDA_OK(d_bp.reserve(n));
  CUDA_OK(cudaMemcpy2DAsync(d_Ap.p, size_t(n) * sizeof(double), d_A.p + size_t(m) * P + m, size_t(P) * sizeof(double),
                            size_t(n) * sizeof(double), n, cudaMemcpyDeviceToDevice, st));
  CUDA_OK(cudaMemcpyAsync(d_bp.p, d_b.p + m, size_t(n) * sizeof(double), cudaMemcpyDeviceToDevice, st));
  if (m > 0) {
    CUDA_OK(d_Amm.reserve(size_t(m) * m)); CUDA_OK(d_V.reserve(size_t(m) * m)); CUDA_OK(d_ev.reserve(m));
    CUDA_OK(d_Vs.reserve(size_t(m) * m)); CUDA_OK(d_Ainv.reserve(size_t(m) * m)); CUDA_OK(d_T.reserve(size_t(n) * m));
    e->launches += ctvio::launch_marg_elementwise(0, m, P, d_A.p, d_Amm.p, nullptr, nullptr, nullptr, eps, st);
    CUDA_OK(ws.eig_scratch.reserve(ctvio::jacobi_log_bytes(std::max(m, n), 40) / sizeof(double) + 1));
    e->launches += ctvio::launch_jacobi_eig(d_Amm.p, d_V.p, d_ev.p, m, ws.eig_scratch.p, st);
    e->launches += ctvio::launch_marg_elementwise(1, m, m, d_V.p, d_Vs.p, d_ev.p, nullptr, nullptr, eps, st);
    e->launches += ctvio::launch_dense_gemm(m, m, m, 1.0, d_Vs.p, m, false, d_V.p, m, true, 0.0, d_Ainv.p, m, st);
    // T = Arm * Amm_inv ; A' = Arr - T * Amr ; b' = brr - T * bmm
    e->launches += ctvio::launch_dense_gemm(n, m, m, 1.0, d_A.p + size_t(m) * P, P, false, d_Ainv.p, m, false, 0.0, d_T.p, m, st);
    e->launches += ctvio::launch_dense_gemm(n, n, m, -1.0, d_T.p, m, false, d_A.p + m, P, false, 1.0, d_Ap.p, n, st);
    e->launches += ctvio::launch_dense_gemm(n, 1, m, -1.0, d_T.p, m, false, d_b.p, 1, false, 1.0, d_bp.p, 1, st);
  }
  CUDA_OK(d_Ap2.reserve(size_t(n) * n)); CUDA_OK(d_V2.reserve(size_t(n) * n)); CUDA_OK(d_ev2.reserve(n));
  CUDA_OK(d_vb.reserve(n)); CUDA_OK(d_J.reserve(size_t(n) * n)); CUDA_OK(d_r.reserve(n));
  e->launches += ctvio::launch_marg_elementwise(2, n, n, d_Ap.p, d_Ap2.p, nullptr, nullptr, nullptr, eps, st);
  CUDA_OK(ws.eig_scratch.reserve(ctvio::jacobi_log_bytes(n, 40) / sizeof(double) + 1));
  e->launches += ctvio::launch_jacobi_eig(d_Ap2.p, d_V2.p, d_ev2.p, n, ws.eig_scratch.p, st);
  e->launches += ctvio::launch_dense_gemm(n, 1, n, 1.0, d_V2.p, n, true, d_bp.p, 1, false, 0.0, d_vb.p, 1, st);
  e->launches += ctvio::launch_marg_elementwise(3, n, n, d_V2.p, d_J.p, d_ev2.p, d_vb.p, d_r.p, eps, st);
  rc = read_scalars(e);
  if (rc) return rc;

  // ---- the new prior: kept blocks with the current state as linearisation point; J_lin / r_lin / x0 STAY in HBM
  //      (ctvio_adopt_prior hands them over device-to-device, ctvio_get_prior fetches them on demand) ----
  ctvio::PriorHost& np_ = e->new_prior;
  np_.n = n;
  e->new_prior_on_host = false;
  for (const auto& kv : blocks) {
    if (kv.second.dropped) continue;
    np_.type.push_back(kv.first.type);
    np_.index.push_back(kv.first.index);
    np_.col.push_back(kv.second.pos - m);
  }
  {
    DevBuf<int32_t>&d_t = ws.pos_cam, &d_i = ws.pos_lm;  // free again: reuse as block type / index uploads
    CUDA_OK(d_t.upload(np_.type, st));
    CUDA_OK(d_i.upload(np_.index, st));
    CUDA_OK(e->d_newprior_x0.reserve(4 * np_.type.size()));
    e->launches += ctvio::launch_prior_x0(e->x[e->cur].ptrs(), d_t.p, d_i.p, int(np_.type.size()), e->d_newprior_x0.p, st);
    CUDA_OK(cudaStreamSynchronize(st));  // the uploads above come from host vectors that are reused by the next call
  }
  *n_out = n;
  *nb_out = int32_t(np_.type.size());
  return CTVIO_OK;
}
int ctvio_get_prior(ctvio_handle e, double* J, double* r, int32_t* type, int32_t* index, int32_t* col, double* x0) {
  if (!e) return fail(CTVIO_ERR_INVALID, "null handle");
  if (e->new_prior.n <= 0) return fail(CTVIO_ERR_STATE, "no prior has been produced");
  cudaSetDevice(e->cfg.device);
  {
    const int rc = fetch_new_prior(e);
    if (rc) return rc;
  }
  const ctvio::PriorHost& p = e->new_prior;
  if (J) std::memcpy(J, p.J.data(), p.J.size() * sizeof(double));
  if (r) std::memcpy(r, p.r.data(), p.r.size() * sizeof(double));
  if (type) std::memcpy(type, p.type.data(), p.type.size() * sizeof(int32_t));
  if (index) std::memcpy(index, p.index.data(), p.index.size() * sizeof(int32_t));
  if (col) std::memcpy(col, p.col.data(), p.col.size() * sizeof(int32_t));
  if (x0) std::memcpy(x0, p.x0.data(), p.x0.size() * sizeof(double));
  return CTVIO_OK;
}
int ctvio_adopt_prior(ctvio_handle e) {
  if (!e) return fail(CTVIO_ERR_INVALID, "null handle");
  if (e->new_prior.n <= 0) return fail(CTVIO_ERR_STATE, "no prior has been produced");
  cudaSetDevice(e->cfg.device);
  // device-to-device: the buffers of the marginalization workspace BECOME the active prior (pointer swap), only the
  // block bookkeeping (a few dozen ints) lives on the host
  e->prior.n = e->new_prior.n;
  e->prior.type = e->new_prior.type; e->prior.index = e->new_prior.index; e->prior.col = e->new_prior.col;
  e->prior.J.clear(); e->prior.r.clear(); e->prior.x0.clear();
  std::swap(e->d_prior_J.p, e->mws.J.p); std::swap(e->d_prior_J.cap, e->mws.J.cap);
  std::swap(e->d_prior_r.p, e->mws.r.p); std::swap(e->d_prior_r.cap, e->mws.r.cap);
  std::swap(e->d_prior_x0.p, e->d_newprior_x0.p); std::swap(e->d_prior_x0.cap, e->d_newprior_x0.cap);
  e->prior_on_device = true;
  e->new_prior = ctvio::PriorHost();  // its device buffers are gone
  e->prior_dirty = true;
  e->masks_dirty = true;
  return CTVIO_OK;
}

int ctvio_set_deterministic(ctvio_handle e, int32_t on) {
  if (!e) return fail(CTVIO_ERR_INVALID, "null handle");
  if (e->world > 1 && on) return fail(CTVIO_ERR_STATE, "deterministic mode is single-GPU");
  e->deterministic = on != 0;
  e->structure_dirty = true;  // K1 work items are rebuilt with single-round chunks
  return CTVIO_OK;
}

int ctvio_enable_prior(ctvio_handle e, int32_t on) {
  if (!e) return fail(CTVIO_ERR_INVALID, "null handle");
  if (e->prior_enabled != (on != 0)) e->masks_dirty = true;
  e->prior_enabled = on != 0;
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
    // grow both state buffers, keeping the current contents (reserve() reallocates without copying)
    for (int b = 0; b < 2; ++b) {
      DevState& x = e->x[b];
      if (x.q.cap < 4 * size_t(n) || x.p.cap < kPStride * size_t(n) || x.tab.cap < size_t(n)) {
        DevBuf<double> nq, np_;
        DevBuf<KnotPair> nt;
        CUDA_OK(nq.reserve(4 * size_t(n) + 64)); CUDA_OK(np_.reserve(kPStride * size_t(n) + 64)); CUDA_OK(nt.reserve(size_t(n) + 16));
        if (b == e->cur) {
          CUDA_OK(cudaMemcpyAsync(nq.p, x.q.p, 4 * size_t(old) * sizeof(double), cudaMemcpyDeviceToDevice, e->stream));
          CUDA_OK(cudaMemcpyAsync(np_.p, x.p.p, kPStride * size_t(old) * sizeof(double), cudaMemcpyDeviceToDevice, e->stream));
        }
        CUDA_OK(cudaStreamSynchronize(e->stream));
        std::swap(x.q.p, nq.p); std::swap(x.q.cap, nq.cap);
        std::swap(x.p.p, np_.p); std::swap(x.p.cap, np_.cap);
        std::swap(x.tab.p, nt.p); std::swap(x.tab.cap, nt.cap);
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
    if (e->x[b].bias.cap < 6 * size_t(std::max(nB_new, 1))) {
      DevBuf<double> nb;
      CUDA_OK(nb.reserve(6 * size_t(nB_new) + 96));
      if (b == e->cur && e->nB) CUDA_OK(cudaMemcpyAsync(nb.p, e->x[b].bias.p, 6 * size_t(e->nB) * sizeof(double), cudaMemcpyDeviceToDevice, e->stream));
      CUDA_OK(cudaStreamSynchronize(e->stream));
      std::swap(e->x[b].bias.p, nb.p); std::swap(e->x[b].bias.cap, nb.cap);
    }
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
    if (t == CTVIO_BLK_ROT || t == CTVIO_BLK_POS) e->prior.index[b] -= drop_knots;
    else if (t == CTVIO_BLK_BG || t == CTVIO_BLK_BA) e->prior.index[b] -= drop_bias;
    if ((t <= CTVIO_BLK_BA) && e->prior.index[b] < 0) return fail(CTVIO_ERR_STATE, "a block of the active prior left the window");
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
  for (int b = 0; b < 2; ++b) CUDA_OK(e->x[b].rho.reserve(size_t(std::max(n_new, e->nL)) + 1) == cudaSuccess ? cudaSuccess : cudaErrorMemoryAllocation);
  if (n_new) {
    CUDA_OK(cudaMemcpyAsync(e->d_tmp.p, init_rho, size_t(n_new) * sizeof(double), cudaMemcpyHostToDevice, st));
    CUDA_OK(cudaMemcpyAsync(e->d_tri_idx.p, old_index, size_t(n_new) * sizeof(int32_t), cudaMemcpyHostToDevice, st));
    e->h2d_bytes += size_t(n_new) * 12;
    // gather into the other state buffer's array, then swap the pointers (no aliasing)
    e->launches += ctvio::launch_remap_rho(e->x[e->cur].rho.p, e->d_tri_idx.p, e->d_tmp.p, n_new, e->x[other].rho.p, st);
    CUDA_OK(cudaStreamSynchronize(st));
    std::swap(e->x[e->cur].rho.p, e->x[other].rho.p);
    std::swap(e->x[e->cur].rho.cap, e->x[other].rho.cap);
  }
  if (n_new != e->nL) e->structure_dirty = true;
  e->mirror_valid = false;
  e->nL = n_new;
  e->have_rho = true;
  return CTVIO_OK;
}

// ---- wire-format ingestion (SURVEY 8f-4) ----------------------------------------------------------
int ctvio_ingest_feature_cloud(ctvio_handle e, int32_t slot, int64_t t_ns, int32_t n, const float* points, const float* ch_id,
                               const float* ch_u, const float* ch_v, const float* ch_vx, const float* ch_vy) {
  (void)ch_u; (void)ch_vx; (void)ch_vy;  // carried by the message, not used by the estimator's factors
  if (!e || slot < 0 || slot >= ctvio_engine::kFrameSlots || n < 0 || n > ctvio_engine::kFrameCap ||
      (n > 0 && (!points || !ch_id || !ch_v)))
    return fail(CTVIO_ERR_INVALID, "bad feature cloud");
  cudaSetDevice(e->cfg.device);
  cudaStream_t st = e->stream;
  CUDA_OK(e->d_frames.reserve(size_t(ctvio_engine::kFrameSlots) * ctvio_engine::kFrameCap));
  CUDA_OK(e->d_frame_t.reserve(ctvio_engine::kFrameSlots));
  CUDA_OK(e->d_cloud_stage.reserve(5 * size_t(ctvio_engine::kFrameCap)));
  e->h_frame_t[slot] = t_ns;
  e->h_frame_n[slot] = n;
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
  CUDA_OK(cudaStreamSynchronize(st));  // the caller's message buffers may go away
  return CTVIO_OK;
}

int ctvio_add_image_features_from_slots(ctvio_handle e, int32_t n, const int32_t* slot_i, const int32_t* idx_i,
                                        const int32_t* slot_j, const int32_t* idx_j, const int32_t* lm, const int32_t* marg) {
  if (!e || n < 0 || (n > 0 && (!slot_i || !idx_i || !slot_j || !idx_j || !lm))) return fail(CTVIO_ERR_INVALID, "null argument");
  if (!e->img.empty() && e->img_desc.empty()) return fail(CTVIO_ERR_STATE, "image factors with host payload are already present");
  for (int k = 0; k < n; ++k) {
    const int si = slot_i[k], sj = slot_j[k];
    if (si < 0 || si >= ctvio_engine::kFrameSlots || sj < 0 || sj >= ctvio_engine::kFrameSlots || idx_i[k] < 0 ||
        idx_i[k] >= e->h_frame_n[si] || idx_j[k] < 0 || idx_j[k] >= e->h_frame_n[sj])
      return fail(CTVIO_ERR_INVALID, "feature slot / index out of range");
    HostImage o{e->h_frame_t[si], e->h_frame_t[sj], 0, 0, {0, 0}, {0, 0}, lm[k], marg ? marg[k] : 0};
    e->img.push_back(o);
    e->img_desc.push_back(ctvio::FactorDesc{si * ctvio_engine::kFrameCap + idx_i[k], sj * ctvio_engine::kFrameCap + idx_j[k], lm[k],
                                            marg ? marg[k] : 0});
  }
  e->structure_dirty = true;
  return CTVIO_OK;
}

int ctvio_ingest_imu(ctvio_handle e, int32_t n, const void* records, int32_t stride, int32_t off_gyro, int32_t off_accel,
                     int64_t drop_before_ns) {
  if (!e || n < 0 || (n > 0 && !records) || stride < 56 || off_gyro < 8 || off_accel < 8 || off_gyro + 24 > stride ||
      off_accel + 24 > stride)
    return fail(CTVIO_ERR_INVALID, "bad IMU record layout");
  cudaSetDevice(e->cfg.device);
  cudaStream_t st = e->stream;
  // retire samples older than drop_before_ns (RemoveIMUData, trajectory_manager.cpp:472-475): a device-side shift
  size_t keep_from = 0;
  while (keep_from < e->h_imu_tab_t.size() && e->h_imu_tab_t[keep_from] < drop_before_ns) ++keep_from;
  const size_t kept = e->h_imu_tab_t.size() - keep_from, total = kept + size_t(n);
  if (e->d_imu_tab_t.cap < total) {
    DevBuf<longlong2> nt;
    DevBuf<double2> ng;
    CUDA_OK(nt.reserve(2 * total + 256)); CUDA_OK(ng.reserve(3 * (2 * total + 256)));
    if (kept) {
      CUDA_OK(cudaMemcpyAsync(nt.p, e->d_imu_tab_t.p + keep_from, kept * sizeof(longlong2), cudaMemcpyDeviceToDevice, st));
      CUDA_OK(cudaMemcpyAsync(ng.p, e->d_imu_tab_ga.p + 3 * keep_from, 3 * kept * sizeof(double2), cudaMemcpyDeviceToDevice, st));
    }
    CUDA_OK(cudaStreamSynchronize(st));
    std::swap(e->d_imu_tab_t.p, nt.p); std::swap(e->d_imu_tab_t.cap, nt.cap);
    std::swap(e->d_imu_tab_ga.p, ng.p); std::swap(e->d_imu_tab_ga.cap, ng.cap);
  } else if (keep_from > 0 && kept > 0) {
    CUDA_OK(e->d_tmp.reserve(8 * kept));
    e->launches += ctvio::launch_shift_imu_table(e->d_imu_tab_t.p, e->d_imu_tab_ga.p, int(keep_from), int(kept), e->d_tmp.p, st);
  }
  e->h_imu_tab_t.erase(e->h_imu_tab_t.begin(), e->h_imu_tab_t.begin() + keep_from);
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
    CUDA_OK(cudaStreamSynchronize(st));
  }
  return CTVIO_OK;
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

int ctvio_transfer_stats(ctvio_handle e, int64_t* h2d_bytes, int64_t* d2h_bytes, int32_t reset) {
  if (!e) return fail(CTVIO_ERR_INVALID, "null handle");
  if (h2d_bytes) *h2d_bytes = int64_t(e->h2d_bytes + g_upload_bytes);
  if (d2h_bytes) *d2h_bytes = int64_t(e->d2h_bytes);
  if (reset) { e->h2d_bytes = e->d2h_bytes = 0; g_upload_bytes = 0; }
  return CTVIO_OK;
}

int ctvio_nccl_unique_id(uint8_t* id128) {
  if (!id128) return fail(CTVIO_ERR_INVALID, "null argument");
  std::string err;
  if (!ctvio::comm_unique_id(id128, &err)) return fail(CTVIO_ERR_NCCL, err);
  return CTVIO_OK;
}
int ctvio_comm_init(ctvio_handle e, int32_t rank, int32_t world, const uint8_t* id128) {
  if (!e || !id128 || world < 1 || rank < 0 || rank >= world) return fail(CTVIO_ERR_INVALID, "bad argument");
  cudaSetDevice(e->cfg.device);
  std::string err;
  void* comm = ctvio::comm_create(rank, world, id128, &err);
  if (!comm) return fail(CTVIO_ERR_NCCL, err);
  ctvio::comm_destroy(e->nccl_comm);
  e->nccl_comm = comm;
  e->rank = rank;
  e->world = world;
  e->shard_checked = false;
  return CTVIO_OK;
}

}  // extern "C"
