// Device data layout + kernel launch wrappers of the CUDA engine.
#pragma once
#include <cuda_runtime.h>

#include <atomic>

#include <cstdint>
#include <utility>

#include "param_blocks.h"
#include "spline_eval.cuh"

namespace ctvio {

constexpr int kPStride = 4;        // knot positions are stored [N][4] (32 B) so that TMA windows are 16-B aligned
constexpr int kVisThreads = 256;   // visual kernel CTA: 128 lane pairs
constexpr int kVisObsPerRound = 128;
constexpr int kVisMinChunk = 64;  // smallest chunk a frame-pair group is cut into to fill the SMs (engine.cu); 32 tips the
                                  // ill-conditioned window 8 of the re-anchoring runner into divergence (DESIGN §6)
constexpr int kLocalDim = 64;      // padded local Jacobian width of one frame-pair group
constexpr int kRowStride = 66;     // shared-memory stride of one Jacobian row (doubles); 16-B aligned
constexpr int kObsStride = 2 * kRowStride + 2;  // stride of one observation's 2 rows: 268 words -> 2-way store conflicts instead of 16-way
constexpr int kWinKnots = 5;       // knots of a padded evaluation window (se3_spline.h:463-503 with 39 ms padding)
constexpr int kColLd = 60, kColR = 61, kColRho = 62;
constexpr int kCholNB = 64;

// ---- state at one linearisation point (all HBM) ------------------------------------------------
struct StatePtrs {
  double* q;       // [nK][4] xyzw
  double* p;       // [nK][4] xyz + pad
  double* bias;    // [nB][6]
  double* rho;     // [nL]
  double* ld;      // [1]
  KnotPair* tab;   // [nK-1] knot-pair table of this state
};

// the state of a parameter block (param_blocks.h): a knot's quaternion or position, a bias node's gyro or accel bias,
// the line delay, an inverse depth
__device__ __forceinline__ const double* block_state(const StatePtrs& st, int type, int index) {
  switch (type) {
    case CTVIO_BLK_ROT: return st.q + 4 * index;
    case CTVIO_BLK_POS: return st.p + kPStride * index;
    case CTVIO_BLK_BG: return st.bias + 6 * index;
    case CTVIO_BLK_BA: return st.bias + 6 * index + 3;
    case CTVIO_BLK_LD: return st.ld;
    default: return st.rho + index;
  }
}

// dx = x [-] x0 of a prior block at state x, linearised at x0 (marginalization_factor.cpp:326-373): the rotation's
// quaternion box-minus, a plain difference otherwise
__device__ __forceinline__ void prior_block_dx(int type, const double* x, const double* x0, double* dx) {
  if (type == CTVIO_BLK_ROT) {
    const double n2 = x0[0] * x0[0] + x0[1] * x0[1] + x0[2] * x0[2] + x0[3] * x0[3];
    const double ax = -x0[0] / n2, ay = -x0[1] / n2, az = -x0[2] / n2, aw = x0[3] / n2;
    const double bx = x[0], by = x[1], bz = x[2], bw = x[3];
    const double qx = aw * bx + ax * bw + ay * bz - az * by;
    const double qy = aw * by + ay * bw + az * bx - ax * bz;
    const double qz = aw * bz + az * bw + ax * by - ay * bx;
    const double qw = aw * bw - ax * bx - ay * by - az * bz;
    const double sg = (qw >= 0) ? 2.0 : -2.0;
    dx[0] = sg * qx; dx[1] = sg * qy; dx[2] = sg * qz;
  } else {
    for (int d = 0; d < block_dim(type); ++d) dx[d] = x[d] - x0[d];
  }
}

// ---- Schur-form normal equations at one linearisation point -------------------------------------
struct NormalEqPtrs {
  double* A;     // [np][np] camera block, UPPER triangle valid (row <= col), unscaled
  double* gc;    // [np]
  double* hl;    // [nL]  landmark diagonal
  double* gl;    // [nL]  landmark gradient
  double* wld;   // [nL]  landmark x line-delay coupling
  double* W;     // landmark x knot coupling, compact per landmark over its knot-dim range [lo, hi)
  double* cost;  // [1]
};

// image observations, sorted by frame-pair group; SoA, 16-byte vector loads (64 B / obs + 8 B rho gather)
struct ImageObsPtrs {
  const longlong2* t;     // {ti, tj}
  const double2* pi;      // anchor bearing xy
  const double2* pj;      // observation xy
  const int4* meta;       // {rowi, rowj, landmark, marg}
  int32_t n;
};

struct VisualItem {  // one CTA work item: a chunk of one frame-pair group
  int32_t start, count;
  int32_t wi0, wj0;  // first knot of the padded anchor / observation windows
};

struct ImuObsPtrs {
  const longlong2* t_node;  // {t, bias node}; sorted by (start knot, bias node)
  const double2* ga;        // [n][3] double2: {gx,gy},{gz,ax},{ay,az}
  int32_t n;
};

struct ImuItem {  // one CTA work item: samples sharing the start knot and the bias node
  int32_t start, count;
  int32_t s, node;
};
constexpr int kImuMaxPerItem = 32;

struct BiasFactorPtrs {
  const int2* ij;
  const double* sqrt_info;  // [n][6]
  int32_t n;
};

struct PriorPtrs {
  int32_t n, n_blocks;
  const double* J;       // [n][n] row-major
  const double* r;       // [n]
  const double* JtJ;     // [n][n]
  const int32_t* type;   // per block
  const int32_t* index;
  const int32_t* col;
  const double* x0;      // [n_blocks][4]
  const int32_t* col2g;  // [n] column -> camera dim (or -1)
  double* dx;            // [n] scratch
  double* res;           // [n] scratch
};

struct ProblemDims {
  int32_t nK, nB, nL, np, idx_bias0, idx_ld;
};

struct LandmarkLayout {
  const int32_t* lo;     // [nL] first camera dim of the landmark's knot range
  const int32_t* hi;     // [nL]
  const int64_t* woff;   // [nL+1] offsets into W
};

// K4 list entry: a landmark with its coupling-row layout inlined (one load instead of a chain of three)
struct SchurEntry {
  int32_t l, lo, hi, pad;
  int64_t woff;  // offset of W_l[lo] in the compact coupling array
};
// K4 work item: part of the landmark list of one 64x64 output tile (ti >= tj) of the reduced system
struct SchurTileItem {
  int32_t ti, tj;        // block row / column of the tile
  int32_t first, count;  // landmark ids schur_list[first, first + count)
};

// scalars exchanged with the host once per LM step
struct LmScalars {
  double cost_eval;        // cost accumulated by the last evaluation pass
  double gd;               // g' delta
  double dHd;              // delta' H delta
  double step_norm2;       // |x - x+|^2 (ambient, active blocks)
  double x_norm2;          // |x|^2 (ambient, active blocks)
  double err_sum;          // (sharded mode) error flag as a double so that it can ride in the scalar all-reduce
  double gmax;             // max |g| over active dims (bounds-projected for the line delay)
  double dir_max;          // max |delta|
  double ld_value;         // line delay of the candidate state
  int32_t chol_fail;       // non-positive pivot / non-finite
  int32_t error_flags;     // bit0: factor time outside its window / spline
  int32_t pad[2];
};
// host-visible copy of the scalar block (mapped pinned memory) with a sequence number: the last kernel of an LM step
// writes it directly, the host spins on `seq` instead of paying a device-to-host copy plus a stream synchronisation
// Step decision of the LM driver, taken on the device by the last kernel of a step (gradient_norm_kernel) so that the
// linear solve of the NEXT step can be enqueued before the host has seen this step's scalars (pipelined driver,
// engine.cu): the speculated reduced_system_kernel reads `radius_next` from device memory.
struct LmDecision {
  double radius_next;         // trust-region radius after an accepted step (Ceres 1.14 trust_region_minimizer.cc)
  double model_cost_change;   // -g'd - d'Hd / 2
  double rho;                 // relative decrease (cost(x) - cost(x + d)) / model_cost_change
  int32_t valid;              // the linear solve succeeded and the model decreases
  int32_t accept;             // valid and rho > min_relative_decrease
  int32_t go;                 // accept, and none of the termination tests fires: the speculated next step is needed
  int32_t pad;
};
struct LmDecideArgs {
  LmDecision* dec;            // device copy (null: no decision is taken)
  double x_cost, radius;      // cost and radius at the current point
  double min_relative_decrease, max_radius;
  double parameter_tolerance, function_tolerance, gradient_tolerance, min_radius;
};
struct LmPublished {
  LmScalars s;
  LmDecision dec;
  unsigned long long seq;
  double rcond;  // written by ctvio_covariance only: pivot ratio of the factored reduced system
};
constexpr int kLmSumScalars = 6;  // cost_eval, gd, dHd, step_norm2, x_norm2, err_sum: plain sums over landmark shards

// Per-device one-time initialisation (cudaFuncSetAttribute applies to the CURRENT device only; one process may
// drive several GPUs) and a cached SM count of the current device.
struct PerDeviceOnce {
  std::atomic<unsigned long long> mask{0};
  bool first() {
    int d = 0;
    cudaGetDevice(&d);
    const unsigned long long bit = 1ull << (d & 63);
    return !(mask.fetch_or(bit) & bit);
  }
};
inline int device_sm_count() {
  static std::atomic<int> cache[64];
  int d = 0;
  cudaGetDevice(&d);
  int v = cache[d & 63].load(std::memory_order_relaxed);
  if (v == 0) {
    cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, d);
    cache[d & 63].store(v, std::memory_order_relaxed);
  }
  return v;
}

// ---- deterministic mode (ctvio_set_deterministic): the fp64 atomics that merge CTA partial sums are kept, but the CTAs
// of a kernel perform their flush in BLOCK-INDEX ORDER (a ticket in global memory: CTA i flushes after CTA i-1 has
// flushed and fenced), so every sum is accumulated in one fixed order and a solve is bit-reproducible run to run.
// Blocks are dispatched in index order, so a waiting CTA's predecessors are always resident or done (no deadlock).
// The serialised flush costs time (K1 runs several times longer at C2); it is a verification / regression mode, off by default.
#if defined(__CUDACC__)
__device__ __forceinline__ int ld_acquire_gpu(const int* p) {
  int v;
  asm volatile("ld.acquire.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_release_gpu(int* p, int v) {
  asm volatile("st.release.gpu.global.s32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ void spin_until_gpu(const int* p, int v) {
  while (ld_acquire_gpu(p) != v) {}
}
__device__ __forceinline__ void det_ticket_wait(const int* ticket, int my) {
  if (!ticket) return;
  if (threadIdx.x == 0) spin_until_gpu(ticket, my);
  __syncthreads();
}
__device__ __forceinline__ void det_ticket_done(int* ticket, int my) {
  if (!ticket) return;
  __threadfence();   // this thread's atomics are performed before the ticket moves on
  __syncthreads();
  if (threadIdx.x == 0) st_release_gpu(ticket, my + 1);
}
// programmatic dependent launch (see launch_chained): both are no-ops in a kernel that was launched without it
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
// reductions over the 32 lanes of a full warp, one fixed xor-shuffle tree: every lane gets the same, reproducible value
__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ double warp_min_d(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmin(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ double warp_max_d(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
#endif

// ---- programmatic dependent launch (PDL) on the pipelined LM driver's main stream ---------------
// pdl = true: the kernel may be launched while the kernel before it on the stream is still running, and runs the part of
// it in front of pdl_wait() early; pdl_wait() returns when that kernel has completed and its writes are visible.
// The rule every kernel launched this way follows:
//   nothing before pdl_wait() reads a buffer the immediately preceding kernel writes, and nothing before it writes a
//   buffer that kernel reads; pdl_launch_dependents() comes no earlier than right after the kernel's own pdl_wait(),
//   and every thread passes pdl_wait() before it exits.
// So a kernel's successor is let in only after everything two launches back has completed: data written two or more
// kernels back may be read before the wait.  The deterministic, sharded and line-search paths launch plainly.
#if defined(__CUDACC__)
template <typename... KArgs, typename... Args>
cudaError_t launch_chained(bool pdl, void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t s,
                           Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = s;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = at;
  cfg.numAttrs = pdl ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kernel, std::forward<Args>(args)...);
}
#endif

// ---- launch wrappers (each returns the number of kernels it launched) ----------------------------
int launch_knot_table(const StatePtrs& st, int nK, cudaStream_t s);

struct VisualLaunch {
  ImageObsPtrs obs;
  const VisualItem* items;
  int32_t n_items;
  StatePtrs st;
  NormalEqPtrs ne;
  LandmarkLayout lm;
  ProblemDims dims;
  SplineParams sp;
  RigParams rig;
  double cauchy;
  const uint8_t* cmask;   // [np] 1 = constant
  LmScalars* scal;
  int* det_ticket = nullptr;  // deterministic mode: flush in block order
};
int launch_visual(const VisualLaunch& a, bool full, cudaStream_t s);
size_t visual_smem_bytes();

struct ImuLaunch {
  ImuObsPtrs obs;
  const ImuItem* items;
  int32_t n_items;
  StatePtrs st;
  NormalEqPtrs ne;
  ProblemDims dims;
  SplineParams sp;
  RigParams rig;
  const uint8_t* cmask;
  LmScalars* scal;
  int* det_ticket = nullptr;
};
int launch_imu(const ImuLaunch& a, bool full, cudaStream_t s);

struct SmallFactorsLaunch {
  BiasFactorPtrs bf;
  PriorPtrs prior;
  StatePtrs st;
  NormalEqPtrs ne;
  ProblemDims dims;
  const uint8_t* cmask;
  LmScalars* scal;
  int deterministic = 0;  // one thread walks the bias factors / prior columns in order
};
int launch_small_factors(const SmallFactorsLaunch& a, bool full, cudaStream_t s);

// probes (parity tests): per-factor residuals / Jacobians in the C-ABI layout, original factor order
int launch_probe_image(const VisualLaunch& a, const int32_t* orig_index, bool want_jac, double* r, int32_t* s,
                       double* J, cudaStream_t st);
int launch_probe_imu(const ImuLaunch& a, const int32_t* orig_index, bool want_jac, double* r, int32_t* s, double* J,
                     cudaStream_t st);

// ---- linear algebra / LM step -------------------------------------------------------------------
struct LinearLaunch {
  ProblemDims dims;
  NormalEqPtrs ne;
  LandmarkLayout lm;
  const SchurEntry* schur_list; // concatenated per-tile landmark lists
  const SchurTileItem* schur_items;
  int32_t n_schur_items;
  int32_t* m_flags;             // [reduced_system_flags_len] K4: tile (ti, tj) of M written (epoch valued, zeroed once)
  const uint8_t* cmask;
  const uint8_t* active;        // [np + nL]
  double* sc;                   // [np] Jacobi scale
  double* sl;                   // [nL]
  double* M;                    // [npad][npad] reduced system, LOWER triangle of 64x64 tiles valid (diagonal tiles full)
  double* Linv;                 // barrier kernel: [npad/NB][NB][NB] inverses of the diagonal Cholesky blocks;
                                // tile-DAG kernel: the per-step packets of the diagonal factorisations (chol_dag_lpub_len)
  double* rhs;                  // [npad]
  double* y;                    // [npad]
  double* yf;                   // [npad] forward-solved right-hand side
  double* chol_part;            // workspace of the tile-DAG Cholesky (chol_dag_part_len doubles); null -> barrier kernel
  int32_t* chol_flags;          // its dependency flags (chol_dag_flags_len ints, zero-initialised once)
  unsigned* chol_seq;           // host counter of tile-DAG launches on this engine (packet buffer parity); may be null
  double* hh;                   // [nL] damped landmark diagonals
  double* diagA;                // [npad] camera diagonal (sharded mode: all-reduced with M and rhs); may be null
  int32_t sharded;              // != 0: M is built WITHOUT damping / identity rows (they are added after the all-reduce)
  double* dc;                   // [np] step (camera dims)
  double* dl;                   // [nL]
  int32_t npad;
  LmScalars* scal;
  int* det_ticket;              // deterministic mode (K4 parts, step kernels): flush in block order; else null
  const int32_t* go;            // speculated step only: &LmDecision::go - the expensive kernels return at once when it is 0
  int32_t pdl = 0;              // pipelined driver: the step's kernels are chained by launch_chained(pdl = true)
};
int launch_jacobi_scale(const LinearLaunch& a, cudaStream_t s);
// builds the damped, scaled reduced system, factors it, solves and back-substitutes: dc, dl, gd, dHd
int launch_lm_step(const LinearLaunch& a, double radius, cudaStream_t s);
// the three stages of launch_lm_step, separately launchable for measurement
// radius_dev != null: the radius is read from device memory (first double of an LmDecision)
int launch_reduced_system(const LinearLaunch& a, double radius, cudaStream_t s, const double* radius_dev = nullptr);
size_t reduced_system_flags_len(int npad);  // ints of LinearLaunch::m_flags
// tile_dag (may be null): set to whether the tile-DAG kernel ran (else the barrier kernel) - the two leave the factor in
// different layouts (CholDagArgs::M in chol_dag.cu, the header of chol_coop.cu)
int launch_factor_solve(const LinearLaunch& a, cudaStream_t s, bool* tile_dag = nullptr);
// tile-DAG variant (chol_dag.cu): usable when every tile gets its own SM
bool chol_dag_supported(int npad, int n_sm);
size_t chol_dag_part_len(int npad);
size_t chol_dag_flags_len(int npad);
size_t chol_dag_lpub_len(int npad);  // doubles of LinearLaunch::Linv: [block inverses of the barrier kernel | 2 packet buffers]
int launch_chol_dag_init(double* linv_buf, double* part_buf, int npad, cudaStream_t s);  // message buffers <- sentinels, once per allocation
int launch_chol_dag(const LinearLaunch& a, cudaStream_t s, bool* tile_dag = nullptr);
// the packet buffer (packets [nb][4][16][80], layout in chol_tiles.cuh) of the last tile-DAG launch on this engine
const double* chol_dag_last_packets(const double* linv_buf, int npad, unsigned chol_seq);

// ---- marginal covariance (covariance.cu, ctvio_covariance) ----------------------------------------
struct CovLaunch {
  int32_t np, npad, nL, idx_ld;
  const double* M;         // K5's factor: strictly-lower tiles of L (transposed inside the slot if tile_dag)
  const double* Linv;      // barrier kernel: [nb][64][64] inverses of the diagonal blocks of L
  const double* packets;   // tile-DAG kernel: the packets of its diagonal factorisations
  int32_t tile_dag;
  const uint8_t* cmask;    // [np] 1 = no covariance (held constant, or touched by no factor)
  const double* sc;        // [np] Jacobi scale the reduced system was formed with
  double* X;               // [npad][npad] L^-1, lower tiles
  double* piv;             // [nb][2] min / max of 1 / L_ii over the block's free dims
  double* cov;             // [np][np] camera-side covariance, both triangles
};
// cmask = !active over [0, np), and 1 on the first n_gauge dims (knots held constant for one call only)
int launch_cov_mask(const uint8_t* active, int np, int n_gauge, uint8_t* cmask, cudaStream_t s);
int launch_cov_inverse(const CovLaunch& c, cudaStream_t s);  // X, piv, cov
struct LandmarkVarLaunch {
  int32_t np, nL, idx_ld;
  const double* cov;
  NormalEqPtrs ne;
  LandmarkLayout lm;
  const uint8_t* active;   // [np + nL]
  double* var;             // [nL]
  LmScalars* scal;         // chol_fail is set when a landmark with a factor has h_l <= 0
};
int launch_landmark_variance(const LandmarkVarLaunch& v, cudaStream_t s);
// rcond = (min / max of the pivots)^2 from piv, then the scalar block + rcond to *pub with sequence number seq
int launch_cov_publish(const double* piv, int nb, const LmScalars* scal, LmPublished* pub, unsigned long long seq,
                       cudaStream_t s);
// ctvio_pose_covariance: one warp per time, out[n][12][12] = J(t) Sigma_sub J(t)' (PoseJacobian, spline_eval.cuh)
struct PoseCovLaunch {
  StatePtrs st;
  SplineParams sp;
  M3 R_CI;
  V3 p_CI;
  int32_t n, np, camera_frame;
  const int64_t* t;        // [n], inside the spline (checked by the caller)
  const double* cov;       // [np][np] the window covariance
  double* out;             // [n][144]
};
int launch_pose_cov(const PoseCovLaunch& a, cudaStream_t s);
// ctvio_relative_pose_covariance: one warp per pair, out[n][6][6] = G Sigma_U G' of the pose at t_b in the frame of the
// pose at t_a, Sigma_U the block of the window covariance at the union of the two segments' knots
// (relative_pose_jacobian_column, spline_eval.cuh), and cross[n][6][6] = J_a Sigma_ab J_b' of the two poses
struct RelativePoseCovLaunch {
  StatePtrs st;
  SplineParams sp;
  M3 R_CI;
  V3 p_CI;
  int32_t n, np, camera_frame;
  const int64_t* t_a;      // [n], inside the spline (checked by the caller)
  const int64_t* t_b;      // [n], inside the spline (checked by the caller)
  const double* cov;       // [np][np] the window covariance
  double* out;             // [n][36]
  double* cross;           // [n][36] or null
};
int launch_relative_pose_cov(const RelativePoseCovLaunch& a, cudaStream_t s);
// ctvio_point_covariance / ctvio_feature_table_point_covariance: one warp per point, out[n][3][3] = G Sigma_25 G' of the
// world point of landmark l anchored at time t with bearing (x, y, 1) (point_jacobian_column, spline_eval.cuh), Sigma_25
// the joint covariance of its segment's 24 knot dims and rho_l
struct FrameFeature;  // frontend.h
struct PointCovLaunch {
  StatePtrs st;
  SplineParams sp;
  M3 R_CI;
  V3 p_CI;
  int32_t n, np, idx_ld;
  // per point either the caller's arrays (landmark != null) ...
  const int32_t* landmark; // [n] 0 .. nL - 1
  const int64_t* t;        // [n] anchor times, inside the spline (checked by the caller)
  const double* bearing;   // [n][2]
  // ... or point l = landmark l of the feature table's window, its anchor the first entry of its observation CSR, the
  // time the anchor slot's frame time (every held slot's time checked by the caller)
  const int32_t* obs_offset;
  const int32_t* obs_slot;
  const int32_t* obs_idx;
  const FrameFeature* table;  // [n_slots][frame_cap]
  const int64_t* frame_t;     // [n_slots]
  int32_t frame_cap;
  const double* cov;       // [np][np] the window covariance
  const double* var;       // [nL] the inverse-depth variances of the same call
  NormalEqPtrs ne;         // the coupling rows the covariance was formed from
  LandmarkLayout lm;
  const uint8_t* active;   // [np + nL]
  double* out;             // [n][9]
};
int launch_point_cov(const PointCovLaunch& a, cudaStream_t s);
int launch_chol_coop(const LinearLaunch& a, cudaStream_t s);
int launch_step_vectors(const LinearLaunch& a, cudaStream_t s);
// sharded mode: the iteration-0 Jacobi scale from the all-reduced camera diagonal (the LM damping and identity rows
// of constant / padding dims are added after the all-reduce by launch_shard_unpack, marginalize.h)
int launch_extract_diag(const LinearLaunch& a, cudaStream_t s);
int launch_jacobi_scale_from_diag(const LinearLaunch& a, cudaStream_t s);
// reset = false: the accumulator was already zeroed by reduced_system_kernel of the same LM step
// pub != nullptr: after the norm the whole scalar block is copied to *pub (mapped host memory) and pub->seq = seq
int launch_gradient_norm(const LinearLaunch& a, const StatePtrs& st, int fix_ld, double ld_lower, double ld_upper,
                         cudaStream_t s, bool reset = true, LmPublished* pub = nullptr, unsigned long long seq = 0,
                         const LmDecideArgs* decide = nullptr);

struct ApplyLaunch {
  int32_t count_camera;     // sharded mode: only rank 0 counts the (replicated) camera blocks in the norms
  ProblemDims dims;
  StatePtrs x, xc;          // current, candidate
  const double* dc;
  const double* dl;
  double alpha;
  const uint8_t* active;
  int32_t clamp_ld;
  double ld_lower, ld_upper;
  LmScalars* scal;
  int* det_ticket = nullptr;
};
int launch_apply_step(const ApplyLaunch& a, cudaStream_t s, bool reset = true);
// step vectors + full step (alpha = 1) applied in one launch; the per-step accumulators must already be zero
int launch_step_and_apply(const LinearLaunch& a, const ApplyLaunch& ap, cudaStream_t s);
int launch_gauge_realign(const StatePtrs& st, int nK, int min_idx, const double* R0_t0_dev, cudaStream_t s);
// ctvio_gauge_realign with R0 / t0 formed on the device from snap_dev = the knot's q (4), p (3) before the solve (the
// odometry cycle); the R0 / t0 it used go to R0_t0_out (12)
int launch_gauge_realign_snapshot(const StatePtrs& st, int nK, int min_idx, const double* snap_dev, double* R0_t0_out,
                                  cudaStream_t s);

struct QueryLaunch {
  StatePtrs st;
  SplineParams sp;
  int32_t n;
  const int64_t* t;
  double *q, *p, *omega, *vel, *acc;
  LmScalars* scal;
};
int launch_query(const QueryLaunch& a, cudaStream_t s);

}  // namespace ctvio
