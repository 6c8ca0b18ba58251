// Small host/device helpers shared by the engine's host code: the prior's host form (prior.cu), Gram kernel, gradient
// dot product, NCCL communicator wrappers.
#pragma once
#include <cuda_runtime.h>

#include <cstdint>
#include <string>
#include <vector>

#include "kernels.h"

namespace ctvio {

// MarginalizationInfo payload (factor/analytic_diff/marginalization_factor.h:96-131) in index-identity form
struct PriorHost {
  int n = 0;
  std::vector<double> J, r, x0;            // n x n row-major, n, n_blocks x 4
  std::vector<int32_t> type, index, col;   // per kept block
};

// G = J' J for a row-major rows x cols matrix (G: cols x cols)
int launch_gram(const double* J, int rows, int cols, double* G, cudaStream_t s);
// scal->gd = gc . dc + gl . dl  (directional derivative of the cost along the step, candidate buffers)
int launch_dot_gradient(const LinearLaunch& a, cudaStream_t s);

// ---- K7 marginalization (marginalize.cu) --------------------------------------------------------
struct MargImageArgs {
  ImageObsPtrs obs;
  const int32_t* marg_index;  // positions (in the sorted observation arrays) of the recorded factors
  int32_t n_marg;
  StatePtrs st;
  SplineParams sp;
  RigParams rig;
  double cauchy;              // CauchyLoss(1) for marginalized features (trajectory_estimator.cpp:321)
  const int32_t* pos_cam;     // [np] camera dim -> position in [dropped | kept] ordering, -1 = not a block
  const int32_t* pos_lm;      // [nL]
  int32_t idx_ld;
  double* Jrow;               // [R][ldj] row-compressed Jacobian, column P = residual; this factor owns rows row0 + 2 m ..
  int32_t ldj, row0;
  int32_t P;
  LmScalars* scal;
};
struct MargImuArgs {
  ImuObsPtrs obs;
  const int32_t* marg_index;
  int32_t n_marg;
  StatePtrs st;
  SplineParams sp;
  RigParams rig;
  const int32_t* pos_cam;
  int32_t idx_bias0;
  double* Jrow;
  int32_t ldj, row0;
  int32_t P;
  LmScalars* scal;
};
struct MargSmallArgs {
  const int2* bf_ij;          // recorded bias factors only
  const double* bf_s;
  int32_t n_bias;
  PriorPtrs prior;            // the old prior (dx / res scratch reused)
  int32_t use_prior;
  const int32_t* prior_pos;   // [prior.n] prior column -> position
  StatePtrs st;
  const int32_t* pos_cam;
  int32_t idx_bias0;
  double* Jrow;
  int32_t ldj, row0_bias, row0_prior;
  int32_t P;
};
// [A | b] = Jrow' Jrow, fixed summation order (A: [P][P] symmetric, b: [P])
int launch_marg_syrk(const double* Jrow, int R, int ldj, int P, double* A, double* b, cudaStream_t s);
int launch_marg_image(const MargImageArgs& a, cudaStream_t s);
int launch_marg_imu(const MargImuArgs& a, cudaStream_t s);
int launch_marg_small(const MargSmallArgs& a, cudaStream_t s);
// symmetric eigen-decomposition (parallel cyclic Jacobi): A overwritten, V <- eigenvectors (columns), ev <- eigenvalues
// log_buf: jacobi_log_bytes(n, 40) bytes of global scratch for the rotation log (eigenvalues by one CTA, eigenvectors
// by a replay kernel with one CTA per row).  Returns the number of kernels launched, or -1 if a launch was refused.
size_t jacobi_log_bytes(int n, int max_sweeps);
int launch_jacobi_eig(double* A, double* V, double* ev, int n, void* log_buf, cudaStream_t s);
// blocked variant (jacobi_blocked.cu): 16 <= n and the padded matrix fits one SM's shared memory (n <= 128)
bool jacobi_blocked_fits(int n);
size_t jacobi_blocked_log_bytes(int n, int max_sweeps);
int launch_jacobi_blocked(const double* A, double* V, double* ev, int n, void* log_buf, int max_sweeps, cudaStream_t s);
int launch_dense_gemm(int m, int n, int k, double alpha, const double* A, int lda, bool ta, const double* B, int ldb,
                      bool tb, double beta, double* C, int ldc, cudaStream_t s);
int launch_marg_elementwise(int mode, int n, int ld, const double* src, double* dst, const double* ev, const double* vb,
                            double* rlin, double eps, cudaStream_t s);

int launch_abs_column_sums(const double* r, int n, int cols, double* out, cudaStream_t s);
int launch_bias_abs_sums(const int2* ij, const double* sq, int n, const double* bias, double* out6, cudaStream_t s);

// measured fp64 FMA throughput of the current device (TFLOP/s); < 0 on error
double measure_fp64_tflops(cudaStream_t s);
// measured fp64 tensor-core (mma.sync.m8n8k4.f64) throughput with `ctas_per_sm` CTAs of 256 threads per SM (TFLOP/s);
// optionally the dependent latency of one mma in cycles; < 0 on error
double measure_fp64_tensor_tflops(cudaStream_t s, int ctas_per_sm = 4, double* dep_latency_cycles = nullptr);

int launch_rho_pack(const double* rho, const uint8_t* owned, double* buf, int nL, cudaStream_t s);
int launch_rho_unpack(double* rho, const double* buf, int nL, cudaStream_t s);

bool comm_unique_id(uint8_t* id128, std::string* err);
void* comm_create(int rank, int world, const uint8_t* id128, std::string* err);
void comm_destroy(void* comm);
// in-place sum-allreduce of n doubles on the stream; returns false on error
bool comm_allreduce_sum(void* comm, double* buf, size_t n, cudaStream_t s, std::string* err);
// recv[rank][n_per_rank] <- every rank's send[n_per_rank]
bool comm_allgather(void* comm, const double* send, double* recv, size_t n_per_rank, cudaStream_t s, std::string* err);

// sharded mode: lower-triangular 64x64 tiles of M + rhs + diagA <-> one contiguous all-reduce buffer
size_t shard_pack_len(int npad);
int launch_shard_pack(const LinearLaunch& a, double* packed, cudaStream_t s);
// after the all-reduce: scatter back, add the LM damping / identity rows
int launch_shard_unpack(const LinearLaunch& a, const double* packed, double radius, cudaStream_t s);
// sharded mode: per-rank scalar blocks (all-gathered, [world][8]) -> the common scalar block: sums of cost / g'd / d'Hd /
// |dx|^2 / |x|^2 / error flag, maxima of the gradient / step max-norms; identical on every rank, published to the mapped
// host block like the single-GPU path does
int launch_shard_scalars_pack(LmScalars* scal, double* send8, cudaStream_t s);
int launch_shard_scalars_reduce(const double* gathered, int world, LmScalars* scal, LmPublished* pub, unsigned long long seq,
                                cudaStream_t s);

}  // namespace ctvio
