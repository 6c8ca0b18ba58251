// K5 (fallback path): blocked right-looking Cholesky of the reduced camera system + both triangular solves in ONE
// cooperative persistent kernel with grid-wide barriers.  The product path is the tile-DAG kernel (chol_dag.cu);
// this one is used when the window is so large that not every 64x64 tile can have its own SM (n_p > ~1000), when the
// runtime refuses the DAG's cooperative launch, or on request (CTVIO_CHOL=coop, A/B measurements).
// Replaces the factor/solve half of Ceres' SPARSE_NORMAL_CHOLESKY step (trajectory_estimator.cpp:374;
// Ceres is not part of the reference repository) on the Schur-reduced system.
//
//   per block column k (NB = 64):
//     phase P  every CTA that owns a panel slab loads the (already updated) diagonal block, factors it
//              and inverts the factor redundantly in shared memory (factor_and_invert_64, chol_tiles.cuh), turns its
//              slabs' TRSM into a GEMM with that inverse, and folds the forward substitution of the right-hand side in;
//     phase U  the trailing tiles are spread over all CTAs (64^3 register-tiled DFMA GEMM each).
//   afterwards CTA 0 runs the backward substitution with the stored block inverses.
// M: lower triangle used; strictly-lower panels are overwritten with L, diagonal blocks are left
// untouched (only their inverses, Linv, are kept).
#include <cooperative_groups.h>

#include <algorithm>
#include <cstdlib>
#include <string>

#include "chol_tiles.cuh"
#include "kernels.h"
#include "marginalize.h"

namespace ctvio {

namespace cg = cooperative_groups;

// optional phase timing of CTA 0 (debug): build with CTVIO_EXTRA_NVCC_FLAGS=-DCTVIO_CHOL_TIMING
#ifdef CTVIO_CHOL_TIMING
__device__ unsigned long long g_chol_stamps[4096];
__device__ __forceinline__ void stamp(int& n) {
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    if (n < 4096) g_chol_stamps[n] = t;
  }
  ++n;
}
#define STAMP() stamp(stamp_n)
#else
#define STAMP()
#endif

__global__ void __launch_bounds__(256, 1)
chol_coop_kernel(double* __restrict__ M, int npad, double* __restrict__ Linv, const double* __restrict__ rhs,
                 double* __restrict__ y, double* __restrict__ yf, LmScalars* scal) {
  extern __shared__ __align__(16) unsigned char chol_smem[];
  double* D = reinterpret_cast<double*>(chol_smem);  // diagonal block -> its factor
  double* Xi = D + kTile;                             // inverse of the factor (lower)
  double* XiT = Xi + kTile;                           // its transpose (B operand of the slab GEMM)
  double* S1 = XiT + kTile;                           // operand A, transposed
  double* S2 = S1 + kTile;                            // operand B, transposed / merge scratch / slab result
  double* rdiag = S2 + kTile;                         // [64]
  double* xk = rdiag + kCholNB;                       // [64]
  double* red = xk + kCholNB;                         // [2][64] partial sums
  __shared__ int s_bad;
  const int tid = threadIdx.x;
  const int ty = tid >> 4, tx = tid & 15;
  const int G = gridDim.x, cta = blockIdx.x;
  const int nb = npad / kCholNB;
  cg::grid_group grid = cg::this_grid();
#ifdef CTVIO_CHOL_TIMING
  int stamp_n = 0;
#endif
  STAMP();
  for (int r = cta * 256 + tid; r < npad; r += G * 256) y[r] = rhs[r];
  grid.sync();
  STAMP();

#pragma unroll 1
  for (int k = 0; k < nb; ++k) {
    const int nslab = nb - k - 1;
    const int d0 = k * kCholNB;
    // ---------------- phase P: diagonal block, panel slabs, forward substitution ----------------
    if (cta == 0 || cta < nslab) {
      for (int e = tid; e < kCholNB * kCholNB / 2; e += 256) {
        const int r = e >> 5, c = (e & 31) * 2;
        *reinterpret_cast<double2*>(D + r * kTS + c) = *reinterpret_cast<const double2*>(M + size_t(d0 + r) * npad + d0 + c);
      }
      __syncthreads();
      STAMP();  // diag block loaded
      const bool ok = factor_and_invert_64(D, Xi, XiT, S2, rdiag, &s_bad);
      if (!ok && cta == 0 && tid == 0) scal->chol_fail = 1;
      STAMP();  // factored + inverted
      // x_k = Xi * y_k  (4 lanes per row)
      {
        const int r = tid >> 2, pt = tid & 3;
        double s = 0.0;
        for (int c = pt; c <= r; c += 4) s = fma(Xi[r * kTS + c], y[d0 + c], s);
        s += __shfl_xor_sync(0xffffffffu, s, 1);
        s += __shfl_xor_sync(0xffffffffu, s, 2);
        if (pt == 0) xk[r] = s;
      }
      if (cta == 0) {  // publish Linv_k
        double* Li = Linv + size_t(k) * kCholNB * kCholNB;
        for (int e = tid; e < kCholNB * kCholNB / 2; e += 256) {
          const int r = e >> 5, c = (e & 31) * 2;
          *reinterpret_cast<double2*>(Li + r * kCholNB + c) = *reinterpret_cast<const double2*>(Xi + r * kTS + c);
        }
      }
      __syncthreads();
      if (cta == 0 && tid < kCholNB) yf[d0 + tid] = xk[tid];  // forward-solved block
      for (int b = cta; b < nslab; b += G) {
        const int r0 = (k + 1 + b) * kCholNB;
        load_tile_transposed(S1, M, npad, r0, d0, tid);
        __syncthreads();
        double acc[4][4];
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
          for (int j = 0; j < 4; ++j) acc[i][j] = 0.0;
        tile_gemm_tt(S1, XiT, acc, ty, tx);  // X = A_slab * Xi^T
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          *reinterpret_cast<double2*>(S2 + (4 * ty + i) * kTS + 4 * tx) = make_double2(acc[i][0], acc[i][1]);
          *reinterpret_cast<double2*>(S2 + (4 * ty + i) * kTS + 4 * tx + 2) = make_double2(acc[i][2], acc[i][3]);
          *reinterpret_cast<double2*>(M + size_t(r0 + 4 * ty + i) * npad + d0 + 4 * tx) = make_double2(acc[i][0], acc[i][1]);
          *reinterpret_cast<double2*>(M + size_t(r0 + 4 * ty + i) * npad + d0 + 4 * tx + 2) = make_double2(acc[i][2], acc[i][3]);
        }
        __syncthreads();
        {  // y_slab -= X * x_k
          const int r = tid >> 2, pt = tid & 3;
          double s = 0.0;
#pragma unroll 4
          for (int c = pt; c < kCholNB; c += 4) s = fma(S2[r * kTS + c], xk[c], s);
          s += __shfl_xor_sync(0xffffffffu, s, 1);
          s += __shfl_xor_sync(0xffffffffu, s, 2);
          if (pt == 0) y[r0 + r] -= s;
        }
        __syncthreads();
      }
    }
    STAMP();  // phase P done
    if (nslab == 0) break;
    grid.sync();
    STAMP();  // sync 1
    // ---------------- phase U: trailing update, tiles (bi >= bj) spread over the grid ----------------
    const int ntiles = nslab * (nslab + 1) / 2;
    for (int t = cta; t < ntiles; t += G) {
      int bi = 0, rem = t;
      while (rem > bi) { rem -= bi + 1; ++bi; }
      const int bj = rem;
      const int ri = (k + 1 + bi) * kCholNB, rj = (k + 1 + bj) * kCholNB;
      load_tile_transposed(S1, M, npad, ri, d0, tid);
      if (bi != bj) load_tile_transposed(S2, M, npad, rj, d0, tid);
      __syncthreads();
      double acc[4][4];
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = 0.0;
      tile_gemm_tt(S1, bi != bj ? S2 : S1, acc, ty, tx);
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        double2* p01 = reinterpret_cast<double2*>(M + size_t(ri + 4 * ty + i) * npad + rj + 4 * tx);
        double2 v01 = p01[0], v23 = p01[1];
        v01.x -= acc[i][0]; v01.y -= acc[i][1]; v23.x -= acc[i][2]; v23.y -= acc[i][3];
        p01[0] = v01; p01[1] = v23;
      }
      __syncthreads();
    }
    STAMP();  // phase U done
    grid.sync();
    STAMP();  // sync 2
  }
  if (cta != 0) return;
  // ---------------- backward substitution  L^T x = yf  (CTA 0) ----------------
  __syncthreads();
#pragma unroll 1
  for (int k = nb - 1; k >= 0; --k) {
    const int d0 = k * kCholNB;
    const int c = tid & 63, pt = tid >> 6;
    // t_c = yf_c - sum_{r below block k} L[r][d0 + c] x_r ; 4 row phases x 4 independent accumulators
    double s0 = 0.0, s1 = 0.0, s2 = 0.0, s3 = 0.0;
    int r = d0 + kCholNB + pt;
    for (; r + 12 < npad; r += 16) {
      s0 = fma(M[size_t(r) * npad + d0 + c], y[r], s0);
      s1 = fma(M[size_t(r + 4) * npad + d0 + c], y[r + 4], s1);
      s2 = fma(M[size_t(r + 8) * npad + d0 + c], y[r + 8], s2);
      s3 = fma(M[size_t(r + 12) * npad + d0 + c], y[r + 12], s3);
    }
    for (; r < npad; r += 4) s0 = fma(M[size_t(r) * npad + d0 + c], y[r], s0);
    const double s = (s0 + s1) + (s2 + s3);
    if (pt < 2) red[pt * kCholNB + c] = s;
    __syncthreads();
    if (pt >= 2) red[(pt - 2) * kCholNB + c] += s;
    __syncthreads();
    if (tid < kCholNB) xk[tid] = yf[d0 + tid] - red[tid] - red[kCholNB + tid];
    __syncthreads();
    // x = Linv_k^T * t
    const double* Li = Linv + size_t(k) * kCholNB * kCholNB;
    double u = 0.0;
    for (int rr = c + ((pt - c) & 3); rr < kCholNB; rr += 4) u = fma(Li[rr * kCholNB + c], xk[rr], u);
    if (pt < 2) red[pt * kCholNB + c] = u;
    __syncthreads();
    if (pt >= 2) red[(pt - 2) * kCholNB + c] += u;
    __syncthreads();
    if (tid < kCholNB) y[d0 + tid] = red[tid] + red[kCholNB + tid];
    __syncthreads();
  }
  STAMP();  // backward substitution done
}

#ifdef CTVIO_CHOL_TIMING
extern "C" int ctvio_debug_chol_stamps(unsigned long long* out, int n) {
  return cudaMemcpyFromSymbol(out, g_chol_stamps, sizeof(unsigned long long) * n) == cudaSuccess ? 0 : -1;
}
// latency probes (debug build only): cycles per dependent op, measured by thread 0 of one CTA with `nthreads` threads
__global__ void latency_probe_kernel(double seed, long long* out, double* sink) {
  __shared__ double sm[512];
  double x = seed + threadIdx.x * 1e-9, y = 1.0 + 1e-9 * seed;
  sm[threadIdx.x] = x;
  __syncthreads();
  long long t0 = clock64();
#pragma unroll 1
  for (int i = 0; i < 64; ++i) {
    x = fma(x, y, 1e-3); x = fma(x, y, 1e-3); x = fma(x, y, 1e-3); x = fma(x, y, 1e-3);
  }
  long long t1 = clock64();
#pragma unroll 1
  for (int i = 0; i < 64; ++i) { x = x * y; x = x * y; x = x * y; x = x * y; }
  long long t2 = clock64();
#pragma unroll 1
  for (int i = 0; i < 64; ++i) x = rsqrt(x + 2.0);
  long long t3 = clock64();
#pragma unroll 1
  for (int i = 0; i < 64; ++i) { sm[threadIdx.x] = x; __syncthreads(); x += sm[(threadIdx.x + 17) % blockDim.x]; __syncthreads(); }
  long long t4 = clock64();
  // 16 independent chains
  double z[16];
#pragma unroll
  for (int j = 0; j < 16; ++j) z[j] = x + j;
#pragma unroll 1
  for (int i = 0; i < 64; ++i) {
#pragma unroll
    for (int j = 0; j < 16; ++j) z[j] = fma(z[j], y, 1e-3);
  }
  long long t5 = clock64();
  float f = float(x);
#pragma unroll 1
  for (int i = 0; i < 64; ++i) { f = fmaf(f, 1.0001f, 1e-3f); f = fmaf(f, 1.0001f, 1e-3f); f = fmaf(f, 1.0001f, 1e-3f); f = fmaf(f, 1.0001f, 1e-3f); }
  long long t6 = clock64();
#pragma unroll
  for (int j = 0; j < 16; ++j) x += z[j];
  x += f;
  if (threadIdx.x == 0) {
    out[0] = t1 - t0; out[1] = t2 - t1; out[2] = t3 - t2; out[3] = t4 - t3; out[4] = t5 - t4; out[5] = t6 - t5;
  }
  sink[threadIdx.x] = x;
}
// DMMA throughput + dependent latency: the fp64 tensor-core micro-benchmark of misc_kernels.cu at a chosen occupancy
extern "C" int ctvio_debug_dmma(int ctas_per_sm, double* tflops, double* dep_latency_cycles) {
  const double v = measure_fp64_tensor_tflops(0, ctas_per_sm, dep_latency_cycles);
  if (v < 0) return -1;
  *tflops = v;
  return 0;
}
extern "C" int ctvio_debug_latency(int nthreads, long long* out6) {
  long long* d; double* sink;
  cudaMalloc(&d, 64); cudaMalloc(&sink, 8 * 1024);
  latency_probe_kernel<<<1, nthreads>>>(1.5, d, sink);
  latency_probe_kernel<<<1, nthreads>>>(1.5, d, sink);
  cudaMemcpy(out6, d, 48, cudaMemcpyDeviceToHost);
  cudaFree(d); cudaFree(sink);
  return cudaGetLastError() == cudaSuccess ? 0 : -1;
}
#endif

int launch_factor_solve(const LinearLaunch& a, cudaStream_t s) {
  // CTVIO_CHOL=coop forces the barrier kernel (A/B measurements, tests/...::test_barrier_cholesky_fallback_*); read on
  // every call (a getenv costs nanoseconds against the kernel) so that one process can exercise both paths
  const char* env = std::getenv("CTVIO_CHOL");
  const int mode = (env && std::string(env) == "coop") ? 1 : 0;
  if (mode == 0 && a.chol_part && a.chol_flags && chol_dag_supported(a.npad, device_sm_count())) return launch_chol_dag(a, s);
  return launch_chol_coop(a, s);
}

int launch_chol_coop(const LinearLaunch& a, cudaStream_t s) {
  static PerDeviceOnce once;
  if (once.first()) cudaFuncSetAttribute(chol_coop_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, int(kCholCoopSmem));
  const int n_sm = device_sm_count();
  const int nb = a.npad / kCholNB;
  const int t0 = nb - 1;
  int grid = std::max(1, std::min(n_sm, std::max(t0, t0 * (t0 + 1) / 2)));
  double* M = a.M;
  int npad = a.npad;
  double* Linv = a.Linv;
  const double* rhs = a.rhs;
  double* y = a.y;
  double* yf = a.yf;
  LmScalars* scal = a.scal;
  void* args[] = {&M, &npad, &Linv, &rhs, &y, &yf, &scal};
  if (cudaLaunchCooperativeKernel(reinterpret_cast<void*>(chol_coop_kernel), dim3(grid), dim3(256), args, kCholCoopSmem, s) !=
      cudaSuccess) {
    // nothing ran: make the step fail loudly (the LM driver treats chol_fail as an invalid step and eventually
    // terminates with FAILURE) instead of consuming a stale solution
    cudaGetLastError();
    cudaMemsetAsync(&scal->chol_fail, 0xff, sizeof(int32_t), s);
  }
  return 1;
}

}  // namespace ctvio
