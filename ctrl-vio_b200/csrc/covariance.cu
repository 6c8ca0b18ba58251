// ctvio_covariance: the marginal covariance of the window at the current state, from the factor of the LM step's own
// reduced camera system (ceres::Covariance with its defaults, which the reference's trajectory_estimator.h:23 makes
// available to its callers; Ceres is not part of the reference repository).
//
//   evaluation  K1-K3 with full Jacobians into the spare normal-equation buffer
//   K4          reduced_system_kernel at radius +inf: no damping, S_s = D S D (D the Jacobi scale) with identity rows on
//               the dims that get no covariance
//   K5          the LM step's Cholesky (tile DAG or barrier kernel), S_s = L L'
//   cov_*       L^-1 tile by tile, Sigma = D L^-T L^-1 D (the camera block of H^-1, by the Schur-complement identity), and
//               the landmark inverse-depth variances 1 / h_l + v_l' Sigma v_l, v_l = W_l / h_l
//
// Every product of 64x64 tiles runs on the fp64 tensor path (mma.sync.m8n8k4.f64, full-tile instantiations only: no
// DMMA under a run-time predicate, DESIGN §4).  No atomics: the result is bitwise reproducible for a given H.
//
// ctvio_pose_covariance forms the same Sigma (with an optional gauge of its own in the mask) and projects it to the
// pose and velocity at each query time on the device (pose_cov_kernel, 12 x 24 Jacobians, plain fp64 fma chains).
// ctvio_relative_pose_covariance projects it to the pose at t_b in the frame of the pose at t_a, over the union of the
// two segments' knots, with the cross-covariance of the two poses (relative_pose_cov_kernel, 6 x 48 Jacobians).
// ctvio_point_covariance and ctvio_feature_table_point_covariance project it, with the landmark-knot cross terms
// -Sigma W_l' / h_l and the variance of rho_l, to anchored landmarks' world points (point_cov_kernel, 3 x 25 Jacobians).
#include <cmath>
#include <cstdio>

#include "chol_tiles.cuh"
#include "dmma_tiles.cuh"
#include "engine_state.h"

namespace ctvio {

namespace {

constexpr size_t kCovTileSmem = 2 * size_t(kTile) * sizeof(double);                          // two operand tiles
constexpr size_t kCovDiagSmem = (4 * size_t(kPacket) + size_t(kTile)) * sizeof(double);      // 4 packets + the inverse

// smem tile (row stride kTS) <- 64x64 row-major global block with row stride ld
__device__ __forceinline__ void load_tile_rm(double* dst, const double* src, int ld, int tid) {
  for (int e = tid; e < kCholNB * kCholNB / 2; e += 256) {
    const int r = e >> 5, c = (e & 31) * 2;
    *reinterpret_cast<double2*>(dst + r * kTS + c) = *reinterpret_cast<const double2*>(src + size_t(r) * ld + c);
  }
}

// At[c][r] = L(ti, tj)[r][c], the A operand layout of tile_gemm_dmma, from K5's output in M
__device__ __forceinline__ void load_factor_tile_t(double* At, const CovLaunch& c, int ti, int tj, int tid) {
  const double* slot = c.M + size_t(ti) * kCholNB * c.npad + size_t(tj) * kCholNB;
  if (c.tile_dag) load_tile_rm(At, slot, c.npad, tid);  // the DAG publishes its tiles transposed inside the slot
  else load_tile_transposed(At, c.M, c.npad, ti * kCholNB, tj * kCholNB, tid);
}

// fragments -> global 64x64 tile (row stride ld)
__device__ __forceinline__ void frag_store_global(double* dst, int ld, const Frag& f, const Lane& L) {
#pragma unroll
  for (int mt = 0; mt < 2; ++mt)
#pragma unroll
    for (int nt = 0; nt < 4; ++nt)
      *reinterpret_cast<double2*>(dst + size_t(L.row(mt)) * ld + L.col(nt)) = make_double2(f.c[mt][nt][0], f.c[mt][nt][1]);
}

// lane's part of sum_b row[col_b] w_b over a landmark's coupling row: its n knot dims lo .. lo + n - 1, then the line
// delay (b = n).  Lane b takes b, b + 32, ... in order; the caller finishes with one fixed shuffle tree.
__device__ __forceinline__ double coupling_dot_part(const double* row, int lo, int n, int ld, const double* Wl, double wld,
                                                    int lane) {
  double s = 0.0;
  for (int b = lane; b <= n; b += 32) s = fma(row[b < n ? lo + b : ld], b < n ? Wl[b] : wld, s);
  return s;
}

// The projections C = G Sigma_blk G' of the window covariance (pose_cov_kernel, point_cov_kernel,
// relative_pose_cov_kernel), one warp each: the block of Sigma, then T = G Sigma_blk (warp_mul), then C = T G'
// (warp_mul_t), every entry one fixed-order fma chain (from 0, k ascending), no atomics.

// S[i * ld + j] = Sigma at dims i, j < m of the union of segments sa and sb (relative_union_knot), m = 6 (4 + off); M: m
// when it is known at compile time.  sa == sb is the 24 x 24 block at the contiguous dims 6 sa .. 6 sa + 23.  Dim i of
// the union is 6 lo + i below the 6 off dims of lo's knots that hi does not share, 6 (hi - off) + i from there on: the
// same dims as relative_union_knot's, without its division by 6 (which costs pose_cov_kernel a spill).
template <int M>
__device__ __forceinline__ void gather_union_block(double* S, int ld, const double* cov, int np, int32_t sa, int32_t sb,
                                                   int lane) {
  const int off = relative_union_offset(sa, sb), m = M ? M : 6 * (4 + off);
  const int d0 = 6 * (sa < sb ? sa : sb), d1 = 6 * ((sa < sb ? sb : sa) - off);
  for (int e = lane; e < m * m; e += 32) {  // row by row
    const int i = e / m, j = e - i * m;
    const int gi = (i < 6 * off ? d0 : d1) + i, gj = (j < 6 * off ? d0 : d1) + j;
    S[i * ld + j] = cov[size_t(gi) * np + gj];
  }
}

// T = A S: T [rows][cols] and A [rows][kn] dense, S [kn][cols] with row stride lds; fma(A[i][k], S[k][b], acc)
template <int UNROLL>
__device__ __forceinline__ void warp_mul(double* T, const double* A, const double* S, int lds, int rows, int cols, int kn,
                                         int lane) {
  for (int e = lane; e < rows * cols; e += 32) {
    const int i = e / cols, b = e - i * cols;
    double acc = 0.0;
#pragma unroll UNROLL
    for (int k = 0; k < kn; ++k) acc = fma(A[i * kn + k], S[k * lds + b], acc);
    T[e] = acc;
  }
}

// out = T B': out [rows][cols], T [rows][kn] and B [cols][kn] dense; fma(T[i][k], B[j][k], acc).  SYM (T B' symmetric,
// rows == cols): the lower triangle is formed and mirrored, so that out is exactly symmetric.
template <int UNROLL, bool SYM>
__device__ __forceinline__ void warp_mul_t(double* out, const double* T, const double* B, int rows, int cols, int kn,
                                           int lane) {
  for (int e = lane; e < (SYM ? rows * (rows + 1) / 2 : rows * cols); e += 32) {
    int i = 0, j;
    if (SYM) {
      while ((i + 1) * (i + 2) / 2 <= e) ++i;
      j = e - i * (i + 1) / 2;
    } else {
      i = e / cols;
      j = e - i * cols;
    }
    double acc = 0.0;
#pragma unroll UNROLL
    for (int k = 0; k < kn; ++k) acc = fma(T[i * kn + k], B[j * kn + k], acc);
    out[i * cols + j] = acc;
    if (SYM) out[j * cols + i] = acc;
  }
}

}  // namespace

__global__ void cov_mask_kernel(const uint8_t* __restrict__ active, int np, int n_gauge, uint8_t* __restrict__ cmask) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < np) cmask[i] = (active[i] && i >= n_gauge) ? 0 : 1;
}

// CTA k: X(k,k) = L(k,k)^-1 (upper triangle zero) and the extreme pivots of block k.  The barrier kernel keeps the
// inverse (Linv); the tile DAG keeps the block as four packets, inverted here as its own backward sweep does.
__global__ void __launch_bounds__(256) cov_diag_inverse_kernel(CovLaunch c) {
  extern __shared__ __align__(16) double cov_smem[];
  double* Xi = cov_smem;
  double* Pk = Xi + kTile;
  __shared__ double red[2][8];
  const int k = blockIdx.x, tid = threadIdx.x;
  if (c.tile_dag) {
    const double* src = c.packets + size_t(k) * 4 * kPacketG;
    for (int e = tid; e < 4 * 16 * 40; e += 256) {  // [s][m][80] -> [s][m][kPS]
      const int row = e / 40, col = (e - row * 40) * 2;
      *reinterpret_cast<double2*>(Pk + row * kPS + col) = *reinterpret_cast<const double2*>(src + row * 80 + col);
    }
    __syncthreads();
    inverse_from_packets(Pk, Xi, tid);
    __syncthreads();
  } else {
    load_tile_rm(Xi, c.Linv + size_t(k) * kCholNB * kCholNB, kCholNB, tid);
    __syncthreads();
  }
  double* dst = c.X + size_t(k) * kCholNB * c.npad + size_t(k) * kCholNB;
  for (int e = tid; e < kCholNB * kCholNB / 2; e += 256) {
    const int r = e >> 5, cc = (e & 31) * 2;
    *reinterpret_cast<double2*>(dst + size_t(r) * c.npad + cc) = *reinterpret_cast<const double2*>(Xi + r * kTS + cc);
  }
  // 1 / L_ii = X_ii over the free dims of the block (constant and padding dims carry the identity)
  double mn = INFINITY, mx = 0.0;
  if (tid < kCholNB) {
    const int g = k * kCholNB + tid;
    if (g < c.np && !c.cmask[g]) mn = mx = Xi[tid * kTS + tid];
  }
  if (tid < kCholNB) {
    mn = warp_min_d(mn);
    mx = warp_max_d(mx);
    if ((tid & 31) == 0) { red[0][tid >> 5] = mn; red[1][tid >> 5] = mx; }
  }
  __syncthreads();
  if (tid == 0) {
    c.piv[2 * k] = fmin(red[0][0], red[0][1]);
    c.piv[2 * k + 1] = fmax(red[1][0], red[1][1]);
  }
}

// CTA j: block column j of X = L^-1, top to bottom: X(i,j) = -X(i,i) sum_{k=j}^{i-1} L(i,k) X(k,j), i > j.  Each step
// reads the blocks of column j this CTA wrote before it (global memory, ordered by the CTA barrier).
__global__ void __launch_bounds__(256) cov_column_kernel(CovLaunch c) {
  extern __shared__ __align__(16) double cov_smem[];
  double* At = cov_smem;
  double* Bt = At + kTile;
  const int j = blockIdx.x, tid = threadIdx.x, nb = c.npad / kCholNB;
  const Lane L = lane_of(tid);
#pragma unroll 1
  for (int i = j + 1; i < nb; ++i) {
    Frag t;
    frag_zero(t);
#pragma unroll 1
    for (int k = j; k < i; ++k) {
      load_factor_tile_t(At, c, i, k, tid);
      load_tile_rm(Bt, c.X + size_t(k) * kCholNB * c.npad + size_t(j) * kCholNB, c.npad, tid);  // Bt[k'][n] = X(k,j)[k'][n]
      __syncthreads();
      tile_gemm_dmma<false>(At, Bt, t, L);
      __syncthreads();
    }
    frag_store(Bt, t, L);
    load_tile_transposed(At, c.X, c.npad, i * kCholNB, i * kCholNB, tid);  // At[c][r] = X(i,i)[r][c]
    __syncthreads();
    Frag x;
    frag_zero(x);
    tile_gemm_dmma<true>(At, Bt, x, L);
    frag_store_global(c.X + size_t(i) * kCholNB * c.npad + size_t(j) * kCholNB, c.npad, x, L);
    __syncthreads();
  }
}

// CTA per lower tile (i, j): Sigma_s(i,j) = sum_{k >= i} X(k,i)' X(k,j), written as D Sigma_s D into both triangles of the
// covariance, zero on the dims that get none.  A diagonal tile writes its lower half and mirrors it: exactly symmetric.
__global__ void __launch_bounds__(256) cov_sigma_kernel(CovLaunch c) {
  extern __shared__ __align__(16) double cov_smem[];
  double* At = cov_smem;
  double* Bt = At + kTile;
  const int tid = threadIdx.x, nb = c.npad / kCholNB;
  int i = 0;
  while ((i + 1) * (i + 2) / 2 <= int(blockIdx.x)) ++i;
  const int j = int(blockIdx.x) - i * (i + 1) / 2;
  const Lane L = lane_of(tid);
  Frag f;
  frag_zero(f);
#pragma unroll 1
  for (int k = i; k < nb; ++k) {
    const double* row = c.X + size_t(k) * kCholNB * c.npad;
    load_tile_rm(At, row + size_t(i) * kCholNB, c.npad, tid);  // At[c][r] = X(k,i)[c][r]
    if (i != j) load_tile_rm(Bt, row + size_t(j) * kCholNB, c.npad, tid);
    __syncthreads();
    tile_gemm_dmma<false>(At, i != j ? Bt : At, f, L);
    __syncthreads();
  }
#pragma unroll
  for (int mt = 0; mt < 2; ++mt)
#pragma unroll
    for (int nt = 0; nt < 4; ++nt)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int r = L.row(mt), cc = L.col(nt) + e;
        const int gi = i * kCholNB + r, gj = j * kCholNB + cc;
        if (gi >= c.np || gj >= c.np || (i == j && cc > r)) continue;
        const double v = (c.cmask[gi] || c.cmask[gj]) ? 0.0 : c.sc[gi] * f.c[mt][nt][e] * c.sc[gj];
        c.cov[size_t(gi) * c.np + gj] = v;
        c.cov[size_t(gj) * c.np + gi] = v;
      }
}

// one warp per landmark: var_l = 1 / h_l + (w_l' Sigma w_l) / h_l^2 over its coupling row [lo, hi) + the line delay;
// lane b takes the columns b, b + 32, ... of every row, then one fixed shuffle tree: bitwise reproducible
__global__ void __launch_bounds__(256) landmark_variance_kernel(LandmarkVarLaunch v) {
  const int lane = threadIdx.x & 31;
  const int l = blockIdx.x * 8 + (threadIdx.x >> 5);
  if (l >= v.nL) return;
  const double hl = v.ne.hl[l];
  if (!v.active[v.np + l]) {
    if (lane == 0) v.var[l] = 0.0;
    return;
  }
  if (!(hl > 0.0)) {  // a landmark with factors but no information: H is singular
    if (lane == 0) { v.var[l] = 0.0; v.scal->chol_fail = 1; }
    return;
  }
  const int lo = v.lm.lo[l], n = v.lm.hi[l] - lo, ld = v.idx_ld;
  const double* Wl = v.ne.W + v.lm.woff[l];
  const double wld = v.ne.wld[l];
  double acc = 0.0;
#pragma unroll 1
  for (int a = 0; a <= n; ++a) {
    const int ga = a < n ? lo + a : ld;
    const double wa = a < n ? Wl[a] : wld;
    acc = fma(wa, coupling_dot_part(v.cov + size_t(ga) * v.np, lo, n, ld, Wl, wld, lane), acc);
  }
  acc = warp_sum_d(acc);
  if (lane == 0) v.var[l] = 1.0 / hl + acc / (hl * hl);
}

// one warp: the extreme pivots over the blocks, rcond, and the scalar block with rcond to mapped host memory
__global__ void cov_publish_kernel(const double* __restrict__ piv, int nb, const LmScalars* scal, LmPublished* pub,
                                   unsigned long long seq) {
  const int lane = threadIdx.x;
  double mn = INFINITY, mx = 0.0;
  for (int b = lane; b < nb; b += 32) { mn = fmin(mn, piv[2 * b]); mx = fmax(mx, piv[2 * b + 1]); }
  mn = warp_min_d(mn);
  mx = warp_max_d(mx);
  if (lane != 0) return;
  // X_ii = 1 / L_ii: min L / max L = min X / max X.  No free dim at all: nothing can be singular
  const double ratio = mx > 0.0 ? mn / mx : 1.0;
  __threadfence();
  pub->s = *scal;
  pub->rcond = ratio * ratio;
  __threadfence_system();
  *reinterpret_cast<volatile unsigned long long*>(&pub->seq) = seq;
}

int launch_cov_mask(const uint8_t* active, int np, int n_gauge, uint8_t* cmask, cudaStream_t s) {
  cov_mask_kernel<<<(np + 255) / 256, 256, 0, s>>>(active, np, n_gauge, cmask);
  return 1;
}

int launch_cov_inverse(const CovLaunch& c, cudaStream_t s) {
  static PerDeviceOnce once;
  if (once.first()) {
    cudaFuncSetAttribute(cov_diag_inverse_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, int(kCovDiagSmem));
    cudaFuncSetAttribute(cov_column_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, int(kCovTileSmem));
    cudaFuncSetAttribute(cov_sigma_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, int(kCovTileSmem));
  }
  const int nb = c.npad / kCholNB;
  cov_diag_inverse_kernel<<<nb, 256, kCovDiagSmem, s>>>(c);
  int n = 1;
  if (nb > 1) {
    cov_column_kernel<<<nb - 1, 256, kCovTileSmem, s>>>(c);
    ++n;
  }
  cov_sigma_kernel<<<nb * (nb + 1) / 2, 256, kCovTileSmem, s>>>(c);
  return n + 1;
}

int launch_landmark_variance(const LandmarkVarLaunch& v, cudaStream_t s) {
  if (v.nL == 0) return 0;
  landmark_variance_kernel<<<(v.nL + 7) / 8, 256, 0, s>>>(v);
  return 1;
}

int launch_cov_publish(const double* piv, int nb, const LmScalars* scal, LmPublished* pub, unsigned long long seq,
                       cudaStream_t s) {
  cov_publish_kernel<<<1, 32, 0, s>>>(piv, nb, scal, pub, seq);
  return 1;
}

// One warp per query time: C = (J Sigma_sub) J' with J = J(t) (12 x 24, PoseJacobian) and Sigma_sub the 24 x 24 block of
// the window covariance at the dims of knots s..s+3, which are contiguous (6s .. 6s + 23).  Every lane evaluates the
// spline (the same values in all lanes) and lanes 0..23 write one column of J each.
constexpr int kPoseCovWarps = 4;
__global__ void __launch_bounds__(32 * kPoseCovWarps) pose_cov_kernel(PoseCovLaunch a) {
  __shared__ double sJ[kPoseCovWarps][12 * 24], sS[kPoseCovWarps][24 * 24], sT[kPoseCovWarps][12 * 24];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int n = blockIdx.x * kPoseCovWarps + w;
  if (n >= a.n) return;
  double* J = sJ[w];
  double* S = sS[w];
  double* T = sT[w];
  int32_t s;
  double u;
  spline_index(a.sp, a.t[n], s, u);
  gather_union_block<24>(S, 24, a.cov, a.np, s, s, lane);
  PoseJacobian pj;
  pose_jacobian<kPStride>(a.sp, a.st.q, a.st.p, a.st.tab, s, u, pj);
  if (lane < 24) {
    double col[12];
    pose_jacobian_column(pj, a.camera_frame != 0, a.R_CI, a.p_CI, lane, col);
#pragma unroll
    for (int i = 0; i < 12; ++i) J[i * 24 + lane] = col[i];
  }
  __syncwarp();
  warp_mul<8>(T, J, S, 24, 12, 24, 24, lane);  // T = J Sigma_sub
  __syncwarp();
  warp_mul_t<8, true>(a.out + size_t(n) * 144, T, J, 12, 12, 24, lane);
}

int launch_pose_cov(const PoseCovLaunch& a, cudaStream_t s) {
  if (a.n <= 0) return 0;
  pose_cov_kernel<<<(a.n + kPoseCovWarps - 1) / kPoseCovWarps, 32 * kPoseCovWarps, 0, s>>>(a);
  return 1;
}

// One warp per point: C = (G Sigma_25) G' with G = d P / d (knots s..s+3, rho_l) (3 x 25, point_jacobian_column) and
// Sigma_25 the joint covariance of the segment's 24 knot dims (6s .. 6s + 23) and rho_l:
//   [[Sigma_sub, c], [c', var_l]],  c = -(Sigma_{6s.., row} W_l') / h_l over the coupling row landmark_variance_kernel walks.
// A landmark without factors has rho constant: c = 0 and var_l = 0.  An inverse depth that is not > 0 and finite leaves
// the point undefined: NaN.  The coupling column is reduced by fixed shuffle trees.
constexpr int kPointCovWarps = 4;
__global__ void __launch_bounds__(32 * kPointCovWarps) point_cov_kernel(PointCovLaunch a) {
  __shared__ double sG[kPointCovWarps][3 * 25], sS[kPointCovWarps][25 * 25], sT[kPointCovWarps][3 * 25];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int n = blockIdx.x * kPointCovWarps + w;
  if (n >= a.n) return;
  double* G = sG[w];
  double* S = sS[w];
  double* T = sT[w];
  int l;
  int64_t t;
  double x, y;
  if (a.landmark) {
    l = a.landmark[n];
    t = a.t[n];
    x = a.bearing[2 * n];
    y = a.bearing[2 * n + 1];
  } else {  // the anchor observation: the first entry of the landmark's CSR row
    l = n;
    const int o = a.obs_offset[l], slot = a.obs_slot[o];
    const FrameFeature f = a.table[size_t(slot) * a.frame_cap + a.obs_idx[o]];
    t = a.frame_t[slot];
    x = f.x;
    y = f.y;
  }
  double* out = a.out + size_t(n) * 9;
  const double rho = a.st.rho[l];
  if (!(rho > 0.0) || !isfinite(rho)) {
    if (lane < 9) out[lane] = NAN;
    return;
  }
  int32_t s;
  double u;
  spline_index(a.sp, t, s, u);
  gather_union_block<24>(S, 25, a.cov, a.np, s, s, lane);
  const double hl = a.ne.hl[l];
  if (a.active[a.np + l] && hl > 0.0) {  // (h_l <= 0 with factors fails the covariance before this kernel runs)
    const int lo = a.lm.lo[l], nw = a.lm.hi[l] - lo;
    const double* Wl = a.ne.W + a.lm.woff[l];
    const double wld = a.ne.wld[l];
#pragma unroll 1
    for (int r = 0; r < 24; ++r) {
      const double c = warp_sum_d(coupling_dot_part(a.cov + size_t(6 * s + r) * a.np, lo, nw, a.idx_ld, Wl, wld, lane));
      if (lane == 0) S[r * 25 + 24] = S[24 * 25 + r] = -c / hl;
    }
  } else if (lane < 24) {
    S[lane * 25 + 24] = S[24 * 25 + lane] = 0.0;
  }
  if (lane == 0) S[24 * 25 + 24] = a.var[l];
  PoseJacobian pj;
  pose_jacobian<kPStride>(a.sp, a.st.q, a.st.p, a.st.tab, s, u, pj);
  if (lane < 25) {
    double col[3];
    point_jacobian_column(pj, a.R_CI, a.p_CI, x, y, rho, lane, col);
#pragma unroll
    for (int i = 0; i < 3; ++i) G[i * 25 + lane] = col[i];
  }
  __syncwarp();
  warp_mul<5>(T, G, S, 25, 3, 25, 25, lane);  // T = G Sigma_25
  __syncwarp();
  warp_mul_t<5, true>(out, T, G, 3, 3, 25, lane);
}

int launch_point_cov(const PointCovLaunch& a, cudaStream_t s) {
  if (a.n <= 0) return 0;
  point_cov_kernel<<<(a.n + kPointCovWarps - 1) / kPointCovWarps, 32 * kPointCovWarps, 0, s>>>(a);
  return 1;
}

// One warp (one CTA) per pair: C = (G Sigma_U) G' with U the union of the knots of t_a's and t_b's segments (4 to 8
// knots, m = 24 .. 48 dims, relative_union_knot), Sigma_U its block of the window covariance and G (6 x m) the
// relative-pose Jacobian (relative_pose_jacobian_column over the two poses' dtheta / dp rows J_a, J_b, 6 x 24 each).
// Shared knots get one column, so their terms cancel inside G rather than between two stacked 24-dim blocks.  The cross
// block X = (J_a Sigma_ab) J_b' reads the same Sigma_U at the two segments' slots.  Every lane evaluates both splines (the
// same values in all lanes).  26.5 KB of static shared memory per CTA.
constexpr int kRelUnion = 48;
__global__ void __launch_bounds__(32) relative_pose_cov_kernel(RelativePoseCovLaunch a) {
  __shared__ double S[kRelUnion * kRelUnion], Ja[6 * 24], Jb[6 * 24], G[6 * kRelUnion], T[6 * kRelUnion], X[6 * 24];
  const int lane = threadIdx.x, n = blockIdx.x;
  const bool camera = a.camera_frame != 0;
  int32_t sa, sb;
  double ua, ub;
  spline_index(a.sp, a.t_a[n], sa, ua);
  spline_index(a.sp, a.t_b[n], sb, ub);
  const int off = relative_union_offset(sa, sb), m = 6 * (4 + off);
  const int fa = relative_union_first(sa, sb), fb = relative_union_first(sb, sa);
  gather_union_block<0>(S, m, a.cov, a.np, sa, sb, lane);
  M3 R[2];
  V3 pos[2];
#pragma unroll 1
  for (int side = 0; side < 2; ++side) {  // a, then b: one PoseJacobian live at a time
    PoseJacobian pj;
    pose_jacobian<kPStride>(a.sp, a.st.q, a.st.p, a.st.tab, side ? sb : sa, side ? ub : ua, pj);
    if (lane < 24) {
      double col[12];
      pose_jacobian_column(pj, camera, a.R_CI, a.p_CI, lane, col);
      double* J = side ? Jb : Ja;
#pragma unroll
      for (int i = 0; i < 6; ++i) J[i * 24 + lane] = col[i];
    }
    frame_pose(pj, camera, a.R_CI, a.p_CI, R[side], pos[side]);
  }
  const RelativePose rel = relative_pose(R[0], pos[0], R[1], pos[1]);
  __syncwarp();
  for (int c = lane; c < m; c += 32) {
    double g[6];
    relative_pose_jacobian_column(rel, Ja, fa, Jb, fb, c, g);
#pragma unroll
    for (int i = 0; i < 6; ++i) G[i * m + c] = g[i];
  }
  __syncwarp();
  warp_mul<6>(T, G, S, m, 6, m, m, lane);  // T = G Sigma_U
  if (a.cross) warp_mul<8>(X, Ja, S + 6 * fa * m + 6 * fb, m, 6, 24, 24, lane);  // X = J_a Sigma_ab: a's rows, b's columns
  __syncwarp();
  warp_mul_t<6, true>(a.out + size_t(n) * 36, T, G, 6, 6, m, lane);
  if (a.cross) warp_mul_t<8, false>(a.cross + size_t(n) * 36, X, Jb, 6, 6, 24, lane);
}

int launch_relative_pose_cov(const RelativePoseCovLaunch& a, cudaStream_t s) {
  if (a.n <= 0) return 0;
  relative_pose_cov_kernel<<<a.n, 32, 0, s>>>(a);
  return 1;
}

}  // namespace ctvio

namespace {

// Sigma of the window at the current state into cws.cov and the inverse-depth variances into cws.var, with the knots
// <= gauge_knot held constant on top of what the options hold constant (-1: the options alone), enqueued on the engine
// stream up to the publication of the rank test's inputs (the scalar block and rcond) to pub with sequence number seq
// and the restore of the LM driver's scalar block: no host wait.  Right after a solve of the same factor set (the
// odometry cycle) prepare() finds structure, masks and prior built and does nothing.
int enqueue_covariance(ctvio_engine* e, int gauge_knot, LmPublished* pub, unsigned long long seq) {
  int rc = prepare(e);
  if (rc) return rc;
  cudaStream_t st = e->stream;
  const ProblemDims d = e->dims();
  const size_t np = size_t(d.np), nL = size_t(e->nL), npad = size_t(e->npad), nb = npad / kCholNB;
  auto& w = e->cws;
  CUDA_OK(w.sc.reserve(np));
  CUDA_OK(w.sl.reserve(nL));
  CUDA_OK(w.cmask.reserve(np));
  CUDA_OK(w.X.reserve(npad * npad));
  CUDA_OK(w.piv.reserve(2 * nb));
  CUDA_OK(w.cov.reserve(np * np));
  CUDA_OK(w.var.reserve(nL));
  CUDA_OK(w.scal.reserve(1));
  // the call leaves no trace in the LM driver's state: its scalar block is saved here and restored at the end, the
  // normal equations go to the buffer the next solve clears before use, and the Jacobi scales / mask are this call's own
  CUDA_OK(cudaMemcpyAsync(w.scal.p, e->d_scal.p, sizeof(LmScalars), cudaMemcpyDeviceToDevice, st));
  ensure_table(e);
  const int nbuf = e->cur ^ 1;
  evaluate(e, e->cur, nbuf, true);
  LinearLaunch lin = linear_launch(e, nbuf);
  lin.sc = w.sc.p;
  lin.sl = w.sl.p;
  lin.cmask = w.cmask.p;
  e->launches += launch_jacobi_scale(lin, st);
  e->launches += launch_cov_mask(e->d_active.p, d.np, 6 * (gauge_knot + 1), w.cmask.p, st);
  if (e->deterministic) cudaMemsetAsync(e->d_ticket.p, 0, 2 * sizeof(int32_t), st);
  // radius +inf: clamp(diag) / radius vanishes, and so does the landmark damping
  e->launches += launch_reduced_system(lin, INFINITY, st);
  bool tile_dag = false;
  e->launches += launch_factor_solve(lin, st, &tile_dag);
  CovLaunch c;
  c.np = d.np; c.npad = int(npad); c.nL = e->nL; c.idx_ld = d.idx_ld;
  c.M = lin.M;
  c.Linv = e->d_Linv.p;
  c.packets = tile_dag ? chol_dag_last_packets(e->d_Linv.p, int(npad), e->chol_seq) : nullptr;
  c.tile_dag = tile_dag ? 1 : 0;
  c.cmask = w.cmask.p;
  c.sc = w.sc.p;
  c.X = w.X.p; c.piv = w.piv.p; c.cov = w.cov.p;
  e->launches += launch_cov_inverse(c, st);
  LandmarkVarLaunch v;
  v.np = d.np; v.nL = e->nL; v.idx_ld = d.idx_ld;
  v.cov = w.cov.p;
  v.ne = e->ne(nbuf);
  v.lm = e->lml();
  v.active = e->d_active.p;
  v.var = w.var.p;
  v.scal = e->d_scal.p;
  e->launches += launch_landmark_variance(v, st);
  e->launches += launch_cov_publish(w.piv.p, int(nb), e->d_scal.p, pub, seq, st);
  CUDA_OK(cudaMemcpyAsync(e->d_scal.p, w.scal.p, sizeof(LmScalars), cudaMemcpyDeviceToDevice, st));
  return CTVIO_OK;
}

// the checks of a covariance call that follow its own argument checks: the gauge knot (-1: none of its own), then
// sharded mode
int check_covariance_call(ctvio_engine* e, int32_t gauge_knot_index, const char* who) {
  if (gauge_knot_index < -1 || gauge_knot_index >= e->nK)
    return fail(CTVIO_ERR_INVALID, std::string(who) + ": gauge_knot_index outside -1 .. n_knots - 1");
  if (e->world > 1) return fail(CTVIO_ERR_STATE, std::string(who) + ": not available in sharded mode");
  return CTVIO_OK;
}

// Sigma as enqueue_covariance forms it on the engine's device, then the rank test.  Returns CTVIO_OK, an error of the
// evaluation, or CTVIO_ERR_STATE "<who>: rank deficient"; *rcond (may be null) is written in these last two cases only.
// Ends with the stream synchronised.
int form_covariance(ctvio_engine* e, int gauge_knot, const char* who, double* rcond) {
  cudaSetDevice(e->cfg.device);
  int rc = enqueue_covariance(e, gauge_knot, e->h_pub, ++e->pub_seq);
  if (rc) return rc;
  rc = read_scalars(e, true);
  const double rc_value = const_cast<const LmPublished*>(e->h_pub)->rcond;
  CUDA_OK(stream_sync(e->stream));  // (the restore behind the published block)
  if (rc) return rc;
  if (rcond) *rcond = rc_value;
  LmPublished pub;
  pub.s = *e->h_scal;
  pub.rcond = rc_value;
  std::string why;
  if ((rc = rank_test(pub, who, &why))) return fail(rc, why);
  return CTVIO_OK;
}

// The projection kernels over the a.n items whose inputs a names into out (device memory), right after Sigma on the
// same stream: each builder fills in the state, the spline, the rig and Sigma.
void launch_pose_covariance(ctvio_engine* e, PoseCovLaunch& a, double* out) {
  a.st = e->x[e->cur].ptrs();
  a.sp = e->sp;
  a.R_CI = e->rig.R_CI;
  a.p_CI = e->rig.p_CI;
  a.np = e->dims().np;
  a.cov = e->cws.cov.p;
  a.out = out;
  e->launches += launch_pose_cov(a, e->stream);
}

void launch_relative_pose_covariance(ctvio_engine* e, RelativePoseCovLaunch& a, double* out) {
  a.st = e->x[e->cur].ptrs();
  a.sp = e->sp;
  a.R_CI = e->rig.R_CI;
  a.p_CI = e->rig.p_CI;
  a.np = e->dims().np;
  a.cov = e->cws.cov.p;
  a.out = out;
  e->launches += launch_relative_pose_cov(a, e->stream);
}

void launch_point_covariance(ctvio_engine* e, PointCovLaunch& a, double* out) {
  const ProblemDims d = e->dims();
  a.st = e->x[e->cur].ptrs();
  a.sp = e->sp;
  a.R_CI = e->rig.R_CI;
  a.p_CI = e->rig.p_CI;
  a.np = d.np; a.idx_ld = d.idx_ld;
  a.cov = e->cws.cov.p;
  a.var = e->cws.var.p;
  a.ne = e->ne(e->cur ^ 1);  // the buffer enqueue_covariance evaluated into
  a.lm = e->lml();
  a.active = e->d_active.p;
  a.out = out;
  e->launches += launch_point_cov(a, e->stream);
}

// the anchors of the feature table's window landmarks: the first entry of each observation CSR row
void table_anchors(ctvio_engine* e, PointCovLaunch& a) {
  auto& ft = e->ft;
  a.obs_offset = ft.obs_offset.p; a.obs_slot = ft.obs_slot.p; a.obs_idx = ft.obs_idx.p;
  a.table = e->d_frames.p; a.frame_t = e->d_frame_t.p; a.frame_cap = ctvio_engine::kFrameCap;
}

// point_cov_kernel over the a.n points whose inputs a names, right after form_covariance on the same stream; the n x 9
// result to cov9.  Ends with the stream synchronised.
int point_covariance(ctvio_engine* e, PointCovLaunch& a, double* cov9) {
  auto& w = e->cws;
  CUDA_OK(w.pose.reserve(9 * size_t(a.n)));
  launch_point_covariance(e, a, w.pose.p);
  return read_result(e, cov9, w.pose.p, 9 * size_t(a.n));
}

}  // namespace

extern "C" int ctvio_covariance(ctvio_handle e, double* cov_cc, double* var_rho, double* rcond) {
  if (!e) return fail(CTVIO_ERR_INVALID, "null handle");
  if (int rc = check_covariance_call(e, -1, "ctvio_covariance")) return rc;
  int rc = form_covariance(e, -1, "ctvio_covariance", rcond);
  if (rc) return rc;
  const size_t np = size_t(e->dims().np), nL = size_t(e->nL);
  auto& w = e->cws;
  if (cov_cc && (rc = copy_to_host(e, cov_cc, w.cov.p, np * np))) return rc;
  if (var_rho && nL && (rc = copy_to_host(e, var_rho, w.var.p, nL))) return rc;
  CUDA_OK(stream_sync(e->stream));
  return CTVIO_OK;
}

extern "C" int ctvio_pose_covariance(ctvio_handle e, int32_t n, const int64_t* t_ns, int32_t gauge_knot_index,
                                     int32_t camera_frame, double* cov12, double* rcond) {
  if (!e) return fail(CTVIO_ERR_INVALID, "null handle");
  if (n < 0 || (n > 0 && (!t_ns || !cov12))) return fail(CTVIO_ERR_INVALID, "ctvio_pose_covariance: bad argument");
  if (camera_frame != 0 && camera_frame != 1) return fail(CTVIO_ERR_INVALID, "ctvio_pose_covariance: camera_frame must be 0 or 1");
  if (int rc = check_covariance_call(e, gauge_knot_index, "ctvio_pose_covariance")) return rc;
  if (n == 0) return CTVIO_OK;
  if (!e->have_knots) return fail(CTVIO_ERR_STATE, "knots have not been set");
  if (!times_inside(e->sp, n, t_ns)) return fail(CTVIO_ERR_TIME_RANGE, "ctvio_pose_covariance: a time outside the spline");
  int rc = form_covariance(e, gauge_knot_index, "ctvio_pose_covariance", rcond);
  if (rc) return rc;
  auto& w = e->cws;
  CUDA_OK(w.t.reserve(size_t(n)));
  CUDA_OK(w.pose.reserve(144 * size_t(n)));
  CUDA_OK(cudaMemcpyAsync(w.t.p, t_ns, size_t(n) * sizeof(int64_t), cudaMemcpyHostToDevice, e->stream));
  e->h2d_bytes += size_t(n) * sizeof(int64_t);
  PoseCovLaunch a = {};
  a.n = n; a.camera_frame = camera_frame;
  a.t = w.t.p;
  launch_pose_covariance(e, a, w.pose.p);
  return read_result(e, cov12, w.pose.p, 144 * size_t(n));
}

extern "C" int ctvio_relative_pose_covariance(ctvio_handle e, int32_t n, const int64_t* t_a_ns, const int64_t* t_b_ns,
                                              int32_t gauge_knot_index, int32_t camera_frame, double* cov6,
                                              double* cross6, double* rcond) {
  if (!e) return fail(CTVIO_ERR_INVALID, "null handle");
  if (n < 0 || (n > 0 && (!t_a_ns || !t_b_ns || !cov6)))
    return fail(CTVIO_ERR_INVALID, "ctvio_relative_pose_covariance: bad argument");
  if (camera_frame != 0 && camera_frame != 1)
    return fail(CTVIO_ERR_INVALID, "ctvio_relative_pose_covariance: camera_frame must be 0 or 1");
  if (int rc = check_covariance_call(e, gauge_knot_index, "ctvio_relative_pose_covariance")) return rc;
  if (n == 0) return CTVIO_OK;
  if (!e->have_knots) return fail(CTVIO_ERR_STATE, "knots have not been set");
  if (!times_inside(e->sp, n, t_a_ns) || !times_inside(e->sp, n, t_b_ns))
    return fail(CTVIO_ERR_TIME_RANGE, "ctvio_relative_pose_covariance: a time outside the spline");
  int rc = form_covariance(e, gauge_knot_index, "ctvio_relative_pose_covariance", rcond);
  if (rc) return rc;
  cudaStream_t st = e->stream;
  auto& w = e->cws;
  const size_t nn = size_t(n);
  CUDA_OK(w.t.reserve(2 * nn));
  CUDA_OK(w.pose.reserve((cross6 ? 72 : 36) * nn));  // cov6, then cross6
  CUDA_OK(cudaMemcpyAsync(w.t.p, t_a_ns, nn * sizeof(int64_t), cudaMemcpyHostToDevice, st));
  CUDA_OK(cudaMemcpyAsync(w.t.p + nn, t_b_ns, nn * sizeof(int64_t), cudaMemcpyHostToDevice, st));
  e->h2d_bytes += 2 * nn * sizeof(int64_t);
  RelativePoseCovLaunch a = {};
  a.n = n; a.camera_frame = camera_frame;
  a.t_a = w.t.p;
  a.t_b = w.t.p + nn;
  a.cross = cross6 ? w.pose.p + 36 * nn : nullptr;
  launch_relative_pose_covariance(e, a, w.pose.p);
  if ((rc = copy_to_host(e, cov6, a.out, 36 * nn))) return rc;
  if (cross6 && (rc = copy_to_host(e, cross6, a.cross, 36 * nn))) return rc;
  CUDA_OK(stream_sync(st));
  return CTVIO_OK;
}

extern "C" int ctvio_point_covariance(ctvio_handle e, int32_t n, const int32_t* landmark, const int64_t* t_anchor_ns,
                                      const double* bearing_xy, int32_t gauge_knot_index, double* cov9, double* rcond) {
  if (!e) return fail(CTVIO_ERR_INVALID, "null handle");
  if (n < 0 || (n > 0 && (!landmark || !t_anchor_ns || !bearing_xy || !cov9)))
    return fail(CTVIO_ERR_INVALID, "ctvio_point_covariance: bad argument");
  for (int32_t i = 0; i < n; ++i)
    if (landmark[i] < 0 || landmark[i] >= e->nL) return fail(CTVIO_ERR_INVALID, "ctvio_point_covariance: landmark out of range");
  if (int rc = check_covariance_call(e, gauge_knot_index, "ctvio_point_covariance")) return rc;
  if (n == 0) return CTVIO_OK;
  if (!e->have_knots) return fail(CTVIO_ERR_STATE, "knots have not been set");
  if (!times_inside(e->sp, n, t_anchor_ns))
    return fail(CTVIO_ERR_TIME_RANGE, "ctvio_point_covariance: an anchor time outside the spline");
  int rc = form_covariance(e, gauge_knot_index, "ctvio_point_covariance", rcond);
  if (rc) return rc;
  cudaStream_t st = e->stream;
  auto& w = e->cws;
  CUDA_OK(w.lm.reserve(size_t(n)));
  CUDA_OK(w.t.reserve(size_t(n)));
  CUDA_OK(w.pose.reserve(11 * size_t(n)));  // outputs, then the bearings
  CUDA_OK(cudaMemcpyAsync(w.lm.p, landmark, size_t(n) * sizeof(int32_t), cudaMemcpyHostToDevice, st));
  CUDA_OK(cudaMemcpyAsync(w.t.p, t_anchor_ns, size_t(n) * sizeof(int64_t), cudaMemcpyHostToDevice, st));
  CUDA_OK(cudaMemcpyAsync(w.pose.p + 9 * size_t(n), bearing_xy, 2 * size_t(n) * sizeof(double), cudaMemcpyHostToDevice, st));
  e->h2d_bytes += 28 * size_t(n);
  PointCovLaunch a = {};
  a.n = n;
  a.landmark = w.lm.p;
  a.t = w.t.p;
  a.bearing = w.pose.p + 9 * size_t(n);
  return point_covariance(e, a, cov9);
}

extern "C" int ctvio_feature_table_point_covariance(ctvio_handle e, int32_t n_landmarks, int32_t gauge_knot_index,
                                                    double* cov9, double* rcond) {
  if (!e) return fail(CTVIO_ERR_INVALID, "null handle");
  if (int rc = check_covariance_call(e, gauge_knot_index, "ctvio_feature_table_point_covariance")) return rc;
  auto& ft = e->ft;
  if (!ft.window_current) return fail(CTVIO_ERR_STATE, "no feature-table window since the last add / slide");
  if (e->nL != ft.n_lm) return fail(CTVIO_ERR_STATE, "the resident inverse depths no longer follow the table's numbering");
  if (n_landmarks != ft.n_lm)
    return fail(CTVIO_ERR_INVALID, "ctvio_feature_table_point_covariance: n_landmarks differs from the window's landmark count");
  if (n_landmarks > 0 && !cov9) return fail(CTVIO_ERR_INVALID, "ctvio_feature_table_point_covariance: null argument");
  if (n_landmarks == 0) return CTVIO_OK;
  if (!e->have_knots) return fail(CTVIO_ERR_STATE, "knots have not been set");
  if (!held_frames_inside(e))  // every anchor is a held slot
    return fail(CTVIO_ERR_TIME_RANGE, "ctvio_feature_table_point_covariance: a held frame time falls outside the spline");
  int rc = form_covariance(e, gauge_knot_index, "ctvio_feature_table_point_covariance", rcond);
  if (rc) return rc;
  // the anchors come from the window's observation CSR and the frame table: nothing goes up
  PointCovLaunch a = {};
  a.n = n_landmarks;
  table_anchors(e, a);
  return point_covariance(e, a, cov9);
}

namespace ctvio::host {

int rank_test(const LmPublished& pub, const char* who, std::string* why) {
  if (pub.s.error_flags & 1) {
    *why = "a factor time left its knot window / the spline (line delay too large?)";
    return CTVIO_ERR_TIME_RANGE;
  }
  const double rc_value = pub.rcond;
  const bool failed = pub.s.chol_fail != 0;
  // Ceres' default min_reciprocal_condition_number; the estimate is the pivot ratio, see include/ctvio.h
  if (failed || !(rc_value >= 1e-14)) {
    char msg[128];
    std::snprintf(msg, sizeof(msg), "%s: rank deficient (rcond %.3e%s)", who, rc_value, failed ? ", non-positive pivot" : "");
    *why = msg;
    return CTVIO_ERR_STATE;
  }
  return CTVIO_OK;
}

bool times_inside(const SplineParams& sp, int n, const int64_t* t) {
  int32_t s;
  double u;
  for (int i = 0; i < n; ++i)
    if (!spline_index(sp, t[i], s, u)) return false;
  return true;
}

bool held_frames_inside(ctvio_engine* e) {
  for (int slot = 0; slot < ctvio_engine::kFrameSlots; ++slot)
    if ((e->ft.held >> slot & 1u) && !times_inside(e->sp, 1, &e->h_frame_t[slot])) return false;
  return true;
}

// the cycle's device workspace cov_out: cov12 (144) | cov6 [15][36] | cov9 [n_landmarks][9]
constexpr size_t kCycleCov6 = 144, kCycleCov9 = kCycleCov6 + 36 * (kKeyframeMaxSlots - 1);

int cycle_covariance_enqueue(ctvio_engine* e, int gauge_knot, bool pose, bool rel, bool points) {
  auto& c = e->cyc;
  auto& cv = c.cov;
  if (!c.cov_host) {
    void* p = nullptr;
    if (cudaHostAlloc(&p, sizeof(CycleCovHost), cudaHostAllocMapped) != cudaSuccess) {
      cudaGetLastError();
      return fail(CTVIO_ERR_CUDA, "could not allocate the mapped covariance buffer");
    }
    c.cov_host = static_cast<CycleCovHost*>(p);
  }
  // sized for any window once: a growing reserve() would free, and cudaFree waits for the device
  CUDA_OK(c.cov_t.reserve(1 + kKeyframeMaxSlots));
  CUDA_OK(c.cov_out.reserve(kCycleCov9 + 9 * size_t(kFeatureTableMaxEntries)));
  CycleCovHost* h = c.cov_host;
  const int nf = cv.n_frames, n_pairs = rel ? nf - 1 : 0;
  // the times go up from the mapped block (the last cycle's copy out of it completed before that cycle ended)
  const int n_t = (pose || n_pairs > 0) ? 1 + (n_pairs > 0 ? nf : 0) : 0;
  h->t[0] = cv.pose_t;
  for (int k = 0; k < nf; ++k) h->t[1 + k] = cv.frame_t[k];
  if (n_t) {
    CUDA_OK(cudaMemcpyAsync(c.cov_t.p, h->t, size_t(n_t) * sizeof(int64_t), cudaMemcpyHostToDevice, e->stream));
    e->h2d_bytes += size_t(n_t) * sizeof(int64_t);
  }
  if (const int rc = enqueue_covariance(e, gauge_knot, &h->pub, ++cv.seq)) return rc;
  if (pose) {  // the camera pose and velocity at the TF time: ctvio_pose_covariance(camera_frame = 1)
    PoseCovLaunch a = {};
    a.n = 1; a.camera_frame = 1;
    a.t = c.cov_t.p;
    launch_pose_covariance(e, a, c.cov_out.p);
    if (const int rc = copy_to_host(e, h->cov12, a.out, 144)) return rc;
  }
  if (n_pairs > 0) {  // the odometry edges (t[i], t[i + 1]): ctvio_relative_pose_covariance(camera_frame = 1)
    RelativePoseCovLaunch a = {};
    a.n = n_pairs; a.camera_frame = 1;
    a.t_a = c.cov_t.p + 1;
    a.t_b = c.cov_t.p + 2;
    launch_relative_pose_covariance(e, a, c.cov_out.p + kCycleCov6);
    if (const int rc = copy_to_host(e, h->cov6, a.out, 36 * size_t(n_pairs))) return rc;
  }
  if (points && cv.n_lm > 0) {  // the window landmarks' world points, anchored as the table holds them: stay on the
                                // device until the map kernel gathers them
    PointCovLaunch a = {};
    a.n = cv.n_lm;
    table_anchors(e, a);
    launch_point_covariance(e, a, c.cov_out.p + kCycleCov9);
  }
  return CTVIO_OK;
}

const double* cycle_point_covariances(ctvio_engine* e) { return e->cyc.cov_out.p + kCycleCov9; }

}  // namespace ctvio::host
