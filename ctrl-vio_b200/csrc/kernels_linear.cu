// Linear-algebra / LM-step kernels of the CUDA engine (sm_90a, fp64).
//
// Replaces what Ceres does inside ceres::Solve for one trust-region step
// (trajectory_estimator.cpp:367-408 -> Ceres 1.14 levenberg_marquardt_strategy.cc +
// SPARSE_NORMAL_CHOLESKY; Ceres is not part of the reference repository):
//   K4  reduced_system         reduced camera system  M = S A S + D^2 - sum_l w_l w_l' / h_l
//   K5  (chol_dag.cu, chol_coop.cu) dense Cholesky (NB = 64) + block triangular solves
//   K6  backsub / quad / apply landmark back-substitution, model cost change, x (+) delta, norms
// The Schur complement is owner-computes by OUTPUT tile: every 64x64 tile of the lower triangle of M gets the list of
// landmarks whose coupling row touches both of its blocks (built on the host), split into parts so that small
// windows still fill the GPU; a CTA builds the scaled rows of 32 landmarks at a time in shared memory and reduces
// them with fp64 tensor-core tiles (m8n8k4), then flushes its tile once.
#include <algorithm>
#include <atomic>

#include "dmma_tiles.cuh"
#include <cstddef>

#include "kernels.h"

namespace ctvio {

// atomic max for non-negative doubles (bit pattern order == value order)
__device__ __forceinline__ void atomic_max_pos(double* addr, double v) {
  atomicMax(reinterpret_cast<unsigned long long*>(addr), static_cast<unsigned long long>(__double_as_longlong(v)));
}

constexpr double kMinLmDiag = 1e-6, kMaxLmDiag = 1e32;  // Ceres min/max_lm_diagonal

// ------------------------------------------------------------------------------------------------
__global__ void jacobi_scale_kernel(LinearLaunch a) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const int np = a.dims.np;
  if (i < np) a.sc[i] = 1.0 / (1.0 + sqrt(a.ne.A[size_t(i) * np + i]));
  if (i < a.dims.nL) a.sl[i] = 1.0 / (1.0 + sqrt(a.ne.hl[i]));
}
int launch_jacobi_scale(const LinearLaunch& a, cudaStream_t s) {
  const int n = max(a.dims.np, a.dims.nL);
  jacobi_scale_kernel<<<(n + 255) / 256, 256, 0, s>>>(a);
  return 1;
}

// ------------------------------------------------------------------------------------------------
// K4: the damped, scaled reduced camera system M = S A S + D^2 - sum_l w_l w_l' / h_l and rhs = S g_c - sum_l w_l c_l,
// in ONE launch.  Blocks [0, T (T + 1) / 2) are BASE CTAs, one per 64x64 tile (ti >= tj) of the lower triangle: each
// writes its tile of S A S + damping (identity / zero on constant and padding dims) and, on the diagonal, its block of
// rhs, then publishes the tile with an epoch-valued release flag.  The remaining blocks are ITEM CTAs, one per
// SchurTileItem: a part of the landmark list of one tile, reduced 32 landmarks at a time on DMMA and subtracted from the
// tile with fp64 RED atomics once the tile's base CTA has published it.  Only the lower tiles are written (the diagonal
// tiles in full); K5 reads nothing else.
//
// Ordering: an item CTA spins only on the flags of base CTAs, whose block indices are all lower than its own.  Blocks
// are dispatched in index order, so those base CTAs are resident or done when the item CTA spins, and a base CTA waits
// for nothing but the preceding kernel (pdl_wait): no deadlock (the argument det_ticket_wait relies on).  Deterministic
// mode: the item CTAs flush in item order, so the atomics land in the order of the item list.
// Before pdl_wait a CTA reads only what was written two or more launches back (A, g_c, W, the landmark diagonals and
// gradients, the Jacobi scales, the work lists): the radius, the go flag and the per-step accumulators belong to the
// preceding gradient_norm_kernel.
constexpr int kSchurKC = 32;   // landmarks per shared-memory operand chunk
constexpr int kBaseTS = kCholNB + 1;  // row stride of a base CTA's tile of A (odd: its column reads are conflict-free)
static_assert(kCholNB * kBaseTS <= 2 * kSchurKC * kTS, "the base tile lives in the item operands' shared memory");

__host__ __device__ __forceinline__ int lower_tile_index(int ti, int tj) { return ti * (ti + 1) / 2 + tj; }
size_t reduced_system_flags_len(int npad) {
  const int T = npad / kCholNB;
  return size_t(lower_tile_index(T, 0));
}

// per-landmark prologue of the Schur complement: damped diagonal hh and the scale is = sl / sqrt(hh) of the coupling row
__device__ __forceinline__ double landmark_hh(double sl, double hl, double radius) {
  const double hs = sl * sl * hl;
  return hl > 0.0 ? hs + fmin(fmax(hs, kMinLmDiag), kMaxLmDiag) / radius : 0.0;
}
__device__ __forceinline__ double landmark_is(double hh, double sl) { return hh > 0.0 ? rsqrt(hh) * sl : 0.0; }

// base CTA b: tile (ti, tj) of S A S + clamp(diag) / radius, rhs = S g_c on the diagonal
__device__ __forceinline__ void reduced_base_block(const LinearLaunch& a, int b, double radius, const double* radius_dev,
                                                   int epoch, double* Ts, double* scR, double* scC, uint8_t* cmR,
                                                   uint8_t* cmC) {
  const int tid = threadIdx.x;
  int ti = 0;
  while (lower_tile_index(ti + 1, 0) <= b) ++ti;
  const int tj = b - lower_tile_index(ti, 0);
  const int npad = a.npad, np = a.dims.np;
  const int r0 = kCholNB * ti, c0 = kCholNB * tj;
  // the tile's block of A, read row-wise from the upper triangle: Ts[x][y] = A[c0 + x][r0 + y]
  // (M[r][c] = A[c][r] below the diagonal; diagonal tiles use Ts[x][y] for x <= y)
#pragma unroll
  for (int k = 0; k < kCholNB * kCholNB / 256; ++k) {
    const int e = tid + 256 * k, x = e / kCholNB, y = e % kCholNB;
    Ts[x * kBaseTS + y] = (c0 + x < np && r0 + y < np) ? a.ne.A[size_t(c0 + x) * np + r0 + y] : 0.0;
  }
  // the first landmark of this thread's share of the hh prologue below
  const int nbase = lower_tile_index(npad / kCholNB, 0), l0 = b * 256 + tid;
  const double sl0 = l0 < a.dims.nL ? a.sl[l0] : 0.0, hl0 = l0 < a.dims.nL ? a.ne.hl[l0] : 0.0;
  double rg = 0.0;
  if (tid < kCholNB) {
    const int i = r0 + tid, j = c0 + tid;
    scR[tid] = i < np ? a.sc[i] : 0.0;
    cmR[tid] = i < np ? a.cmask[i] : 1;
    scC[tid] = j < np ? a.sc[j] : 0.0;
    cmC[tid] = j < np ? a.cmask[j] : 1;
    if (ti == tj && i < np) rg = a.ne.gc[i];
  }
  __syncthreads();
  pdl_wait();
  pdl_launch_dependents();
  if (radius_dev) radius = *radius_dev;  // speculated step: decided by the previous step's gradient_norm_kernel
  const double ident = a.sharded ? 0.0 : 1.0;  // sharded: identity rows are set after the all-reduce
  double* tile = a.M + size_t(r0) * npad + c0;
#pragma unroll 4
  for (int k = 0; k < kCholNB * kCholNB / 256; ++k) {
    const int e = tid + 256 * k, rr = e / kCholNB, cc = e % kCholNB;
    const int i = r0 + rr, j = c0 + cc;
    double m;
    if (i < np && j < np) {
      if (cmR[rr] || cmC[cc]) {
        m = (i == j) ? ident : 0.0;
      } else {
        const double v = (i <= j) ? Ts[rr * kBaseTS + cc] : Ts[cc * kBaseTS + rr];
        m = scR[rr] * v * scC[cc];
        if (i == j) {
          if (a.sharded) a.diagA[i] = v;  // unscaled local diagonal, summed over ranks with M
          else m += fmin(fmax(m, kMinLmDiag), kMaxLmDiag) / radius;
        }
      }
    } else {
      m = (i == j) ? ident : 0.0;
      if (a.sharded && i == j) a.diagA[i] = 0.0;
    }
    if (a.sharded && i == j && i < np && cmR[rr]) a.diagA[i] = 0.0;
    tile[size_t(rr) * npad + cc] = m;
  }
  if (ti == tj && tid < kCholNB) a.rhs[r0 + tid] = (r0 + tid < np && !cmR[tid]) ? scR[tid] * rg : 0.0;
  __syncthreads();
  if (tid == 0) {
    __threadfence();
    st_release_gpu(a.m_flags + b, epoch);
  }
  // the landmark diagonals (step_apply_kernel reads them), and the per-step accumulators of the kernels that follow in
  // this LM step (no separate memsets on the stream); nothing in this launch reads either
  if (l0 < a.dims.nL) a.hh[l0] = landmark_hh(sl0, hl0, radius);
  for (int l = l0 + nbase * 256; l < a.dims.nL; l += nbase * 256) a.hh[l] = landmark_hh(a.sl[l], a.ne.hl[l], radius);
  if (b == 0 && tid == 0) {
    a.scal->gd = 0.0;
    a.scal->dHd = 0.0;
    a.scal->dir_max = 0.0;
    a.scal->chol_fail = 0;
    a.scal->step_norm2 = 0.0;
    a.scal->x_norm2 = 0.0;
    a.scal->cost_eval = 0.0;
    a.scal->gmax = 0.0;
  }
}

// landmark k of chunk [c0, c0 + 32) of an item (thread = (landmark k, 8 consecutive dims)): its coupling row restricted
// to the tile's blocks and its scalars, as loaded; nothing here depends on the trust-region radius
struct SchurRow {
  double va[8], vb[8];
  double sl, hl, gl, wld;
  int32_t lo, hi;  // the landmark's knot-dim range; lo < 0: no landmark in this slot
};
__device__ __forceinline__ void schur_load(const LinearLaunch& a, const SchurTileItem& it, int c0, int k, int dseg, bool diag,
                                           SchurRow& r) {
#pragma unroll
  for (int e = 0; e < 8; ++e) r.va[e] = r.vb[e] = 0.0;
  r.lo = -1;
  if (c0 + k >= it.count) return;
  const SchurEntry en = a.schur_list[it.first + c0 + k];
  const double* Wl = a.ne.W + en.woff - en.lo;
  const int ga0 = kCholNB * it.ti + dseg, gb0 = kCholNB * it.tj + dseg;
  r.lo = en.lo;
  r.hi = en.hi;
  r.sl = a.sl[en.l];
  r.hl = a.ne.hl[en.l];
  r.gl = a.ne.gl[en.l];
  r.wld = a.ne.wld[en.l];
  if (ga0 + 8 > en.lo && ga0 < en.hi) {
#pragma unroll
    for (int e = 0; e < 8; ++e)
      if (ga0 + e >= en.lo && ga0 + e < en.hi) r.va[e] = Wl[ga0 + e];
  }
  if (!diag && gb0 + 8 > en.lo && gb0 < en.hi) {
#pragma unroll
    for (int e = 0; e < 8; ++e)
      if (gb0 + e >= en.lo && gb0 + e < en.hi) r.vb[e] = Wl[gb0 + e];
  }
}
// -> the scaled rows v = is W_l S in place, and cl = {c_l = is g_l, v_l[line delay], first-block flag}
__device__ __forceinline__ void schur_scale(const SchurTileItem& it, int dseg, const double* scA, const double* scB,
                                            double sc_ld, bool diag, double radius, SchurRow& r, double cl[3]) {
  cl[0] = cl[1] = cl[2] = 0.0;
  if (r.lo < 0) return;
  const double is = landmark_is(landmark_hh(r.sl, r.hl, radius), r.sl);
  const int ga0 = kCholNB * it.ti + dseg, gb0 = kCholNB * it.tj + dseg;
  cl[0] = is * r.gl;
  cl[1] = is * r.wld * sc_ld;
  cl[2] = r.lo / kCholNB == it.ti ? 1.0 : 0.0;  // exactly one diagonal tile counts the landmark's ld-ld / ld-rhs terms
#pragma unroll
  for (int e = 0; e < 8; ++e)
    if (ga0 + e >= r.lo && ga0 + e < r.hi) r.va[e] = is * r.va[e] * scA[dseg + e];
  if (!diag) {
#pragma unroll
    for (int e = 0; e < 8; ++e)
      if (gb0 + e >= r.lo && gb0 + e < r.hi) r.vb[e] = is * r.vb[e] * scB[dseg + e];
  }
}

// item CTA: part `item` of the landmark list of one output tile
__device__ __forceinline__ void reduced_item_block(const LinearLaunch& a, int item, double radius, const double* radius_dev,
                                                   int epoch, double* At, double* Bt, double* scA, double* scB,
                                                   double (*cvec)[kSchurKC]) {
  const SchurTileItem it = a.schur_items[item];
  const int tid = threadIdx.x;
  const Lane L = lane_of(tid);
  const int np = a.dims.np, npad = a.npad, ild = a.dims.idx_ld;
  const bool diag = it.ti == it.tj;
  if (tid < kCholNB) {
    const int ga = kCholNB * it.ti + tid, gb = kCholNB * it.tj + tid;
    scA[tid] = (ga < np && !a.cmask[ga]) ? a.sc[ga] : 0.0;
    scB[tid] = (gb < np && !a.cmask[gb]) ? a.sc[gb] : 0.0;
  }
  const double sc_ld = a.cmask[ild] ? 0.0 : a.sc[ild];
  const int k = tid >> 3, dseg = (tid & 7) * 8;
  SchurRow row;
  schur_load(a, it, 0, k, dseg, diag, row);  // the first chunk's loads fly through the wait
  __syncthreads();
  pdl_wait();
  pdl_launch_dependents();
  const int go = a.go ? *a.go : 1;
  if (radius_dev) radius = *radius_dev;  // (one round trip for both loads)
  if (!go) return;  // speculated step behind a rejected / terminating one
  Frag acc;
  frag_zero(acc);
  // diagonal tiles also own, for their block: rhs -= sum_l v_l c_l and the line-delay row M[ld][block] -= sum_l v_l vld_l;
  // lanes 0..31 of warp 0 (one landmark slot each) collect the ld-ld and ld-rhs terms of the landmarks starting here
  double racc = 0.0, lacc = 0.0, ll = 0.0, lr = 0.0;
  for (int c0 = 0; c0 < it.count; c0 += kSchurKC) {
    double cl[3];
    schur_scale(it, dseg, scA, scB, sc_ld, diag, radius, row, cl);
#pragma unroll
    for (int e = 0; e < 8; e += 2) {
      *reinterpret_cast<double2*>(At + k * kTS + dseg + e) = make_double2(row.va[e], row.va[e + 1]);
      if (!diag) *reinterpret_cast<double2*>(Bt + k * kTS + dseg + e) = make_double2(row.vb[e], row.vb[e + 1]);
    }
    if ((tid & 7) == 0) { cvec[0][k] = cl[0]; cvec[1][k] = cl[1]; cvec[2][k] = cl[2]; }
    __syncthreads();
    // the next chunk's global loads fly while the tensor cores chew on this one
    if (c0 + kSchurKC < it.count) schur_load(a, it, c0 + kSchurKC, k, dseg, diag, row);
    tile_gemm_dmma<false, kSchurKC>(At, diag ? At : Bt, acc, L);
    if (diag) {
      if (tid < kCholNB) {
#pragma unroll 8
        for (int kk = 0; kk < kSchurKC; ++kk) {
          const double v = At[kk * kTS + tid];
          racc = fma(v, cvec[0][kk], racc);
          lacc = fma(v, cvec[1][kk], lacc);
        }
      } else if (tid < kCholNB + kSchurKC) {
        const int kk = tid - kCholNB;
        const double vld = cvec[1][kk] * cvec[2][kk];
        ll = fma(vld, cvec[1][kk], ll);
        lr = fma(vld, cvec[0][kk], lr);
      }
    }
    __syncthreads();
  }
  // flush: M_tile -= acc (several parts may share a tile: fp64 RED atomics), rhs_block -= racc, once the base CTAs of the
  // tiles written here have published them: the tile itself and, for a diagonal tile, the line-delay row's tiles
  {
    const int tl = ild / kCholNB;
    if (tid == 0) spin_until_gpu(a.m_flags + lower_tile_index(it.ti, it.tj), epoch);
    else if (diag && tid == 32) spin_until_gpu(a.m_flags + lower_tile_index(tl, it.ti), epoch);
    else if (diag && tid == 64) spin_until_gpu(a.m_flags + lower_tile_index(tl, tl), epoch);
    __syncthreads();
  }
  det_ticket_wait(a.det_ticket, item);
  double* tile = a.M + size_t(kCholNB) * it.ti * npad + kCholNB * it.tj;
#pragma unroll
  for (int mt = 0; mt < 2; ++mt)
#pragma unroll
    for (int nt = 0; nt < 4; ++nt)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const double v = acc.c[mt][nt][e];
        if (v != 0.0) atomicAdd(tile + size_t(L.row(mt)) * npad + L.col(nt) + e, -v);
      }
  if (diag) {
    if (tid < kCholNB) {
      if (racc != 0.0) atomicAdd(a.rhs + kCholNB * it.ti + tid, -racc);
      if (lacc != 0.0) atomicAdd(a.M + size_t(ild) * npad + kCholNB * it.ti + tid, -lacc);  // row ld is the last one: lower
    } else if (tid < kCholNB + kSchurKC) {
      ll = warp_sum_d(ll);
      lr = warp_sum_d(lr);
      if (tid == kCholNB) {
        if (ll != 0.0) atomicAdd(a.M + size_t(ild) * npad + ild, -ll);
        if (lr != 0.0) atomicAdd(a.rhs + ild, -lr);
      }
    }
  }
  det_ticket_done(a.det_ticket, item);
}

__global__ void __launch_bounds__(256, 2) reduced_system_kernel(LinearLaunch a, double radius,
                                                                const double* __restrict__ radius_dev, int epoch) {
  __shared__ __align__(16) double opnd[2 * kSchurKC * kTS];  // item: At | Bt; base: the tile of A
  __shared__ double scA[kCholNB], scB[kCholNB], cvec[3][kSchurKC];
  __shared__ uint8_t cmA[kCholNB], cmB[kCholNB];
  const int nbase = lower_tile_index(a.npad / kCholNB, 0);
  if (int(blockIdx.x) < nbase) reduced_base_block(a, blockIdx.x, radius, radius_dev, epoch, opnd, scA, scB, cmA, cmB);
  else reduced_item_block(a, blockIdx.x - nbase, radius, radius_dev, epoch, opnd, opnd + kSchurKC * kTS, scA, scB, cvec);
}

// ------------------------------------------------------------------------------------------------
// K5 (blocked Cholesky + triangular solves) lives in chol_coop.cu

// ------------------------------------------------------------------------------------------------
// K6
// camera part of the step: dc = -sc o y ; gd += gc.dc ; dHd += dc' A dc ; dir_max
__device__ __forceinline__ void camera_step_block(const LinearLaunch& a, int block, double* dsh) {
  __shared__ double red[3][8];
  const int np = a.dims.np;
  const int i = block * 8 + (threadIdx.x >> 5);  // one warp per row
  const int lane = threadIdx.x & 31;
  double gd = 0, dHd = 0, dmax = 0;
  // the part of the step this CTA's rows need (columns >= first row), staged once: the row loops then only stream A
  const int j0 = block * 8;
  for (int j = j0 + threadIdx.x; j < np; j += blockDim.x) dsh[j - j0] = a.cmask[j] ? 0.0 : -a.sc[j] * a.y[j];
  __syncthreads();
  if (i < np) {
    const double di = dsh[i - j0];
    if (lane == 0) {
      a.dc[i] = di;
      gd = a.ne.gc[i] * di;
      dmax = fabs(di);
      if (!isfinite(di)) a.scal->chol_fail = 1;
    }
    if (di != 0.0) {
      double s = 0;
      for (int j = i + lane; j < np; j += 32) s = fma(a.ne.A[size_t(i) * np + j] * (j == i ? 0.5 : 1.0), dsh[j - j0], s);
      dHd = 2.0 * di * s;
    }
  }
  dHd = warp_sum_d(dHd);
  if (lane == 0) { red[0][threadIdx.x >> 5] = gd; red[1][threadIdx.x >> 5] = dHd; red[2][threadIdx.x >> 5] = dmax; }
  __syncthreads();
  det_ticket_wait(a.det_ticket ? a.det_ticket + 1 : nullptr, blockIdx.x);
  if (threadIdx.x == 0) {
    double g = 0, h = 0, m = 0;
    for (int w = 0; w < 8; ++w) { g += red[0][w]; h += red[1][w]; m = fmax(m, red[2][w]); }
    atomicAdd(&a.scal->gd, g);
    atomicAdd(&a.scal->dHd, h);
    atomic_max_pos(&a.scal->dir_max, m);
  }
  det_ticket_done(a.det_ticket ? a.det_ticket + 1 : nullptr, blockIdx.x);
}

// landmark back-substitution + landmark parts of gd / dHd: one WARP per landmark (coalesced reads of
// its coupling row), reads y (not dc) so that it can run concurrently with camera_step_kernel.
__device__ __forceinline__ void landmark_step_block(const LinearLaunch& a, int block, const ApplyLaunch* ap = nullptr) {
  __shared__ double red[3][8];
  __shared__ double red2[2][8];
  double xn = 0, sn = 0;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int l = block * 8 + warp;
  double gd = 0, dHd = 0, dmax = 0;
  if (l < a.dims.nL) {
    const double sl = a.sl[l];
    const int lo = a.lm.lo[l], hi = a.lm.hi[l], ild = a.dims.idx_ld;
    const double* Wl = a.ne.W + a.lm.woff[l] - lo;
    double wy = 0;  // W_l . (sc o y)
    for (int g = lo + lane; g < hi; g += 32) wy = fma(Wl[g], a.cmask[g] ? 0.0 : a.sc[g] * a.y[g], wy);
    wy = warp_sum_d(wy);
    if (lane == 0) {
      wy = fma(a.ne.wld[l], a.cmask[ild] ? 0.0 : a.sc[ild] * a.y[ild], wy);
      const double hh = a.hh[l];
      const double yl = hh > 0.0 ? (sl * a.ne.gl[l] - sl * wy) / hh : 0.0;
      const double d = -sl * yl;
      a.dl[l] = d;
      gd = a.ne.gl[l] * d;
      dHd = 2.0 * d * (-wy) + a.ne.hl[l] * d * d;  // W_l . dc = -wy
      dmax = fabs(d);
      if (!isfinite(d)) a.scal->chol_fail = 1;
      if (ap) {  // fused apply (alpha = 1): candidate inverse depth and its share of the norms
        const double v = ap->x.rho[l], vn = v + d;
        ap->xc.rho[l] = vn;
        if (ap->active[a.dims.np + l]) { xn = v * v; sn = (v - vn) * (v - vn); }
      }
    }
  }
  if (lane == 0) { red[0][warp] = gd; red[1][warp] = dHd; red[2][warp] = dmax; red2[0][warp] = xn; red2[1][warp] = sn; }
  __syncthreads();
  det_ticket_wait(a.det_ticket ? a.det_ticket + 1 : nullptr, blockIdx.x);
  if (threadIdx.x == 0) {
    double g = 0, h = 0, m = 0, x = 0, s = 0;
    for (int w = 0; w < 8; ++w) { g += red[0][w]; h += red[1][w]; m = fmax(m, red[2][w]); x += red2[0][w]; s += red2[1][w]; }
    if (g != 0.0) atomicAdd(&a.scal->gd, g);
    if (h != 0.0) atomicAdd(&a.scal->dHd, h);
    if (m > 0.0) atomic_max_pos(&a.scal->dir_max, m);
    if (x != 0.0) atomicAdd(&a.scal->x_norm2, x);
    if (s != 0.0) atomicAdd(&a.scal->step_norm2, s);
  }
  det_ticket_done(a.det_ticket ? a.det_ticket + 1 : nullptr, blockIdx.x);
}

// after the all-reduce of [M | rhs | diagA]
// both halves of the step in ONE launch: blocks [0, ncb) take camera rows, the rest take landmarks (the landmark
// half reads y, not dc, so the two are independent)
__global__ void __launch_bounds__(256) step_vectors_kernel(LinearLaunch a, int ncb) {
  extern __shared__ double step_dsh[];  // [np]
  if (int(blockIdx.x) < ncb) camera_step_block(a, blockIdx.x, step_dsh);
  else landmark_step_block(a, blockIdx.x - ncb, nullptr);
}

__global__ void extract_diag_kernel(LinearLaunch a) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= a.npad) return;
  a.diagA[i] = i < a.dims.np ? a.ne.A[size_t(i) * a.dims.np + i] : 0.0;
}
int launch_extract_diag(const LinearLaunch& a, cudaStream_t s) {
  extract_diag_kernel<<<(a.npad + 255) / 256, 256, 0, s>>>(a);
  return 1;
}
__global__ void jacobi_scale_from_diag_kernel(LinearLaunch a) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < a.dims.np) a.sc[i] = 1.0 / (1.0 + sqrt(a.diagA[i]));
  if (i < a.dims.nL) a.sl[i] = 1.0 / (1.0 + sqrt(a.ne.hl[i]));
}
int launch_jacobi_scale_from_diag(const LinearLaunch& a, cudaStream_t s) {
  const int n = max(a.dims.np, a.dims.nL);
  jacobi_scale_from_diag_kernel<<<(n + 255) / 256, 256, 0, s>>>(a);
  return 1;
}

int launch_reduced_system(const LinearLaunch& a, double radius, cudaStream_t s, const double* radius_dev) {
  // process-wide unique, never 0 (flag buffers start zeroed): a tile flag never holds the epoch of a launch before it
  static std::atomic<unsigned> epoch_src{0};
  const int epoch = int(epoch_src.fetch_add(1, std::memory_order_relaxed) % 0x7ffffffeu) + 1;
  const int nbase = lower_tile_index(a.npad / kCholNB, 0);
  launch_chained(a.pdl, reduced_system_kernel, dim3(unsigned(nbase + a.n_schur_items)), dim3(256), 0, s, a, radius,
                 radius_dev, epoch);
  return 1;
}

int launch_step_vectors(const LinearLaunch& a, cudaStream_t s) {
  const int ncb = (a.dims.np + 7) / 8, nlb = (a.dims.nL + 7) / 8;
  step_vectors_kernel<<<ncb + nlb, 256, size_t(a.dims.np) * sizeof(double), s>>>(a, ncb);
  return 1;
}

int launch_lm_step(const LinearLaunch& a, double radius, cudaStream_t s) {
  return launch_reduced_system(a, radius, s) + launch_factor_solve(a, s) + launch_step_vectors(a, s);
}

// max-norm of the (bounds-projected) gradient over the active parameters; a few CTAs (one per 1024 entries, at most
// 16), combined with an integer atomicMax on the bit pattern (the values are non-negative); the CTA that arrives
// last hands the finished scalar block of the LM step to `pub` (mapped host memory)
__global__ void __launch_bounds__(1024) gradient_norm_kernel(LinearLaunch a, StatePtrs st, int fix_ld, double ld_lower,
                                                             double ld_upper, LmPublished* pub, unsigned long long seq,
                                                             LmDecideArgs da) {
  __shared__ double red[32];
  pdl_wait();
  pdl_launch_dependents();
  const int np = a.dims.np, nL = a.dims.nL;
  double v = 0.0;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < np + nL; i += gridDim.x * blockDim.x) {
    if (!a.active[i]) continue;
    double x;
    if (i < np) {
      x = fabs(a.ne.gc[i]);
      if (i == a.dims.idx_ld && !fix_ld) {
        const double ld = *st.ld;
        x = fabs(ld - fmin(fmax(ld - a.ne.gc[i], ld_lower), ld_upper));
      }
    } else {
      x = fabs(a.ne.gl[i - np]);
    }
    v = fmax(v, x);
  }
  v = warp_max_d(v);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  if (threadIdx.x < 32) {
    v = warp_max_d(red[threadIdx.x]);
    if (threadIdx.x == 0) {
      bool last = true;
      if (gridDim.x > 1) {
        atomicMax(reinterpret_cast<unsigned long long*>(&a.scal->gmax), static_cast<unsigned long long>(__double_as_longlong(v)));
        __threadfence();
        last = atomicAdd(&a.scal->pad[0], 1) == int(gridDim.x) - 1;
        if (last) a.scal->pad[0] = 0;  // (the arrival counter of the next launch)
      } else {
        a.scal->gmax = fmax(a.scal->gmax, v);
      }
      if (last && pub) {
        // the other kernels' atomics into the scalar block are complete (stream order) and live in L2: fetch the block
        // with six independent 16-byte L2 loads (one latency instead of eleven volatile reads) and hand it
        // to the host
        static_assert(sizeof(LmScalars) == 88, "scalar block is copied as five 16-byte words + one 8-byte word");
        __threadfence();
        const uint4* src = reinterpret_cast<const uint4*>(a.scal);
        uint4 w[5];
#pragma unroll
        for (int k = 0; k < 5; ++k) w[k] = __ldcg(src + k);
        const uint2 w5 = __ldcg(reinterpret_cast<const uint2*>(src + 5));
        uint4* dst = reinterpret_cast<uint4*>(&pub->s);
#pragma unroll
        for (int k = 0; k < 5; ++k) dst[k] = w[k];
        *reinterpret_cast<uint2*>(dst + 5) = w5;
        if (da.dec) {
          // accept / reject and the next radius, exactly as the host driver would compute them (the host ADOPTS these
          // values in pipelined mode, so the two can not disagree); no fused multiply-adds: same roundings as the
          // plain C++ expressions of the oracle
          LmScalars sc;
          uint4* loc = reinterpret_cast<uint4*>(&sc);
#pragma unroll
          for (int k = 0; k < 5; ++k) loc[k] = w[k];
          *reinterpret_cast<uint2*>(loc + 5) = w5;
          LmDecision d;
          d.model_cost_change = __dsub_rn(-sc.gd, __dmul_rn(0.5, sc.dHd));
          d.valid = (!sc.chol_fail && isfinite(d.model_cost_change) && d.model_cost_change > 0.0) ? 1 : 0;
          d.rho = __ddiv_rn(__dsub_rn(da.x_cost, sc.cost_eval), d.model_cost_change);
          d.accept = (d.valid && d.rho > da.min_relative_decrease) ? 1 : 0;
          const double t = __dsub_rn(__dmul_rn(2.0, d.rho), 1.0);
          const double t3 = __dmul_rn(__dmul_rn(t, t), t);
          d.radius_next = fmin(da.max_radius, __ddiv_rn(da.radius, fmax(1.0 / 3.0, __dsub_rn(1.0, t3))));
          // the driver's termination tests (same order as the host): a speculated step behind a terminating or
          // rejected one returns at once instead of running for nothing
          const double step_norm = sqrt(sc.step_norm2), x_norm = sqrt(sc.x_norm2);
          const bool stop = step_norm <= __dmul_rn(da.parameter_tolerance, __dadd_rn(x_norm, da.parameter_tolerance)) ||
                            fabs(__dsub_rn(da.x_cost, sc.cost_eval)) <= __dmul_rn(da.function_tolerance, da.x_cost) ||
                            fmax(sc.gmax, v) <= da.gradient_tolerance || d.radius_next < da.min_radius;
          d.go = (d.accept && !stop) ? 1 : 0;
          d.pad = 0;
          *da.dec = d;
          pub->dec = d;
        }
        __threadfence_system();
        *reinterpret_cast<volatile unsigned long long*>(&pub->seq) = seq;
      }
    }
  }
}
int launch_gradient_norm(const LinearLaunch& a, const StatePtrs& st, int fix_ld, double ld_lower, double ld_upper,
                         cudaStream_t s, bool reset, LmPublished* pub, unsigned long long seq, const LmDecideArgs* decide) {
  if (reset) cudaMemsetAsync(&a.scal->gmax, 0, sizeof(double), s);
  LmDecideArgs da{};
  if (decide) da = *decide;
  const int n = a.dims.np + a.dims.nL;
  const int grid = std::min(16, std::max(1, (n + 1023) / 1024));
  launch_chained(a.pdl, gradient_norm_kernel, dim3(grid), dim3(1024), 0, s, a, st, fix_ld, ld_lower, ld_upper, pub, seq, da);
  return 1;
}

// camera part of the step either from the stored vector dc or straight from the solution y of the reduced system
// (dc = -sc o y on the non-constant dims), so that the state update does not have to wait for the kernel that writes dc
struct StepSource {
  const double* dc;      // non-null: stored step
  const double* y;       // else: -sc[g] * y[g]
  const double* sc;
  const uint8_t* cmask;
  __device__ __forceinline__ double operator()(int g) const {
    if (dc) return dc[g];
    return cmask[g] ? 0.0 : -sc[g] * y[g];
  }
};

__device__ __forceinline__ Q4 stepped_knot(const ApplyLaunch& a, const StepSource& src, int i) {
  const double d0 = src(6 * i), d1 = src(6 * i + 1), d2 = src(6 * i + 2);
  const Q4 q = load_q(a.x.q, i);
  if (d0 != 0.0 || d1 != 0.0 || d2 != 0.0) return so3_mul(q, so3_exp(V3{a.alpha * d0, a.alpha * d1, a.alpha * d2}));
  return q;
}

// x+ = x (+) alpha * delta for element i of [knots | bias dims | line delay | landmarks (only if with_landmarks)]
__device__ __forceinline__ void apply_step_block(const ApplyLaunch& a, const StepSource& src, int block, bool with_landmarks) {
  __shared__ double red[2][8];
  const int i = block * blockDim.x + threadIdx.x;
  const int nK = a.dims.nK, nB = a.dims.nB, nL = with_landmarks ? a.dims.nL : 0;
  double xn = 0, sn = 0;
  if (i < nK) {
    const Q4 q = load_q(a.x.q, i);
    const Q4 qn = stepped_knot(a, src, i);
    a.xc.q[4 * i] = qn.x; a.xc.q[4 * i + 1] = qn.y; a.xc.q[4 * i + 2] = qn.z; a.xc.q[4 * i + 3] = qn.w;
    if (i + 1 < nK) {
      // K0 folded in: knot-pair table entry i of the candidate (knot i+1 is recomputed here, bit-identical to what
      // its own thread stores)
      const Q4 qm = stepped_knot(a, src, i + 1);
      const double q2[8] = {qn.x, qn.y, qn.z, qn.w, qm.x, qm.y, qm.z, qm.w};
      KnotPair kp;
      make_knot_pair(q2, 0, kp);
      a.xc.tab[i] = kp;
    }
    if (a.count_camera && a.active[6 * i]) {
      xn += q.x * q.x + q.y * q.y + q.z * q.z + q.w * q.w;
      sn += (q.x - qn.x) * (q.x - qn.x) + (q.y - qn.y) * (q.y - qn.y) + (q.z - qn.z) * (q.z - qn.z) + (q.w - qn.w) * (q.w - qn.w);
    }
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const double p = a.x.p[kPStride * i + c];
      const double pn = p + a.alpha * src(6 * i + 3 + c);
      a.xc.p[kPStride * i + c] = pn;
      if (a.count_camera && a.active[6 * i + 3 + c]) { xn += p * p; sn += (p - pn) * (p - pn); }
    }
    a.xc.p[kPStride * i + 3] = 0.0;
  } else if (i < nK + 6 * nB) {
    const int b = i - nK;
    const double v = a.x.bias[b];
    const double vn = v + a.alpha * src(a.dims.idx_bias0 + b);
    a.xc.bias[b] = vn;
    if (a.count_camera && a.active[a.dims.idx_bias0 + b]) { xn += v * v; sn += (v - vn) * (v - vn); }
  } else if (i == nK + 6 * nB) {
    const double v = *a.x.ld;
    double vn = v + a.alpha * src(a.dims.idx_ld);
    if (a.clamp_ld) vn = fmin(fmax(vn, a.ld_lower), a.ld_upper);
    *a.xc.ld = vn;
    a.scal->ld_value = vn;
    if (a.count_camera && a.active[a.dims.idx_ld]) { xn += v * v; sn += (v - vn) * (v - vn); }
  } else if (i < nK + 6 * nB + 1 + nL) {
    const int l = i - (nK + 6 * nB + 1);
    const double v = a.x.rho[l];
    const double vn = v + a.alpha * a.dl[l];
    a.xc.rho[l] = vn;
    if (a.active[a.dims.np + l]) { xn += v * v; sn += (v - vn) * (v - vn); }
  }
  xn = warp_sum_d(xn); sn = warp_sum_d(sn);
  if ((threadIdx.x & 31) == 0) { red[0][threadIdx.x >> 5] = xn; red[1][threadIdx.x >> 5] = sn; }
  __syncthreads();
  det_ticket_wait(a.det_ticket ? a.det_ticket + 1 : nullptr, blockIdx.x);
  if (threadIdx.x == 0) {
    double x = 0, s = 0;
    for (int w = 0; w < 8; ++w) { x += red[0][w]; s += red[1][w]; }
    if (x != 0.0) atomicAdd(&a.scal->x_norm2, x);
    if (s != 0.0) atomicAdd(&a.scal->step_norm2, s);
  }
  det_ticket_done(a.det_ticket ? a.det_ticket + 1 : nullptr, blockIdx.x);
}

__global__ void __launch_bounds__(256) apply_step_kernel(ApplyLaunch a) {
  apply_step_block(a, StepSource{a.dc, nullptr, nullptr, nullptr}, blockIdx.x, true);
}

int launch_apply_step(const ApplyLaunch& a, cudaStream_t s, bool reset) {
  const int n = a.dims.nK + 6 * a.dims.nB + 1 + a.dims.nL;
  if (reset) cudaMemsetAsync(&a.scal->step_norm2, 0, 2 * sizeof(double), s);  // step_norm2, x_norm2 are adjacent
  apply_step_kernel<<<(n + 255) / 256, 256, 0, s>>>(a);  // also writes the candidate's knot-pair table (K0)
  return 1;
}

// K6 in ONE launch for the full step (alpha = 1): blocks [0, ncb) camera rows (dc, g'd, d'Hd), [ncb, ncb + nlb)
// landmarks (back-substitution + the candidate's inverse depths + their norms), the rest the candidate's knots,
// biases, line delay and knot-pair table computed straight from y.
__global__ void __launch_bounds__(256) step_apply_kernel(LinearLaunch a, ApplyLaunch ap, int ncb, int nlb) {
  extern __shared__ double step_dsh[];  // [np]
  const int b = blockIdx.x;
  pdl_wait();
  pdl_launch_dependents();
  if (b < ncb) camera_step_block(a, b, step_dsh);
  else if (b < ncb + nlb) landmark_step_block(a, b - ncb, &ap);
  else apply_step_block(ap, StepSource{nullptr, a.y, a.sc, a.cmask}, b - ncb - nlb, false);
}

int launch_step_and_apply(const LinearLaunch& a, const ApplyLaunch& ap, cudaStream_t s) {
  const int ncb = (a.dims.np + 7) / 8, nlb = (a.dims.nL + 7) / 8;
  const int nab = (a.dims.nK + 6 * a.dims.nB + 1 + 255) / 256;
  launch_chained(a.pdl, step_apply_kernel, dim3(ncb + nlb + nab), dim3(256), size_t(a.dims.np) * sizeof(double), s, a, ap,
                 ncb, nlb);
  return 1;
}

// ------------------------------------------------------------------------------------------------
// TrajectoryManager::double2vector (trajectory_manager.cpp:485-516) + R2ypr / ypr2R (eigen_utils.hpp:114-150)
__device__ void r2ypr_deg(const M3& R, double ypr[3]) {
  const double nx = R.m[0], ny = R.m[3], nz = R.m[6];
  const double ox = R.m[1], oy = R.m[4];
  const double ax = R.m[2], ay = R.m[5];
  const double y = atan2(ny, nx);
  const double p = atan2(-nz, nx * cos(y) + ny * sin(y));
  const double r = atan2(ax * sin(y) - ay * cos(y), -ox * sin(y) + oy * cos(y));
  const double k = 180.0 / 3.14159265358979323846;
  ypr[0] = y * k; ypr[1] = p * k; ypr[2] = r * k;
}

__device__ __forceinline__ void gauge_realign_apply(StatePtrs st, int nK, int min_idx, const double* R0t0) {
  __shared__ double T[16];  // qd (4), tran_diff (3)
  if (threadIdx.x == 0) {
    M3 R0;
    for (int e = 0; e < 9; ++e) R0.m[e] = R0t0[e];
    const V3 t0 = V3{R0t0[9], R0t0[10], R0t0[11]};
    const M3 R00 = so3_matrix(load_q(st.q, min_idx));
    const V3 t00 = load_p<kPStride>(st.p, min_idx);
    double e0[3], e00[3];
    r2ypr_deg(R0, e0);
    r2ypr_deg(R00, e00);
    const double y = (e0[0] - e00[0]) / 180.0 * 3.14159265358979323846;
    M3 rd = m3_identity();
    rd.m[0] = cos(y); rd.m[1] = -sin(y); rd.m[3] = sin(y); rd.m[4] = cos(y);
    if (fabs(fabs(e0[1]) - 90.0) < 1.0 || fabs(fabs(e00[1]) - 90.0) < 1.0) rd = m3_mul_bt(R0, R00);
    const V3 td = t0 - m3_vec(rd, t00);
    const Q4 qd = quat_from_matrix(rd);
    T[0] = qd.x; T[1] = qd.y; T[2] = qd.z; T[3] = qd.w; T[4] = td.x; T[5] = td.y; T[6] = td.z;
  }
  __syncthreads();
  const Q4 qd = Q4{T[0], T[1], T[2], T[3]};
  const V3 td = V3{T[4], T[5], T[6]};
  for (int i = min_idx + threadIdx.x; i < nK; i += blockDim.x) {
    const Q4 qn = so3_mul(qd, load_q(st.q, i));
    const V3 pn = so3_rotate(qd, load_p<kPStride>(st.p, i)) + td;
    st.q[4 * i] = qn.x; st.q[4 * i + 1] = qn.y; st.q[4 * i + 2] = qn.z; st.q[4 * i + 3] = qn.w;
    st.p[kPStride * i] = pn.x; st.p[kPStride * i + 1] = pn.y; st.p[kPStride * i + 2] = pn.z;
  }
}

__global__ void gauge_realign_kernel(StatePtrs st, int nK, int min_idx, const double* R0t0) {
  gauge_realign_apply(st, nK, min_idx, R0t0);
}

// numpy's cross(a, b) component c: each product rounded, then the difference (no contraction)
__device__ __forceinline__ double np_cross(const double* a, const double* b, int c) {
  const int i = (c + 1) % 3, j = (c + 2) % 3;
  return __dsub_rn(__dmul_rn(a[i], b[j]), __dmul_rn(a[j], b[i]));
}

// The realignment of the odometry cycle: R0 / t0 formed on the device from the snapshot q (4), p (3) of the knot taken
// before the solve, with the operations of the host's R0 = qrot(q, I).T (synthetic.py, numpy): column j of R is
// v + w uv + qv x uv, uv = 2 (qv x v), v = e_j.  R0t0_out receives R0 (row-major) and t0 (12 doubles).
__global__ void gauge_realign_snapshot_kernel(StatePtrs st, int nK, int min_idx, const double* snap, double* R0t0_out) {
  __shared__ double R0t0[12];
  if (threadIdx.x == 0) {
    const double qv[3] = {snap[0], snap[1], snap[2]}, w = snap[3];
    for (int j = 0; j < 3; ++j) {
      const double v[3] = {j == 0 ? 1.0 : 0.0, j == 1 ? 1.0 : 0.0, j == 2 ? 1.0 : 0.0};
      double uv[3];
      for (int c = 0; c < 3; ++c) uv[c] = __dmul_rn(2.0, np_cross(qv, v, c));
      for (int c = 0; c < 3; ++c) R0t0[3 * c + j] = __dadd_rn(__dadd_rn(v[c], __dmul_rn(w, uv[c])), np_cross(qv, uv, c));
    }
    for (int c = 0; c < 3; ++c) R0t0[9 + c] = snap[4 + c];
    for (int k = 0; k < 12; ++k) R0t0_out[k] = R0t0[k];
  }
  __syncthreads();
  gauge_realign_apply(st, nK, min_idx, R0t0);
}

int launch_gauge_realign(const StatePtrs& st, int nK, int min_idx, const double* R0_t0_dev, cudaStream_t s) {
  gauge_realign_kernel<<<1, 256, 0, s>>>(st, nK, min_idx, R0_t0_dev);
  return 1 + launch_knot_table(st, nK, s);
}

int launch_gauge_realign_snapshot(const StatePtrs& st, int nK, int min_idx, const double* snap_dev, double* R0_t0_out,
                                  cudaStream_t s) {
  gauge_realign_snapshot_kernel<<<1, 256, 0, s>>>(st, nK, min_idx, snap_dev, R0_t0_out);
  return 1 + launch_knot_table(st, nK, s);
}

}  // namespace ctvio
