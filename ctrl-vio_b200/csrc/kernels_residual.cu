// Residual / Jacobian / normal-equation kernels of the CUDA engine (sm_90a, fp64).
//
//   knot_table_kernel   K0  per linearisation point: d_k, |d_k|, Jr^-1(d_k) for every knot pair
//   visual_kernel       K1  replaces ImageFeatureDelayFactor::Evaluate (image_feature_factor.h:63-269)
//                           + loss corrector + Ceres' J'J / J'r build for all image factors
//   imu_kernel          K2  replaces IMUFactor::Evaluate (trajectory_value_factor.h:141-248)
//   small_factors_kernel K3 replaces BiasFactor::Evaluate (:45-99) and MarginalizationFactor::Evaluate
//                           (marginalization_factor.cpp:326-373)
//
// K1 design (GPU-first, not a translation of the reference's per-factor virtual calls):
//   * observations are pre-sorted by frame-pair group = (first knot of the padded anchor window,
//     first knot of the padded observation window); one CTA owns a chunk of one group, so every
//     Jacobian row of the chunk lives in the same 61-dim local space
//     [anchor window 5 knots x 6 | observation window 5 knots x 6 | line delay] (+ residual column);
//   * the 10 active control knots and their knot-pair table entries are staged in shared memory
//     by TMA bulk copies (cp.async.bulk + mbarrier) — 6 copies, ~2 KB per CTA;
//   * a LANE PAIR evaluates one observation: even lane = anchor pose, odd lane = observation pose
//     (eval_side), 18 doubles exchanged by warp shuffles, each lane then chain-rules its own 4 knots;
//   * Jacobian rows never go to HBM: they are written to a shared-memory tile (128 obs x 2 rows x 64)
//     and reduced by a SYRK on the fp64 tensor cores (syrk_round) into a shared accumulator that
//     is flushed once per CTA with fp64 atomics into the upper-triangular camera block A and g;
//   * landmark Schur pieces (h_l, g_l, W_l) are reduced with fp64 RED atomics into the compact
//     per-landmark rows.
// Algorithmic HBM traffic per observation: 64 B record + 8 B inverse-depth gather.
#include <cstdio>

#include "kernels.h"

namespace ctvio {

// ------------------------------------------------------------------------------------------------
// small PTX helpers: shared-memory addresses, mbarrier, TMA bulk copy

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void tma_bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smem_u32(dst)),
               "l"(src), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t phase) {
  uint32_t ok;
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
      "selp.u32 %0, 1, 0, p;\n"
      "}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(phase)
      : "memory");
  return ok != 0;
}

// ------------------------------------------------------------------------------------------------
// K0

__global__ void knot_table_kernel(StatePtrs st, int nK) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= nK - 1) return;
  KnotPair kp;
  make_knot_pair(st.q, k, kp);
  st.tab[k] = kp;
}

int launch_knot_table(const StatePtrs& st, int nK, cudaStream_t s) {
  if (nK < 2) return 0;
  knot_table_kernel<<<(nK - 1 + 127) / 128, 128, 0, s>>>(st, nK);
  return 1;
}

// ------------------------------------------------------------------------------------------------
// K1

struct VisArgs {
  ImageObsPtrs obs;
  const VisualItem* items;
  StatePtrs st;
  NormalEqPtrs ne;
  LandmarkLayout lm;
  ProblemDims dims;
  SplineParams sp;
  RigParams rig;
  double cauchy;
  const uint8_t* cmask;
  LmScalars* scal;
  int* det_ticket;
};

struct __align__(128) VisStatic {
  KnotPair tab[2][4];            // 1024 B
  double q[2][kWinKnots][4];     // 320 B
  double p[2][kWinKnots][4];     // 320 B
  double cost_part[8];
  unsigned long long bar;
  int err;
};

// upper-triangular tiles of the 8x8 tile grid over the 64 local dims
__constant__ uint8_t c_tile_i[36] = {0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 1, 1, 1, 2, 2, 2,
                                     2, 2, 2, 3, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 6, 6, 7};
__constant__ uint8_t c_tile_j[36] = {0, 1, 2, 3, 4, 5, 6, 7, 1, 2, 3, 4, 5, 6, 7, 2, 3, 4,
                                     5, 6, 7, 3, 4, 5, 6, 7, 4, 5, 6, 7, 5, 6, 7, 6, 7, 7};

#ifdef CTVIO_CHOL_TIMING
__device__ long long g_vis_clk[8];
__device__ long long g_imu_clk[8];
#define VCLK(i) do { if (blockIdx.x == 0 && threadIdx.x == 0) g_vis_clk[(i)] = clock64(); } while (0)
#define ICLK(i) do { if (blockIdx.x == 0 && threadIdx.x == 0) g_imu_clk[(i)] = clock64(); } while (0)
extern "C" int ctvio_debug_vis_clk(long long* out) {
  return cudaMemcpyFromSymbol(out, g_vis_clk, sizeof(g_vis_clk)) == cudaSuccess ? 0 : -1;
}
extern "C" int ctvio_debug_imu_clk(long long* out) {
  return cudaMemcpyFromSymbol(out, g_imu_clk, sizeof(g_imu_clk)) == cudaSuccess ? 0 : -1;
}
#else
#define VCLK(i)
#define ICLK(i)
#endif

size_t visual_smem_bytes() {
  return size_t(kVisObsPerRound) * kObsStride * sizeof(double) + size_t(36) * 64 * sizeof(double);
}

// SYRK of one round's Jacobian rows into the CTA accumulator (upper 8x8 tiles of the 64 local dims) on the fp64
// tensor cores (m8n8k4; K = Jacobian rows).  The 36 upper tiles are grouped into 16x16 blocks, one or two per warp
// (warps 0..5: the six off-diagonal blocks, warps 6, 7: two diagonal blocks each), so that every tile has ONE owner
// warp over all rows: no cross-warp merge, the partial sums of earlier rounds are simply reloaded from accs.
// Rows of inactive observation slots are zero (written by the evaluation phase), so K runs in whole 4-row steps.
// The two kinds of warp are two instantiations (every DMMA unconditional, see DESIGN §4 on WARPSYNC).
template <bool DIAG>
__device__ __noinline__ void syrk_round_warp(const double* Jt, double* accs, int nround, int warp, int lane) {
  constexpr int NB = DIAG ? 2 : 1;
  const int g = lane >> 2, q = lane & 3;
  int bi[NB], bj[NB];
  if constexpr (DIAG) {
    bi[0] = bj[0] = 2 * (warp - 6);
    bi[1] = bj[1] = 2 * (warp - 6) + 1;
  } else {
    bi[0] = warp < 3 ? 0 : (warp < 5 ? 1 : 2);
    bj[0] = warp < 3 ? warp + 1 : (warp < 5 ? warp - 1 : 3);
  }
  double acc[NB][2][2][2];
#pragma unroll
  for (int b = 0; b < NB; ++b)
#pragma unroll
    for (int mi = 0; mi < 2; ++mi)
#pragma unroll
      for (int nj = 0; nj < 2; ++nj) {
        if (DIAG && mi == 1 && nj == 0) continue;  // strictly lower tile of a diagonal block
        const int ti = 2 * bi[b] + mi, tj = 2 * bj[b] + nj;
        const double2 v = *reinterpret_cast<const double2*>(accs + (ti * 8 - ti * (ti - 1) / 2 + (tj - ti)) * 64 + g * 8 + 2 * q);
        acc[b][mi][nj][0] = v.x; acc[b][mi][nj][1] = v.y;
      }
  const int nsteps = (2 * nround + 3) >> 2;
#pragma unroll 2
  for (int st = 0; st < nsteps; ++st) {
    const int row = 4 * st + q;
    const double* rp = Jt + size_t(row >> 1) * kObsStride + (row & 1) * kRowStride + g;
#pragma unroll
    for (int b = 0; b < NB; ++b) {
      double av[2], bv[2];
#pragma unroll
      for (int m = 0; m < 2; ++m) {
        av[m] = rp[16 * bi[b] + 8 * m];
        bv[m] = DIAG ? av[m] : rp[16 * bj[b] + 8 * m];
      }
#pragma unroll
      for (int mi = 0; mi < 2; ++mi)
#pragma unroll
        for (int nj = 0; nj < 2; ++nj) {
          if (DIAG && mi == 1 && nj == 0) continue;
          asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};"
                       : "+d"(acc[b][mi][nj][0]), "+d"(acc[b][mi][nj][1])
                       : "d"(av[mi]), "d"(bv[nj]));
        }
    }
  }
#pragma unroll
  for (int b = 0; b < NB; ++b)
#pragma unroll
    for (int mi = 0; mi < 2; ++mi)
#pragma unroll
      for (int nj = 0; nj < 2; ++nj) {
        if (DIAG && mi == 1 && nj == 0) continue;
        const int ti = 2 * bi[b] + mi, tj = 2 * bj[b] + nj;
        *reinterpret_cast<double2*>(accs + (ti * 8 - ti * (ti - 1) / 2 + (tj - ti)) * 64 + g * 8 + 2 * q) =
            make_double2(acc[b][mi][nj][0], acc[b][mi][nj][1]);
      }
}

__device__ __forceinline__ void syrk_round(const double* Jt, double* accs, int nround, int tid) {
  const int warp = tid >> 5, lane = tid & 31;
  if (warp < 6) syrk_round_warp<false>(Jt, accs, nround, warp, lane);
  else syrk_round_warp<true>(Jt, accs, nround, warp, lane);
  __syncthreads();
}

// deterministic mode, one round of visual_kernel<true>: the landmark pieces (hl, gl, wld, W) of the round's observations
// from the finished rows of the shared tile.  The observations of one landmark are adjacent in an item (sorted by
// landmark), and several of them can share a round (target frames whose knot windows coincide); the lane of the first
// one adds them all in slot order, so that no two lanes of the CTA add to the same entry at the same time.  The two knot
// windows of an observation may overlap (same global dims): anchor side first, then the other one.  (Out of line: it
// runs in deterministic mode only and must not cost the fast path registers.)
__device__ __noinline__ void det_landmark_round(const VisArgs& a, const double* Jt, int base) {
  // (the lane's slot and side and the item are re-derived here: nothing extra stays live across the call)
  const VisualItem item = a.items[blockIdx.x];
  const int o0 = item.start + base, nround = min(kVisObsPerRound, item.count - base);
  const int ol = threadIdx.x >> 1, side = threadIdx.x & 1, wk0 = side ? item.wj0 : item.wi0;
  for (int ph = 0; ph < 2; ++ph) {
    if (ol < nround && side == ph) {
      const int l = a.obs.meta[o0 + ol].z;
      if (ol == 0 || a.obs.meta[o0 + ol - 1].z != l) {
        double* Wl = a.ne.W + (a.lm.woff[l] - a.lm.lo[l]) + 6 * wk0;
        const int cb = side * 30;
        for (int o = ol; o < nround && a.obs.meta[o0 + o].z == l; ++o) {
          const double* r0 = Jt + size_t(o) * kObsStride;
          const double* r1 = r0 + kRowStride;
          const double j0 = r0[kColRho], j1 = r1[kColRho];
          if (j0 == 0.0 && j1 == 0.0) continue;  // invalid observation (its rows are zero): nothing to add
          if (side == 0) {
            atomicAdd(a.ne.hl + l, j0 * j0 + j1 * j1);
            atomicAdd(a.ne.gl + l, j0 * r0[kColR] + j1 * r1[kColR]);
          } else {
            atomicAdd(a.ne.wld + l, r0[kColLd] * j0 + r1[kColLd] * j1);
          }
          for (int c = 0; c < 30; ++c) {
            const double v = r0[cb + c] * j0 + r1[cb + c] * j1;
            if (v != 0.0) atomicAdd(Wl + c, v);
          }
        }
      }
    }
    __threadfence();
    __syncthreads();
  }
}

template <bool FULL>
__global__ void __launch_bounds__(kVisThreads, 1) visual_kernel(const __grid_constant__ VisArgs a) {
  extern __shared__ __align__(128) unsigned char dyn_smem[];
  double* Jt = reinterpret_cast<double*>(dyn_smem);                 // [128 obs][2 rows][64 cols], padded strides
  double* accs = Jt + size_t(kVisObsPerRound) * kObsStride;         // [36][64]
  __shared__ VisStatic sm;

  const int tid = threadIdx.x;
  const int lane = tid & 31, warp = tid >> 5;
  const VisualItem item = a.items[blockIdx.x];
  const int nK = a.dims.nK;
  VCLK(0);

  // ---- stage the 10 active knots + 8 knot-pair entries (TMA bulk copies, one mbarrier) ----
  const int w0[2] = {item.wi0, item.wj0};
  if (tid == 0) {
    sm.err = 0;
    mbar_init(reinterpret_cast<uint64_t*>(&sm.bar), 1);
    fence_mbar_init();
  }
  __syncthreads();
  if (tid == 0) {
    uint32_t bytes = 0;
#pragma unroll
    for (int sd = 0; sd < 2; ++sd) {
      const int nk = min(kWinKnots, nK - w0[sd]);
      const int npair = min(4, nK - 1 - w0[sd]);
      bytes += uint32_t(nk) * 64u + uint32_t(npair) * uint32_t(sizeof(KnotPair));
    }
    mbar_expect_tx(reinterpret_cast<uint64_t*>(&sm.bar), bytes);
#pragma unroll
    for (int sd = 0; sd < 2; ++sd) {
      const int nk = min(kWinKnots, nK - w0[sd]);
      const int npair = min(4, nK - 1 - w0[sd]);
      tma_bulk_g2s(&sm.q[sd][0][0], a.st.q + 4 * w0[sd], uint32_t(nk) * 32u, reinterpret_cast<uint64_t*>(&sm.bar));
      tma_bulk_g2s(&sm.p[sd][0][0], a.st.p + 4 * w0[sd], uint32_t(nk) * 32u, reinterpret_cast<uint64_t*>(&sm.bar));
      tma_bulk_g2s(&sm.tab[sd][0], a.st.tab + w0[sd], uint32_t(npair) * uint32_t(sizeof(KnotPair)),
                   reinterpret_cast<uint64_t*>(&sm.bar));
    }
  }
  if (FULL)
    for (int i = tid; i < 36 * 64; i += kVisThreads) accs[i] = 0.0;
  while (!mbar_try_wait(reinterpret_cast<uint64_t*>(&sm.bar), 0)) {
  }
  __syncthreads();

  const double ld = *a.st.ld;
  const int64_t ld_ns = int64_t(ld * 1e9);  // image_feature_factor.h:72 (truncation)
  const int side = tid & 1;
  double cost_local = 0.0;
  VCLK(1);

  for (int base = 0; base < item.count; base += kVisObsPerRound) {
    const int nround = min(kVisObsPerRound, item.count - base);
    const int ol = tid >> 1;  // observation slot of this lane pair
    const bool active = ol < nround;
    double* row0 = Jt + size_t(ol) * kObsStride;
    double* row1 = row0 + kRowStride;
    bool valid = false;
    const unsigned m_act = __ballot_sync(0xffffffffu, active);  // lane pairs are active together
    if (active) {
      const int oi = item.start + base + ol;
      const longlong2 tt = a.obs.t[oi];
      const double2 pi = a.obs.pi[oi];
      const double2 pj = a.obs.pj[oi];
      const int4 meta = a.obs.meta[oi];
      const double rho = a.st.rho[meta.z];
      // the landmark's coupling-row base (two dependent L2 loads): issued here so that the pose evaluation hides them
      const int64_t w_base = FULL ? a.lm.woff[meta.z] - a.lm.lo[meta.z] : 0;
      const int64_t t_eval = side == 0 ? tt.x + int64_t(meta.x) * ld_ns : tt.y + int64_t(meta.y) * ld_ns;
      int32_t s;
      double u;
      bool ok = spline_index(a.sp, t_eval, s, u);
      const int slot = s - w0[side];
      ok = ok && (slot == 0 || slot == 1);
      const bool ok_both = __shfl_xor_sync(m_act, ok ? 1 : 0, 1) && ok;
      const unsigned m_ok = __ballot_sync(m_act, ok_both);  // lanes that run the exchange below
      valid = ok_both;
      if (!ok_both) {
        atomicOr(&sm.err, 1);
      } else {
        PoseStage ev;
        pose_stage<FULL, kPStride>(a.sp, &sm.q[side][0][0], &sm.p[side][0][0], sm.tab[side], slot, u, ev);
        // exchange pose (and velocities) with the partner lane
        M3 Ro;
        V3 po, omo, vo;
#pragma unroll
        for (int e = 0; e < 9; ++e) Ro.m[e] = __shfl_xor_sync(m_ok, ev.R.m[e], 1);
        po = V3{__shfl_xor_sync(m_ok, ev.p.x, 1), __shfl_xor_sync(m_ok, ev.p.y, 1), __shfl_xor_sync(m_ok, ev.p.z, 1)};
        if (FULL) {
          omo = V3{__shfl_xor_sync(m_ok, ev.omega.x, 1), __shfl_xor_sync(m_ok, ev.omega.y, 1),
                   __shfl_xor_sync(m_ok, ev.omega.z, 1)};
          vo = V3{__shfl_xor_sync(m_ok, ev.vel.x, 1), __shfl_xor_sync(m_ok, ev.vel.y, 1),
                  __shfl_xor_sync(m_ok, ev.vel.z, 1)};
        }
        const M3& R_i = side == 0 ? ev.R : Ro;
        const M3& R_j = side == 0 ? Ro : ev.R;
        const V3 p_i = side == 0 ? ev.p : po;
        const V3 p_j = side == 0 ? po : ev.p;
        ImageCommon cm;
        const double pixy[2] = {pi.x, pi.y}, pjxy[2] = {pj.x, pj.y};
        image_common(a.rig, pixy, pjxy, rho, R_i, p_i, R_j, p_j, a.cauchy, cm);
        if (side == 0) cost_local += cm.cost;
        if (FULL) {
          double jrho[2], lhs[6];
          image_jrho(a.rig, cm, R_i, rho, jrho);
          image_side_lhs(side, cm, ev.R, lhs);
          // one knot at a time: chain rule -> constant masking -> the lane's local columns of the shared tile
          // (5 knot slots x 6 per side) -> landmark coupling W_l += J_c' J_rho (fp64 RED), so that no 2x24
          // block array stays live in registers
          const int cb = side * 30;
          const int gk0 = w0[side];
          const int l = meta.z;
          double* Wl = a.ne.W + w_base;
          {
            const int unused = cb + (slot == 0 ? 4 : 0) * 6;
#pragma unroll
            for (int c = 0; c < 6; ++c) { row0[unused + c] = 0.0; row1[unused + c] = 0.0; }
          }
          const double sgn = side == 0 ? 1.0 : -1.0;
          jacobian_stage(sm.tab[side], ev, [&](int k, const M3& Jk) {
            double rk[6];
            mul23_33(lhs, Jk, rk);
            const int gd = 6 * (gk0 + slot + k);
            const int col = cb + (slot + k) * 6;
            const double ck = sgn * ev.c[k];
#pragma unroll
            for (int c = 0; c < 3; ++c) {
              const bool mr = a.cmask[gd + c] != 0, mp = a.cmask[gd + 3 + c] != 0;
              const double r0v = mr ? 0.0 : rk[c], r1v = mr ? 0.0 : rk[3 + c];
              const double p0v = mp ? 0.0 : ck * cm.JvR[c], p1v = mp ? 0.0 : ck * cm.JvR[3 + c];
              row0[col + c] = r0v; row1[col + c] = r1v;
              row0[col + 3 + c] = p0v; row1[col + 3 + c] = p1v;
              if (!a.det_ticket) {  // (deterministic mode: recomputed from the shared tile inside the ordered flush)
                if (!mr) atomicAdd(Wl + gd + c, r0v * jrho[0] + r1v * jrho[1]);
                if (!mp) atomicAdd(Wl + gd + 3 + c, p0v * jrho[0] + p1v * jrho[1]);
              }
            }
          });
          if (side == 0) {
            row0[kColR] = cm.r[0]; row1[kColR] = cm.r[1];
            row0[kColRho] = jrho[0]; row1[kColRho] = jrho[1];
          } else {
            double jld[2];
            image_jld(a.rig, cm, meta.x, meta.y, R_i, omo, vo, R_j, ev.omega, ev.vel, jld);
            const bool ld_const = a.cmask[a.dims.idx_ld] != 0;
            row0[kColLd] = ld_const ? 0.0 : jld[0];
            row1[kColLd] = ld_const ? 0.0 : jld[1];
            row0[63] = 0.0; row1[63] = 0.0;
          }
          if (!a.det_ticket) {
            if (side == 0) {
              atomicAdd(a.ne.hl + l, jrho[0] * jrho[0] + jrho[1] * jrho[1]);
              atomicAdd(a.ne.gl + l, jrho[0] * cm.r[0] + jrho[1] * cm.r[1]);
            } else {
              atomicAdd(a.ne.wld + l, row0[kColLd] * jrho[0] + row1[kColLd] * jrho[1]);
            }
          }
        }
      }
    }
    if (FULL) {
      if (!valid && ol < kVisObsPerRound) {
        // inactive / invalid observation: its half of the two rows is zero
        const int cb = side * 30;
        for (int c = 0; c < 30; ++c) { row0[cb + c] = 0.0; row1[cb + c] = 0.0; }
        if (side == 0) { row0[kColR] = row1[kColR] = 0.0; row0[kColRho] = row1[kColRho] = 0.0; }
        else { row0[kColLd] = row1[kColLd] = 0.0; row0[63] = row1[63] = 0.0; }
      }
      VCLK(2);
      __syncthreads();
      VCLK(3);
      if (a.det_ticket) {
        // deterministic mode: the landmark pieces of this round's observations from the finished rows of the shared tile
        // (same products as the per-lane atomics of the fast path), issued in the CTA's turn
        det_ticket_wait(a.det_ticket, blockIdx.x * 1024 + base / kVisObsPerRound);
        det_landmark_round(a, Jt, base);
        det_ticket_done(a.det_ticket, blockIdx.x * 1024 + base / kVisObsPerRound);
      }
      syrk_round(Jt, accs, nround, tid);
      VCLK(4);
    }
  }

  // ---- cost + flush ----
  const int n_rounds = (item.count + kVisObsPerRound - 1) / kVisObsPerRound;
  det_ticket_wait(a.det_ticket, blockIdx.x * 1024 + (FULL ? n_rounds : 0));
  cost_local = warp_sum_d(cost_local);
  if (lane == 0) sm.cost_part[warp] = cost_local;
  __syncthreads();
  if (tid == 0) {
    double c = 0;
#pragma unroll
    for (int w = 0; w < kVisThreads / 32; ++w) c += sm.cost_part[w];
    atomicAdd(a.ne.cost, c);
    if (sm.err) atomicOr(&a.scal->error_flags, 1);
  }
  if (FULL) {
    const int np = a.dims.np;
    // Fast mode: one pass.  Deterministic mode: when the two knot windows overlap, different LOCAL entries of this CTA land
    // on the same global entry; the flush then runs in 11 classes (side of the row dim x side of the column dim, the
    // mixed class split by the order of the global indices) inside each of which the local -> global map is injective,
    // with a fence + barrier between classes, so the order of the additions to every address is fixed.
    const int n_class = a.det_ticket ? 11 : 1;
    for (int cls = 0; cls < n_class; ++cls) {
      for (int idx = tid; idx < 36 * 64; idx += kVisThreads) {
        const double val = accs[idx];
        if (val == 0.0) continue;
        const int tile = idx >> 6, e = idx & 63;
        const int la = c_tile_i[tile] * 8 + (e >> 3), lb = c_tile_j[tile] * 8 + (e & 7);
        if (la > lb || lb > kColR || la >= kColR) continue;
        const int sa = la < 30 ? 0 : (la < 60 ? 1 : 2);
        const int ga = sa == 0 ? 6 * item.wi0 + la : (sa == 1 ? 6 * item.wj0 + (la - 30) : a.dims.idx_ld);
        if (lb == kColR) {
          if (n_class > 1 && cls != 8 + sa) continue;
          atomicAdd(a.ne.gc + ga, val);
          continue;
        }
        const int sb = lb < 30 ? 0 : (lb < 60 ? 1 : 2);
        const int gb = sb == 0 ? 6 * item.wi0 + lb : (sb == 1 ? 6 * item.wj0 + (lb - 30) : a.dims.idx_ld);
        if (n_class > 1) {
          int c;
          if (sb == 2) c = 5 + sa;                                  // (anchor | obs | ld) x ld
          else if (sa == sb) c = sa == 0 ? 0 : 4;                   // anchor x anchor, obs x obs
          else c = ga < gb ? 1 : (ga > gb ? 2 : 3);                 // anchor x obs by the order of the global dims
          if (c != cls) continue;
        }
        const double v = (la != lb && ga == gb) ? 2.0 * val : val;
        const int g0 = min(ga, gb), g1 = max(ga, gb);
        atomicAdd(a.ne.A + size_t(g0) * np + g1, v);
      }
      if (n_class > 1) {
        __threadfence();
        __syncthreads();
      }
    }
  }
  // the next CTA's first ticket value: (blockIdx.x + 1) * 1024
  if (a.det_ticket) {
    __threadfence();
    __syncthreads();
    if (tid == 0) asm volatile("st.release.gpu.global.s32 [%0], %1;" ::"l"(a.det_ticket), "r"((int(blockIdx.x) + 1) * 1024) : "memory");
  }
  VCLK(5);
}

int launch_visual(const VisualLaunch& l, bool full, cudaStream_t s) {
  if (l.n_items <= 0) return 0;
  VisArgs a{l.obs, l.items, l.st, l.ne, l.lm, l.dims, l.sp, l.rig, l.cauchy, l.cmask, l.scal, l.det_ticket};
  static PerDeviceOnce once;
  if (once.first()) {
    cudaFuncSetAttribute(visual_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, int(visual_smem_bytes()));
    cudaFuncSetAttribute(visual_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, int(visual_smem_bytes()));
  }
  if (full) visual_kernel<true><<<l.n_items, kVisThreads, visual_smem_bytes(), s>>>(a);
  else visual_kernel<false><<<l.n_items, kVisThreads, 0, s>>>(a);
  return 1;
}

// ------------------------------------------------------------------------------------------------
// K2: IMU factors.  One CTA of four warps per (start knot, bias node) run of samples (<= 32).  Lane l of every warp
// evaluates sample l up to its residual (imu_stage), then warp w writes a quarter of the sample's 6 x 31 Jacobian rows
// (24 knot dims | 6 bias dims | residual): the gyro (w = 0, 1) or accel (w = 2, 3) rows of the knots 2 (w & 1) and
// 2 (w & 1) + 1, warps 1 and 3 also the bias columns and the residual.  The rows go column-major to shared memory and
// J'J is formed on the fp64 tensor cores (m8n8k4, K = Jacobian rows): each of the 10 upper 8x8 tiles of the 32 local
// dims has one owner warp over all rows and is flushed from its fragments, one fp64 atomic per non-zero entry per CTA.

struct ImuArgs {
  ImuObsPtrs obs;
  const ImuItem* items;
  StatePtrs st;
  NormalEqPtrs ne;
  ProblemDims dims;
  SplineParams sp;
  RigParams rig;
  const uint8_t* cmask;
  LmScalars* scal;
  int* det_ticket;
};

constexpr int kImuThreads = 128;
constexpr int kImuCols = 32;          // 24 knot dims + 6 bias dims + residual + zero pad
constexpr int kImuColStride = 196;    // doubles per column: 6 x 32 rows + 4; = 4 mod 16, so the fragment loads of a
                                      // half-warp (4 columns x 4 rows) hit 16 different banks
static_assert(kImuColStride >= 6 * kImuMaxPerItem && kImuColStride % 16 == 4, "K2 shared column stride");

// Tile t of warp w as 4 ti + tj, chosen so that a warp loads 2 or 3 of the 4 column tiles per 4-row step:
// warp 0 (0,0) (0,1) (1,1), warp 1 (2,2) (2,3) (3,3), warp 2 (0,2) (0,3), warp 3 (1,2) (1,3)
__host__ __device__ constexpr int imu_tile(int w, int t) {
  return w == 0 ? (t == 0 ? 0 : t == 1 ? 1 : 5)
       : w == 1 ? (t == 0 ? 10 : t == 1 ? 11 : 15)
       : w == 2 ? (t == 0 ? 2 : 3)
                : (t == 0 ? 6 : 7);
}
__host__ __device__ constexpr int imu_ntiles(int w) { return w < 2 ? 3 : 2; }
__host__ __device__ constexpr bool imu_uses(int w, int c) {
  bool u = false;
  for (int t = 0; t < imu_ntiles(w); ++t) u = u || imu_tile(w, t) >> 2 == c || (imu_tile(w, t) & 3) == c;
  return u;
}

// Zero this warp's part of one sample's rows (an invalid sample, or the sample after the last one when the row count is
// not a multiple of the 4-row step)
__device__ __forceinline__ void imu_zero_part(double* J, int warp) {
  const int r0 = 3 * (warp >> 1), c0 = 12 * (warp & 1), c1 = (warp & 1) ? kImuCols : 12;
  for (int c = c0; c < c1; ++c)
#pragma unroll
    for (int r = 0; r < 3; ++r) J[c * kImuColStride + r0 + r] = 0.0;
}

template <bool ACCEL, int H>
__device__ __forceinline__ void imu_write_part(const ImuArgs& a, const ImuStage& st, int s, int node, double* J) {
  constexpr int r0 = ACCEL ? 3 : 0;
  imu_jacobian_half<ACCEL, H>(a.rig, a.st.tab, s, st, [&](int k, const double rot[9], const double pos[9]) {
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const bool mr = a.cmask[6 * (s + k) + c] != 0, mp = a.cmask[6 * (s + k) + 3 + c] != 0;
#pragma unroll
      for (int r = 0; r < 3; ++r) {
        J[(k * 6 + c) * kImuColStride + r0 + r] = mr ? 0.0 : rot[3 * r + c];
        J[(k * 6 + 3 + c) * kImuColStride + r0 + r] = mp ? 0.0 : pos[3 * r + c];
      }
    }
  });
  if (H == 1) {
    const int gb0 = a.dims.idx_bias0 + 6 * node;
#pragma unroll
    for (int c = 0; c < 6; ++c) {
      const bool mb = a.cmask[gb0 + c] != 0;
#pragma unroll
      for (int r = 0; r < 3; ++r) J[(24 + c) * kImuColStride + r0 + r] = (c == r0 + r && !mb) ? a.rig.imu_info[r0 + r] : 0.0;
    }
#pragma unroll
    for (int r = 0; r < 3; ++r) {
      J[30 * kImuColStride + r0 + r] = st.r[r0 + r];
      J[31 * kImuColStride + r0 + r] = 0.0;
    }
  }
}

// This warp's J'J tiles over all rows: lane (g, q) of a step reads rows 4 st + q of the local columns 8 t + g
template <int W>
__device__ __forceinline__ void imu_syrk(const double* Js, int nsteps, int lane, double acc[3][2]) {
  const double* rp = Js + (lane >> 2) * kImuColStride + (lane & 3);
#pragma unroll
  for (int t = 0; t < 3; ++t) acc[t][0] = acc[t][1] = 0.0;
#pragma unroll 4
  for (int st = 0; st < nsteps; ++st, rp += 4) {
    double v[4];
#pragma unroll
    for (int c = 0; c < 4; ++c) v[c] = imu_uses(W, c) ? rp[8 * c * kImuColStride] : 0.0;
#pragma unroll
    for (int t = 0; t < imu_ntiles(W); ++t)
      asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};"
                   : "+d"(acc[t][0]), "+d"(acc[t][1])
                   : "d"(v[imu_tile(W, t) >> 2]), "d"(v[imu_tile(W, t) & 3]));
  }
}

// Flush of this warp's tiles: lane (g, q) holds the entries (8 ti + g, 8 tj + 2 q + {0, 1})
template <int W>
__device__ __forceinline__ void imu_flush(const ImuArgs& a, const ImuItem& item, int lane, const double acc[3][2]) {
  const int np = a.dims.np;
#pragma unroll
  for (int t = 0; t < imu_ntiles(W); ++t)
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      const double val = acc[t][e];
      const int la = 8 * (imu_tile(W, t) >> 2) + (lane >> 2), lb = 8 * (imu_tile(W, t) & 3) + 2 * (lane & 3) + e;
      if (val == 0.0 || la > lb || lb > 30 || la >= 30) continue;
      const int ga = la < 24 ? 6 * item.s + la : a.dims.idx_bias0 + 6 * item.node + (la - 24);
      if (lb == 30) {
        atomicAdd(a.ne.gc + ga, val);
        continue;
      }
      const int gb = lb < 24 ? 6 * item.s + lb : a.dims.idx_bias0 + 6 * item.node + (lb - 24);
      atomicAdd(a.ne.A + size_t(ga) * np + gb, val);  // ga <= gb: knot dims precede bias dims
    }
}

template <bool FULL>
__global__ void __launch_bounds__(kImuThreads) imu_kernel(const __grid_constant__ ImuArgs a) {
  extern __shared__ __align__(128) unsigned char dyn_smem[];
  double* Js = reinterpret_cast<double*>(dyn_smem);  // [kImuCols][kImuColStride]: column-major rows 6 l + r of sample l
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const ImuItem item = a.items[blockIdx.x];
  double cost = 0.0;
  ICLK(0);
  if ((FULL || warp == 0) && lane < item.count) {
    const int n = item.start + lane;
    const longlong2 tn = a.obs.t_node[n];
    const double2 g0 = a.obs.ga[3 * n], g1 = a.obs.ga[3 * n + 1], g2 = a.obs.ga[3 * n + 2];
    const double gyro[3] = {g0.x, g0.y, g1.x}, accel[3] = {g1.y, g2.x, g2.y};
    const int node = item.node;
    double bias[6];
#pragma unroll
    for (int c = 0; c < 6; ++c) bias[c] = a.st.bias[6 * node + c];
    int32_t s;
    double u;
    const bool ok = spline_index(a.sp, tn.x, s, u) && s == item.s;
    double* J = Js + 6 * lane;
    if (!ok) {
      if (warp == 0) atomicOr(&a.scal->error_flags, 1);
      if (FULL) imu_zero_part(J, warp);
    } else {
      ImuStage st;
      imu_stage<kPStride>(a.sp, a.rig, a.st.q, a.st.p, a.st.tab, s, u, gyro, accel, bias, st);
      cost = st.cost;
      if (FULL) {
        switch (warp) {
          case 0: imu_write_part<false, 0>(a, st, s, node, J); break;
          case 1: imu_write_part<false, 1>(a, st, s, node, J); break;
          case 2: imu_write_part<true, 0>(a, st, s, node, J); break;
          default: imu_write_part<true, 1>(a, st, s, node, J); break;
        }
      }
    }
  } else if (FULL && lane == item.count) {
    imu_zero_part(Js + 6 * lane, warp);
  }
  if (FULL) {
    ICLK(1);
    __syncthreads();
    ICLK(2);
    const int nsteps = (6 * item.count + 3) >> 2;
    double acc[3][2];
    switch (warp) {
      case 0: imu_syrk<0>(Js, nsteps, lane, acc); break;
      case 1: imu_syrk<1>(Js, nsteps, lane, acc); break;
      case 2: imu_syrk<2>(Js, nsteps, lane, acc); break;
      default: imu_syrk<3>(Js, nsteps, lane, acc); break;
    }
    ICLK(3);
    ICLK(4);  // (no shared-memory reduction: every tile has one owner warp)
    det_ticket_wait(a.det_ticket, blockIdx.x);
    switch (warp) {
      case 0: imu_flush<0>(a, item, lane, acc); break;
      case 1: imu_flush<1>(a, item, lane, acc); break;
      case 2: imu_flush<2>(a, item, lane, acc); break;
      default: imu_flush<3>(a, item, lane, acc); break;
    }
    ICLK(5);
  }
  if (!FULL) det_ticket_wait(a.det_ticket, blockIdx.x);
  if (warp == 0) {  // every warp evaluated the same samples; warp 0's lanes hold them in sample order
    cost = warp_sum_d(cost);
    if (lane == 0 && cost != 0.0) atomicAdd(a.ne.cost, cost);
  }
  det_ticket_done(a.det_ticket, blockIdx.x);
}

int launch_imu(const ImuLaunch& l, bool full, cudaStream_t s) {
  if (l.n_items <= 0) return 0;
  ImuArgs a{l.obs, l.items, l.st, l.ne, l.dims, l.sp, l.rig, l.cmask, l.scal, l.det_ticket};
  const size_t smem = size_t(kImuCols) * kImuColStride * sizeof(double);
  static PerDeviceOnce once;
  if (once.first()) cudaFuncSetAttribute(imu_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem));
  if (full) imu_kernel<true><<<l.n_items, kImuThreads, smem, s>>>(a);
  else imu_kernel<false><<<l.n_items, kImuThreads, 0, s>>>(a);
  return 1;
}

// ------------------------------------------------------------------------------------------------
// K3: bias random-walk factors + marginalization prior (one CTA; the n x n J'J of the prior is a
// constant and is added by a separate elementwise kernel).

struct SmallArgs {
  BiasFactorPtrs bf;
  PriorPtrs prior;
  StatePtrs st;
  NormalEqPtrs ne;
  ProblemDims dims;
  const uint8_t* cmask;
  LmScalars* scal;
  int deterministic;
};

template <bool FULL>
__global__ void __launch_bounds__(256) small_factors_kernel(const __grid_constant__ SmallArgs a) {
  __shared__ double red[8];
  const int tid = threadIdx.x;
  double cost = 0.0;
  const int np = a.dims.np;
  // bias factors (trajectory_value_factor.h:45-99); deterministic mode: thread 0 walks them in order
  for (int n = a.deterministic ? (tid == 0 ? 0 : a.bf.n) : tid; n < a.bf.n; n += a.deterministic ? 1 : blockDim.x) {
    const int2 ij = a.bf.ij[n];
#pragma unroll
    for (int k = 0; k < 6; ++k) {
      const double s = a.bf.sqrt_info[6 * n + k];
      const double r = s * (a.st.bias[6 * ij.y + k] - a.st.bias[6 * ij.x + k]);
      cost += 0.5 * r * r;
      if (FULL) {
        const int gi = a.dims.idx_bias0 + 6 * ij.x + k, gj = a.dims.idx_bias0 + 6 * ij.y + k;
        const double ji = a.cmask[gi] ? 0.0 : -s, jj = a.cmask[gj] ? 0.0 : s;
        atomicAdd(a.ne.gc + gi, ji * r);
        atomicAdd(a.ne.gc + gj, jj * r);
        atomicAdd(a.ne.A + size_t(gi) * np + gi, ji * ji);
        atomicAdd(a.ne.A + size_t(gj) * np + gj, jj * jj);
        atomicAdd(a.ne.A + size_t(min(gi, gj)) * np + max(gi, gj), ji * jj);
      }
    }
  }
  // prior (marginalization_factor.cpp:326-373)
  const int n = a.prior.n;
  if (n > 0) {
    for (int b = tid; b < a.prior.n_blocks; b += blockDim.x) {
      const int type = a.prior.type[b];
      prior_block_dx(type, block_state(a.st, type, a.prior.index[b]), a.prior.x0 + 4 * b, a.prior.dx + a.prior.col[b]);
    }
    __syncthreads();
    for (int i = tid; i < n; i += blockDim.x) {
      double s = a.prior.r[i];
      const double* Ji = a.prior.J + size_t(i) * n;
      for (int j = 0; j < n; ++j) s = fma(Ji[j], a.prior.dx[j], s);
      a.prior.res[i] = s;
      cost += 0.5 * s * s;
    }
    if (FULL) {
      __syncthreads();
      for (int j = tid; j < n; j += blockDim.x) {
        const int g = a.prior.col2g[j];
        if (g < 0) continue;
        double s = 0;
        for (int i = 0; i < n; ++i) s = fma(a.prior.J[size_t(i) * n + j], a.prior.res[i], s);
        atomicAdd(a.ne.gc + g, s);
      }
    }
  }
  cost = warp_sum_d(cost);
  if ((tid & 31) == 0) red[tid >> 5] = cost;
  __syncthreads();
  if (tid == 0) {
    double c = 0;
    for (int w = 0; w < 8; ++w) c += red[w];
    if (c != 0.0) atomicAdd(a.ne.cost, c);
  }
}

__global__ void prior_add_jtj_kernel(PriorPtrs pr, double* A, int np) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  const int n = pr.n;
  if (idx >= n * n) return;
  const int i = idx / n, j = idx % n;
  if (j < i) return;
  const int gi = pr.col2g[i], gj = pr.col2g[j];
  if (gi < 0 || gj < 0) return;
  const double v = pr.JtJ[idx];
  if (v == 0.0) return;
  // distinct prior columns map to distinct camera dims, so no diagonal doubling is needed
  atomicAdd(A + size_t(min(gi, gj)) * np + max(gi, gj), v);
}

int launch_small_factors(const SmallFactorsLaunch& l, bool full, cudaStream_t s) {
  if (l.bf.n <= 0 && l.prior.n <= 0) return 0;
  SmallArgs a{l.bf, l.prior, l.st, l.ne, l.dims, l.cmask, l.scal, l.deterministic};
  int launches = 1;
  if (full) small_factors_kernel<true><<<1, 256, 0, s>>>(a);
  else small_factors_kernel<false><<<1, 256, 0, s>>>(a);
  if (full && l.prior.n > 0) {
    const int n2 = l.prior.n * l.prior.n;
    prior_add_jtj_kernel<<<(n2 + 255) / 256, 256, 0, s>>>(l.prior, l.ne.A, l.dims.np);
    ++launches;
  }
  return launches;
}

// ------------------------------------------------------------------------------------------------
// probes: per-factor outputs in the C-ABI layout (one thread per factor, both sides in one thread;
// an independent path from the fused lane-pair kernel, used by the parity tests)

__global__ void probe_image_kernel(VisArgs a, const int32_t* orig_index, int want_jac, double* r, int32_t* sidx,
                                   double* J) {
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= a.obs.n) return;
  const longlong2 tt = a.obs.t[n];
  const double2 pi = a.obs.pi[n], pj = a.obs.pj[n];
  const int4 meta = a.obs.meta[n];
  const double rho = a.st.rho[meta.z];
  const int64_t ld_ns = int64_t(*a.st.ld * 1e9);
  int32_t si, sj;
  double ui, uj;
  const int out = orig_index[n];
  if (!spline_index(a.sp, tt.x + int64_t(meta.x) * ld_ns, si, ui) ||
      !spline_index(a.sp, tt.y + int64_t(meta.y) * ld_ns, sj, uj)) {
    atomicOr(&a.scal->error_flags, 1);
    return;
  }
  SideEval ea, eb;
  if (want_jac) {
    eval_side<true, kPStride>(a.sp, a.st.q, a.st.p, a.st.tab, si, ui, ea);
    eval_side<true, kPStride>(a.sp, a.st.q, a.st.p, a.st.tab, sj, uj, eb);
  } else {
    eval_side<false, kPStride>(a.sp, a.st.q, a.st.p, a.st.tab, si, ui, ea);
    eval_side<false, kPStride>(a.sp, a.st.q, a.st.p, a.st.tab, sj, uj, eb);
  }
  ImageCommon cm;
  const double pixy[2] = {pi.x, pi.y}, pjxy[2] = {pj.x, pj.y};
  image_common(a.rig, pixy, pjxy, rho, ea.R, ea.p, eb.R, eb.p, a.cauchy, cm);
  atomicAdd(a.ne.cost, cm.cost);
  if (r) { r[2 * out] = cm.r[0]; r[2 * out + 1] = cm.r[1]; }
  if (sidx) { sidx[2 * out] = si; sidx[2 * out + 1] = sj; }
  if (!want_jac || !J) return;
  double* Jo = J + size_t(out) * 100;
  double rot[4][6], pos[4][6];
  image_side_blocks(0, cm, ea, rot, pos);
  for (int k = 0; k < 4; ++k)
    for (int e = 0; e < 6; ++e) { Jo[k * 12 + e] = rot[k][e]; Jo[k * 12 + 6 + e] = pos[k][e]; }
  image_side_blocks(1, cm, eb, rot, pos);
  for (int k = 0; k < 4; ++k)
    for (int e = 0; e < 6; ++e) { Jo[48 + k * 12 + e] = rot[k][e]; Jo[48 + k * 12 + 6 + e] = pos[k][e]; }
  image_jrho(a.rig, cm, ea.R, rho, Jo + 96);
  image_jld(a.rig, cm, meta.x, meta.y, ea.R, ea.omega, ea.vel, eb.R, eb.omega, eb.vel, Jo + 98);
}

int launch_probe_image(const VisualLaunch& l, const int32_t* orig_index, bool want_jac, double* r, int32_t* s,
                       double* J, cudaStream_t st) {
  if (l.obs.n <= 0) return 0;
  VisArgs a{l.obs, l.items, l.st, l.ne, l.lm, l.dims, l.sp, l.rig, l.cauchy, l.cmask, l.scal, nullptr};
  probe_image_kernel<<<(l.obs.n + 63) / 64, 64, 0, st>>>(a, orig_index, want_jac ? 1 : 0, r, s, J);
  return 1;
}

__global__ void probe_imu_kernel(ImuArgs a, const int32_t* orig_index, int want_jac, double* r, int32_t* sidx, double* J) {
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= a.obs.n) return;
  const int out = orig_index[n];
  const longlong2 tn = a.obs.t_node[n];
  const double2 g0 = a.obs.ga[3 * n], g1 = a.obs.ga[3 * n + 1], g2 = a.obs.ga[3 * n + 2];
  const double gyro[3] = {g0.x, g0.y, g1.x}, accel[3] = {g1.y, g2.x, g2.y};
  const int node = int(tn.y);
  double bias[6];
  for (int c = 0; c < 6; ++c) bias[c] = a.st.bias[6 * node + c];
  int32_t s;
  double u;
  if (!spline_index(a.sp, tn.x, s, u)) {
    atomicOr(&a.scal->error_flags, 1);
    return;
  }
  ImuEvalOut o;
  if (want_jac) eval_imu<true, kPStride>(a.sp, a.rig, a.st.q, a.st.p, a.st.tab, s, u, gyro, accel, bias, o);
  else eval_imu<false, kPStride>(a.sp, a.rig, a.st.q, a.st.p, a.st.tab, s, u, gyro, accel, bias, o);
  atomicAdd(a.ne.cost, o.cost);
  if (r) for (int k = 0; k < 6; ++k) r[6 * out + k] = o.r[k];
  if (sidx) sidx[out] = s;
  if (!want_jac || !J) return;
  double* Jo = J + size_t(out) * 156;
  for (int k = 0; k < 4; ++k)
    for (int e = 0; e < 18; ++e) { Jo[k * 36 + e] = o.Jrot[k][e]; Jo[k * 36 + 18 + e] = o.Jpos[k][e]; }
  for (int k = 0; k < 3; ++k) {
    Jo[144 + k] = a.rig.imu_info[k]; Jo[147 + k] = 0; Jo[150 + k] = 0; Jo[153 + k] = a.rig.imu_info[3 + k];
  }
}

int launch_probe_imu(const ImuLaunch& l, const int32_t* orig_index, bool want_jac, double* r, int32_t* s, double* J,
                     cudaStream_t st) {
  if (l.obs.n <= 0) return 0;
  ImuArgs a{l.obs, l.items, l.st, l.ne, l.dims, l.sp, l.rig, l.cmask, l.scal, nullptr};
  probe_imu_kernel<<<(l.obs.n + 63) / 64, 64, 0, st>>>(a, orig_index, want_jac ? 1 : 0, r, s, J);
  return 1;
}

// ------------------------------------------------------------------------------------------------
// spline query service (Trajectory::poseNs / GetIMUState, spline/trajectory.cpp:27-55)

__global__ void query_kernel(QueryLaunch a) {
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= a.n) return;
  int32_t s;
  double u;
  if (!spline_index(a.sp, a.t[n], s, u)) {
    atomicOr(&a.scal->error_flags, 1);
    return;
  }
  SideEval ev;
  eval_side<true, kPStride>(a.sp, a.st.q, a.st.p, a.st.tab, s, u, ev);
  if (a.q) {
    const Q4 q = quat_from_matrix(ev.R);
    a.q[4 * n] = q.x; a.q[4 * n + 1] = q.y; a.q[4 * n + 2] = q.z; a.q[4 * n + 3] = q.w;
  }
  if (a.p) { a.p[3 * n] = ev.p.x; a.p[3 * n + 1] = ev.p.y; a.p[3 * n + 2] = ev.p.z; }
  if (a.omega) { a.omega[3 * n] = ev.omega.x; a.omega[3 * n + 1] = ev.omega.y; a.omega[3 * n + 2] = ev.omega.z; }
  if (a.vel) { a.vel[3 * n] = ev.vel.x; a.vel[3 * n + 1] = ev.vel.y; a.vel[3 * n + 2] = ev.vel.z; }
  if (a.acc) {
    double c2[4];
    plain_coeffs<2>(u, a.sp.inv_dt, c2);
    V3 acc = c2[0] * load_p<kPStride>(a.st.p, s);
    for (int k = 1; k < 4; ++k) acc = acc + c2[k] * load_p<kPStride>(a.st.p, s + k);
    a.acc[3 * n] = acc.x; a.acc[3 * n + 1] = acc.y; a.acc[3 * n + 2] = acc.z;
  }
}

int launch_query(const QueryLaunch& a, cudaStream_t s) {
  if (a.n <= 0) return 0;
  query_kernel<<<(a.n + 127) / 128, 128, 0, s>>>(a);
  return 1;
}

}  // namespace ctvio
