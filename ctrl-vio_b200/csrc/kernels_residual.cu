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
//     and reduced by a register-tiled SYRK (8x8 tiles, 7 row groups) into a shared accumulator that
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
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
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

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
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
  int use_tma;
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
#define VCLK(i) do { if (blockIdx.x == 0 && threadIdx.x == 0) g_vis_clk[(i)] = clock64(); } while (0)
extern "C" int ctvio_debug_vis_clk(long long* out) {
  return cudaMemcpyFromSymbol(out, g_vis_clk, sizeof(g_vis_clk)) == cudaSuccess ? 0 : -1;
}
#else
#define VCLK(i)
#endif

size_t visual_smem_bytes() {
  return size_t(kVisObsPerRound) * kObsStride * sizeof(double) + size_t(36) * 64 * sizeof(double);
}

// SYRK of one round's Jacobian rows into the CTA accumulator (upper 8x8 tiles of the 64 local dims) on the fp64
// tensor cores (m8n8k4; K = Jacobian rows).  The 36 upper tiles are grouped into 16x16 blocks, one or two per warp
// (warps 0..5: the six off-diagonal blocks, warps 6, 7: two diagonal blocks each), so that every tile has ONE owner
// warp over all rows: no cross-warp merge, the partial sums of earlier rounds are simply reloaded from accs.
// Rows of inactive observation slots are zero (written by the evaluation phase), so K runs in whole 4-row steps.
__device__ __noinline__ void syrk_round(const double* Jt, double* accs, int nround, int tid) {
  const int warp = tid >> 5, lane = tid & 31, g = lane >> 2, q = lane & 3;
  const int nblk = warp < 6 ? 1 : 2;
  int bi[2], bj[2];
  if (warp < 6) {
    bi[0] = warp < 3 ? 0 : (warp < 5 ? 1 : 2);
    bj[0] = warp < 3 ? warp + 1 : (warp < 5 ? warp - 1 : 3);
    bi[1] = bj[1] = 0;
  } else {
    bi[0] = bj[0] = 2 * (warp - 6);
    bi[1] = bj[1] = 2 * (warp - 6) + 1;
  }
  const bool dg = warp >= 6;
  double acc[2][2][2][2];
#pragma unroll
  for (int b = 0; b < 2; ++b)
#pragma unroll
    for (int mi = 0; mi < 2; ++mi)
#pragma unroll
      for (int nj = 0; nj < 2; ++nj) {
        const int ti = 2 * bi[b] + mi, tj = 2 * bj[b] + nj;
        double2 v = make_double2(0.0, 0.0);
        if (b < nblk && ti <= tj) v = *reinterpret_cast<const double2*>(accs + (ti * 8 - ti * (ti - 1) / 2 + (tj - ti)) * 64 + g * 8 + 2 * q);
        acc[b][mi][nj][0] = v.x; acc[b][mi][nj][1] = v.y;
      }
  const int nsteps = (2 * nround + 3) >> 2;
#pragma unroll 2
  for (int st = 0; st < nsteps; ++st) {
    const int row = 4 * st + q;
    const double* rp = Jt + size_t(row >> 1) * kObsStride + (row & 1) * kRowStride + g;
#pragma unroll
    for (int b = 0; b < 2; ++b) {
      if (b < nblk) {
        double av[2], bv[2];
#pragma unroll
        for (int m = 0; m < 2; ++m) {
          av[m] = rp[16 * bi[b] + 8 * m];
          bv[m] = dg ? av[m] : rp[16 * bj[b] + 8 * m];
        }
#pragma unroll
        for (int mi = 0; mi < 2; ++mi)
#pragma unroll
          for (int nj = 0; nj < 2; ++nj) {
            if (dg && mi == 1 && nj == 0) continue;  // strictly lower tile of a diagonal block
            asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};"
                         : "+d"(acc[b][mi][nj][0]), "+d"(acc[b][mi][nj][1])
                         : "d"(av[mi]), "d"(bv[nj]));
          }
      }
    }
  }
#pragma unroll
  for (int b = 0; b < 2; ++b)
#pragma unroll
    for (int mi = 0; mi < 2; ++mi)
#pragma unroll
      for (int nj = 0; nj < 2; ++nj) {
        const int ti = 2 * bi[b] + mi, tj = 2 * bj[b] + nj;
        if (b < nblk && ti <= tj)
          *reinterpret_cast<double2*>(accs + (ti * 8 - ti * (ti - 1) / 2 + (tj - ti)) * 64 + g * 8 + 2 * q) =
              make_double2(acc[b][mi][nj][0], acc[b][mi][nj][1]);
      }
  __syncthreads();
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
  if (a.use_tma) {
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
  } else {
    if (tid == 0) sm.err = 0;
    // plain cooperative loads (debug path, CTVIO_NO_TMA=1)
    for (int i = tid; i < 2 * kWinKnots * 4; i += kVisThreads) {
      const int sd = i / (kWinKnots * 4), r = i % (kWinKnots * 4);
      const int k = w0[sd] + r / 4;
      (&sm.q[sd][0][0])[r] = k < nK ? a.st.q[4 * k + (r & 3)] : 0.0;
      (&sm.p[sd][0][0])[r] = k < nK ? a.st.p[4 * k + (r & 3)] : 0.0;
    }
    for (int i = tid; i < 2 * 4 * 16; i += kVisThreads) {
      const int sd = i / 64, r = i % 64;
      const int k = w0[sd] + r / 16;
      reinterpret_cast<double*>(&sm.tab[sd][0])[r] = k < nK - 1 ? reinterpret_cast<const double*>(a.st.tab + k)[r & 15] : 0.0;
    }
  }
  if (FULL)
    for (int i = tid; i < 36 * 64; i += kVisThreads) accs[i] = 0.0;
  if (a.use_tma) {
    while (!mbar_try_wait(reinterpret_cast<uint64_t*>(&sm.bar), 0)) {
    }
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
#ifndef CTVIO_EXPERIMENT_NO_W_ATOMICS
              if (!a.det_ticket) {  // (deterministic mode: recomputed from the shared tile inside the ordered flush)
                if (!mr) atomicAdd(Wl + gd + c, r0v * jrho[0] + r1v * jrho[1]);
                if (!mp) atomicAdd(Wl + gd + 3 + c, p0v * jrho[0] + p1v * jrho[1]);
              }
#endif
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
        if (active && valid) {
          const int oi = item.start + base + ol;
          const int l = a.obs.meta[oi].z;
          const double j0 = row0[kColRho], j1 = row1[kColRho];
          if (side == 0) {
            atomicAdd(a.ne.hl + l, j0 * j0 + j1 * j1);
            atomicAdd(a.ne.gl + l, j0 * row0[kColR] + j1 * row1[kColR]);
          } else {
            atomicAdd(a.ne.wld + l, row0[kColLd] * j0 + row1[kColLd] * j1);
          }
        }
        // the two knot windows of an observation may overlap (same global dims): anchor side first, then the other one
        for (int ph = 0; ph < 2; ++ph) {
          if (active && valid && side == ph) {
            const int oi = item.start + base + ol;
            const int l = a.obs.meta[oi].z;
            const double j0 = row0[kColRho], j1 = row1[kColRho];
            double* Wl = a.ne.W + (a.lm.woff[l] - a.lm.lo[l]);
            const int cb = side * 30, gk0 = w0[side];
            for (int c = 0; c < 30; ++c) {
              const double v = row0[cb + c] * j0 + row1[cb + c] * j1;
              if (v != 0.0) atomicAdd(Wl + 6 * gk0 + c, v);
            }
          }
          __threadfence();
          __syncthreads();
        }
        det_ticket_done(a.det_ticket, blockIdx.x * 1024 + base / kVisObsPerRound);
      }
      syrk_round(Jt, accs, nround, tid);
      VCLK(4);
    }
  }

  // ---- cost + flush ----
  const int n_rounds = (item.count + kVisObsPerRound - 1) / kVisObsPerRound;
  det_ticket_wait(a.det_ticket, blockIdx.x * 1024 + (FULL ? n_rounds : 0));
  cost_local = warp_sum(cost_local);
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
  VisArgs a{l.obs, l.items, l.st, l.ne, l.lm, l.dims, l.sp, l.rig, l.cauchy, l.cmask, l.scal, l.use_tma ? 1 : 0, l.det_ticket};
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
// K2: IMU factors.  One CTA per (start knot, bias node) run of samples (<= 32): lanes of warp 0 evaluate
// one sample each, the 6 x 31 Jacobian rows (24 knot dims | 6 bias dims | residual) go to shared memory and
// all 64 threads reduce J'J with the same 8x8 register-tiled SYRK as K1 (10 upper tiles x 6 row groups),
// flushing one fp64 atomic per non-zero entry per CTA.

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

constexpr int kImuThreads = 64;
constexpr int kImuCols = 32;      // 24 knot dims + 6 bias dims + residual + pad
constexpr int kImuRowStride = 34; // doubles; 16-B aligned rows, fewer store conflicts
__constant__ uint8_t c_imu_tile_i[10] = {0, 0, 0, 0, 1, 1, 1, 2, 2, 3};
__constant__ uint8_t c_imu_tile_j[10] = {0, 1, 2, 3, 1, 2, 3, 2, 3, 3};

template <bool FULL>
__global__ void __launch_bounds__(kImuThreads) imu_kernel(const __grid_constant__ ImuArgs a) {
  extern __shared__ __align__(16) unsigned char dyn_smem[];
  double* Js = reinterpret_cast<double*>(dyn_smem);            // [32 samples x 6 rows][kImuRowStride]
  double* accs = Js + kImuMaxPerItem * 6 * kImuRowStride;      // [10][64]
  const int tid = threadIdx.x;
  const ImuItem item = a.items[blockIdx.x];
  double cost = 0.0;
  if (FULL)
    for (int i = tid; i < 10 * 64; i += kImuThreads) accs[i] = 0.0;
  if (tid < item.count) {
    const int n = item.start + tid;
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
    double* J = Js + size_t(tid) * 6 * kImuRowStride;
    if (!ok) {
      atomicOr(&a.scal->error_flags, 1);
      if (FULL)
        for (int e = 0; e < 6 * kImuRowStride; ++e) J[e] = 0.0;
    } else {
      ImuEvalOut o;
      eval_imu<FULL, kPStride>(a.sp, a.rig, a.st.q, a.st.p, a.st.tab, s, u, gyro, accel, bias, o);
      cost = o.cost;
      if (FULL) {
        const int gb0 = a.dims.idx_bias0 + 6 * node;
#pragma unroll
        for (int r = 0; r < 6; ++r) {
          double* Jr = J + r * kImuRowStride;
#pragma unroll
          for (int k = 0; k < 4; ++k)
#pragma unroll
            for (int c = 0; c < 3; ++c) {
              Jr[k * 6 + c] = a.cmask[6 * (s + k) + c] ? 0.0 : o.Jrot[k][3 * r + c];
              Jr[k * 6 + 3 + c] = a.cmask[6 * (s + k) + 3 + c] ? 0.0 : o.Jpos[k][3 * r + c];
            }
#pragma unroll
          for (int c = 0; c < 6; ++c) Jr[24 + c] = (c == r && !a.cmask[gb0 + c]) ? a.rig.imu_info[r] : 0.0;
          Jr[30] = o.r[r];
          Jr[31] = 0.0;
        }
      }
    }
  }
  if (FULL) {
    __syncthreads();
    const int grp = tid / 10, tile = tid % 10;
    double acc[64];
    if (tid < 60) {
      const int ti = c_imu_tile_i[tile], tj = c_imu_tile_j[tile];
#pragma unroll
      for (int e = 0; e < 64; ++e) acc[e] = 0.0;
      const int nrows = 6 * item.count;
      for (int row = grp; row < nrows; row += 6) {
        const double2* ra = reinterpret_cast<const double2*>(Js + size_t(row) * kImuRowStride + ti * 8);
        const double2* rb = reinterpret_cast<const double2*>(Js + size_t(row) * kImuRowStride + tj * 8);
        double av[8], bv[8];
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const double2 x = ra[e], y = rb[e];
          av[2 * e] = x.x; av[2 * e + 1] = x.y;
          bv[2 * e] = y.x; bv[2 * e + 1] = y.y;
        }
#pragma unroll
        for (int i = 0; i < 8; ++i)
#pragma unroll
          for (int j = 0; j < 8; ++j) acc[i * 8 + j] = fma(av[i], bv[j], acc[i * 8 + j]);
      }
    }
    for (int g = 0; g < 6; ++g) {
      if (tid < 60 && grp == g) {
#pragma unroll
        for (int e = 0; e < 64; ++e) accs[tile * 64 + e] += acc[e];
      }
      __syncthreads();
    }
    const int np = a.dims.np;
    det_ticket_wait(a.det_ticket, blockIdx.x);
    for (int idx = tid; idx < 10 * 64; idx += kImuThreads) {
      const double val = accs[idx];
      if (val == 0.0) continue;
      const int tile2 = idx >> 6, e = idx & 63;
      const int la = c_imu_tile_i[tile2] * 8 + (e >> 3), lb = c_imu_tile_j[tile2] * 8 + (e & 7);
      if (la > lb || lb > 30 || la >= 30) continue;
      const int ga = la < 24 ? 6 * item.s + la : a.dims.idx_bias0 + 6 * item.node + (la - 24);
      if (lb == 30) {
        atomicAdd(a.ne.gc + ga, val);
        continue;
      }
      const int gb = lb < 24 ? 6 * item.s + lb : a.dims.idx_bias0 + 6 * item.node + (lb - 24);
      atomicAdd(a.ne.A + size_t(ga) * np + gb, val);  // ga <= gb: knot dims precede bias dims
    }
  }
  if (!FULL) det_ticket_wait(a.det_ticket, blockIdx.x);
  cost = warp_sum(cost);
  if (tid == 0 && cost != 0.0) atomicAdd(a.ne.cost, cost);  // only warp 0 evaluates (count <= 32)
  det_ticket_done(a.det_ticket, blockIdx.x);
}

int launch_imu(const ImuLaunch& l, bool full, cudaStream_t s) {
  if (l.n_items <= 0) return 0;
  ImuArgs a{l.obs, l.items, l.st, l.ne, l.dims, l.sp, l.rig, l.cmask, l.scal, l.det_ticket};
  const size_t smem = (size_t(kImuMaxPerItem) * 6 * kImuRowStride + 10 * 64) * sizeof(double);
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

__device__ __forceinline__ const double* block_data(const StatePtrs& st, int type, int index) {
  switch (type) {
    case 0: return st.q + 4 * index;
    case 1: return st.p + kPStride * index;
    case 2: return st.bias + 6 * index;
    case 3: return st.bias + 6 * index + 3;
    case 4: return st.ld;
    default: return st.rho + index;
  }
}

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
      const double* x = block_data(a.st, type, a.prior.index[b]);
      const double* x0 = a.prior.x0 + 4 * b;
      double* dx = a.prior.dx + a.prior.col[b];
      if (type == 0) {
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
        const int sz = (type == 4 || type == 5) ? 1 : 3;
        for (int d = 0; d < sz; ++d) dx[d] = x[d] - x0[d];
      }
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
  cost = warp_sum(cost);
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
  VisArgs a{l.obs, l.items, l.st, l.ne, l.lm, l.dims, l.sp, l.rig, l.cauchy, l.cmask, l.scal, 0, nullptr};
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
