// Shared device helpers of the dense Cholesky kernels (K5): 64x64 fp64 tiles in shared memory, 256 threads,
// thread (ty, tx) = (tid >> 4, tid & 15) owns the 4x4 register block rows 4ty.., cols 4tx...
#pragma once
#include "kernels.h"

namespace ctvio {

#ifdef CTVIO_CHOL_TIMING
__device__ long long g_fac_clk[8 * 4 * 8];
#define FCLK(s, i) do { if (blockIdx.x == 0 && (threadIdx.x & 31) == 0) g_fac_clk[(threadIdx.x >> 5) * 32 + (s) * 8 + (i)] = clock64(); } while (0)
#else
#define FCLK(s, i)
#endif

constexpr int kTS = kCholNB + 4;  // shared tile row stride (doubles): rows stay 16-B aligned; 68 = 4 mod 8 keeps the
                                  // m8n8k4 fragment loads ([4 k-rows][8 consecutive]) of a half-warp on distinct banks
constexpr int kTile = kCholNB * kTS;
constexpr size_t kCholCoopSmem = (5 * size_t(kTile) + 4 * kCholNB) * sizeof(double);

// acc[4][4] += A * B^T for 64x64 operands, BOTH stored transposed in smem: At[c][i] = A[i][c], Bt[c][j] = B[j][c].
// 256 threads, thread (ty, tx) owns rows 4ty.., cols 4tx..; four 16-byte shared loads feed 16 FMAs per k.
__device__ __forceinline__ void tile_gemm_tt(const double* At, const double* Bt, double acc[4][4], int ty, int tx) {
#pragma unroll 8
  for (int c = 0; c < kCholNB; ++c) {
    const double2 a01 = *reinterpret_cast<const double2*>(At + c * kTS + 4 * ty);
    const double2 a23 = *reinterpret_cast<const double2*>(At + c * kTS + 4 * ty + 2);
    const double2 b01 = *reinterpret_cast<const double2*>(Bt + c * kTS + 4 * tx);
    const double2 b23 = *reinterpret_cast<const double2*>(Bt + c * kTS + 4 * tx + 2);
    const double av[4] = {a01.x, a01.y, a23.x, a23.y};
    const double bv[4] = {b01.x, b01.y, b23.x, b23.y};
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) acc[i][j] = fma(av[i], bv[j], acc[i][j]);
  }
}

// smem tile <- TRANSPOSE of the 64x64 global block at M[r0.., c0..]: dst[c][r] = M[r0 + r][c0 + c]
// (coalesced 16-byte global reads along c)
__device__ __forceinline__ void load_tile_transposed(double* dst, const double* M, int npad, int r0, int c0, int tid) {
  for (int e = tid; e < kCholNB * kCholNB / 2; e += 256) {
    const int r = e >> 5, c = (e & 31) * 2;
    const double2 v = *reinterpret_cast<const double2*>(M + size_t(r0 + r) * npad + c0 + c);
    dst[c * kTS + r] = v.x;
    dst[(c + 1) * kTS + r] = v.y;
  }
}

// 1/sqrt(x) for a positive, normal x without the special-case branch of rsqrt(): hardware seed (2^-22.9) plus one
// third-order step  y (1 + e/2 + 3 e^2/8),  e = 1 - x y^2  -> relative error ~ e^3, i.e. full double precision.
// Branch-free on purpose: the call sits in the serial pivot chain of the factorisation and a branch would stop the
// compiler from interleaving the chain with the independent update FMAs around it.
__device__ __forceinline__ double rsqrt_pos(double x) {
  double y;
  asm("rsqrt.approx.ftz.f64 %0, %1;" : "=d"(y) : "d"(x));
  const double e = fma(-(y * y), x, 1.0);
  const double p = fma(e, 0.375, 0.5);
  const double ye = y * e;
  return fma(p, ye, y);
}

// Lower Cholesky of the 64x64 block D (row-major, row stride kTS; destroyed) by 256 threads, producing the inverse
// factor Xi = L^-1 (lower triangular, row-major) and XiT = Xi^T.  T is scratch (>= 256 + 16 * kTS + 16 * kX16Stride doubles),
// rdiag[64] receives 1 / L_jj.  Returns false on a non-positive pivot (the pivot is replaced by 1 so that the
// sweep terminates with finite numbers).
//
// The serial pivot chain (rsqrt -> scale -> rank-1 update of the next pivot) is what bounds this routine, so it is
// organised around that chain: four 16-column steps, each
//   P1  ONE warp factors the 16x16 diagonal block out of registers (lane = row, columns broadcast by shuffles, the
//       running diagonal kept in its own register so that the next pivot needs a single shuffle): no barriers or
//       shared-memory round trips inside the 16 dependent columns;
//   P2  the panel below and the block row of the inverse as small tensor-core products with the explicit 16x16
//       inverse, which the 16 otherwise idle lanes of the P1 warp compute alongside the factorisation;
//   P3  the trailing update of D and of the running sums in Xi as m8n8k4 fp64 tensor-core tiles (K = 16), overlapped
//       with P1 of the next step (warp 0 updates the next diagonal block first and starts its pivot chain at once).
//
// `side(s)` is called by the threads of warps 1..7 (tid >= 32) at the start of 16-column step s, i.e. while warp 0
// runs the P1 chain and they would otherwise idle at the barrier: room for unrelated work per step.
struct NoSideJob {
  __device__ __forceinline__ void operator()(int) const {}
};
constexpr int kX16Stride = 20;  // row stride (doubles) of the 16x16 inverse block: m8n8k4 fragment loads conflict-free

// P1 of 16-column step s (c0 = 16 s): executed by ONE full warp.  Lanes 0..15 hold the rows of the diagonal block;
// lanes 16..31 run the SAME instruction stream on the columns of the identity, i.e. lane 16 + c forward-substitutes
// column c of X16 = L16^-1 one pivot behind the factorisation, for free (SIMT).  XT16[m][k] = X16[k][m].
template <int XS = kX16Stride>
__device__ __forceinline__ void factor_p1_warp(double* D, double* L16t, double* XT16, double* rdiag, int* s_bad, int c0, int lane) {
  const int r = lane & 15;
  const bool real = lane < 16;
  double a[16];
  const double* row = D + (c0 + r) * kTS + c0;
#pragma unroll
  for (int c = 0; c < 16; c += 2) {
    const double2 v = *reinterpret_cast<const double2*>(row + c);
    a[c] = real ? v.x : (c == r ? 1.0 : 0.0);
    a[c + 1] = real ? v.y : (c + 1 == r ? 1.0 : 0.0);
  }
  double d = row[r];  // running diagonal element of this lane's row: the next pivot needs one shuffle only
  bool bad = false;
  // Software pipelined: the pivot of column j + 1 (shuffle, test, reciprocal square root: the long dependent part) is
  // issued BEFORE the 15 - j shared-memory loads and update FMAs of column j, which then execute in its shadow.  In
  // program order "pivot, then updates" the in-order issue of the update block delayed every pivot.
  double ajj = __shfl_sync(0xffffffffu, d, 0);
  {
    // positive and normal <=> biased exponent in [1, 2046] and sign clear (integer test: off the fp64 pipe)
    const unsigned hi = static_cast<unsigned>(__double2hiint(ajj));
    if (hi - 0x00100000u >= 0x7fe00000u) { bad = true; ajj = 1.0; }
  }
  double rinv = rsqrt_pos(ajj);
#pragma unroll
  for (int j = 0; j < 16; ++j) {
    const double lij = a[j] * rinv;  // lanes 0..15: L[row][j];  lanes 16..31: X16[j][column]
    a[j] = lij;
    d = fma(-lij, lij, d);
    // column j goes to the others through its (final) line of the transposed block: L16t[j][row]
    if (real) L16t[j * 16 + r] = lij;
    if (lane == j) rdiag[c0 + j] = rinv;
    double rinv_next = 0.0;
    if (j + 1 < 16) {
      ajj = __shfl_sync(0xffffffffu, d, j + 1);
      const unsigned hi = static_cast<unsigned>(__double2hiint(ajj));
      if (hi - 0x00100000u >= 0x7fe00000u) { bad = true; ajj = 1.0; }
      rinv_next = rsqrt_pos(ajj);
    }
    __syncwarp();
#pragma unroll
    for (int k = j + 1; k < 16; ++k) a[k] = fma(-lij, L16t[j * 16 + k], a[k]);
    rinv = rinv_next;
  }
  if (!real) {
#pragma unroll
    for (int k = 0; k < 16; k += 2) *reinterpret_cast<double2*>(XT16 + r * XS + k) = make_double2(a[k], a[k + 1]);
  }
  if (bad && lane == 0) *s_bad = 1;
}

// P3 of step s for one fragment column ct (B fragments loaded once, fragment rows two at a time); rows < skip_below
// are left out (they belong to the look-ahead warp)
__device__ __forceinline__ void factor_p3_column(double* D, double* Xi, const double* Pt, int c0, int C, int ct, int rt_first,
                                                 int g, int q) {
  const bool inv = 8 * ct < C;
  const double* pb = inv ? Xi + (c0 + q) * kTS + 8 * ct + g : Pt + q * kTS + 8 * ct + g;
  double* base = (inv ? Xi : D) + g * kTS + 8 * ct + 2 * q;
  double bv[4];
#pragma unroll
  for (int kk = 0; kk < 4; ++kk) bv[kk] = pb[4 * kk * kTS];
  int rt = rt_first;
  for (; rt + 1 < 8; rt += 2) {
    double2 c0v = *reinterpret_cast<const double2*>(base + 8 * rt * kTS);
    double2 c1v = *reinterpret_cast<const double2*>(base + 8 * (rt + 1) * kTS);
    const double* pa = Pt + q * kTS + 8 * rt + g;
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
      const double a0 = -pa[4 * kk * kTS], a1 = -pa[4 * kk * kTS + 8];
      asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};"
                   : "+d"(c0v.x), "+d"(c0v.y) : "d"(a0), "d"(bv[kk]));
      asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};"
                   : "+d"(c1v.x), "+d"(c1v.y) : "d"(a1), "d"(bv[kk]));
    }
    *reinterpret_cast<double2*>(base + 8 * rt * kTS) = c0v;
    *reinterpret_cast<double2*>(base + 8 * (rt + 1) * kTS) = c1v;
  }
  if (rt < 8) {
    double2 c0v = *reinterpret_cast<const double2*>(base + 8 * rt * kTS);
    const double* pa = Pt + q * kTS + 8 * rt + g;
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
      const double a0 = -pa[4 * kk * kTS];
      asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};"
                   : "+d"(c0v.x), "+d"(c0v.y) : "d"(a0), "d"(bv[kk]));
    }
    *reinterpret_cast<double2*>(base + 8 * rt * kTS) = c0v;
  }
}

template <class Side = NoSideJob>
__device__ __forceinline__ bool factor_and_invert_64(double* D, double* Xi, double* XiT, double* T, double* rdiag, int* s_bad,
                                                     Side side = Side()) {
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int g = lane >> 2, q = lane & 3;
  double* L16t = T;      // [16][16] current diagonal block of L, transposed: L16t[c][r] = L[r][c] (r >= c valid)
  double* Pt = T + 256;  // [16][kTS] current block column of L, transposed: Pt[m][row]
  double* XT16 = T + 256 + 16 * kTS;  // [16][kX16Stride] inverse of the current diagonal block, transposed
  if (tid == 0) *s_bad = 0;
  for (int e = tid; e < kTile; e += 256) Xi[e] = 0.0;
  __syncthreads();
  FCLK(0, 0);
  if (warp == 0) factor_p1_warp(D, L16t, XT16, rdiag, s_bad, 0, lane);
  else side(0);
  FCLK(0, 1);
  __syncthreads();
#pragma unroll 1
  for (int s = 0; s < 4; ++s) {
    const int c0 = 16 * s;
    const int R = 48 - c0, C = c0 + 16;
    {
      // ---- P2 as small tensor-core products with the explicit 16x16 inverse from P1:
      //   P2a  panel  L(rows below, c0..c0+15) = A_panel * X16^T            -> Pt (transposed, the operand of P3)
      //   P2b  block row of the inverse  X(c0..c0+15, cols < c0) = X16 * W   (in place in Xi), plus the diagonal block
      // one task = one panel row fragment (both column fragments) / one fragment column of the block row (both row
      // fragments: the product is in place) / the copy of the diagonal block ----
      const int n_a = R >> 3, n_b = c0 >> 3, ntask = n_a + n_b + 1;  // = 7 in every step: one task per warp
      for (int t = warp; t < ntask; t += 8) {
        if (t < n_a) {
          // both column fragments of one panel row fragment: shared A operand, two independent accumulator chains
          const int i0 = c0 + 16 + 8 * t;
          const double* pa = D + (i0 + g) * kTS + c0 + q;        // A[i0 + g][k0 + q]
          const double* pb = XT16 + q * kX16Stride + g;          // B[k0 + q][n0 + g] = X16[n0 + g][k0 + q]
          double2 cl = make_double2(0.0, 0.0), ch = make_double2(0.0, 0.0);
#pragma unroll
          for (int kk = 0; kk < 4; ++kk) {
            const double av = pa[4 * kk];
            if (kk < 2)                                           // X16 is lower triangular: k <= n
              asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};"
                           : "+d"(cl.x), "+d"(cl.y) : "d"(av), "d"(pb[4 * kk * kX16Stride]));
            asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};"
                         : "+d"(ch.x), "+d"(ch.y) : "d"(av), "d"(pb[4 * kk * kX16Stride + 8]));
          }
          Pt[(2 * q) * kTS + i0 + g] = cl.x;
          Pt[(2 * q + 1) * kTS + i0 + g] = cl.y;
          Pt[(8 + 2 * q) * kTS + i0 + g] = ch.x;
          Pt[(8 + 2 * q + 1) * kTS + i0 + g] = ch.y;
        } else if (t < n_a + n_b) {
          const int n0 = 8 * (t - n_a);
          double bv[4];
#pragma unroll
          for (int kk = 0; kk < 4; ++kk) bv[kk] = Xi[(c0 + 4 * kk + q) * kTS + n0 + g];   // W rows (running sums)
          const double* pa = XT16 + q * kX16Stride + g;          // A[r0 + g][k0 + q] = X16[r0 + g][k0 + q]
          double2 c0v = make_double2(0.0, 0.0), c1v = make_double2(0.0, 0.0);
#pragma unroll
          for (int kk = 0; kk < 4; ++kk) {
            if (kk < 2)
              asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};"
                           : "+d"(c0v.x), "+d"(c0v.y) : "d"(pa[4 * kk * kX16Stride]), "d"(bv[kk]));
            asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};"
                         : "+d"(c1v.x), "+d"(c1v.y) : "d"(pa[4 * kk * kX16Stride + 8]), "d"(bv[kk]));
          }
          // every lane's W values went through the mma above before any lane gets here: in place is safe
          *reinterpret_cast<double2*>(Xi + (c0 + g) * kTS + n0 + 2 * q) = c0v;
          *reinterpret_cast<double2*>(Xi + (c0 + 8 + g) * kTS + n0 + 2 * q) = c1v;
        } else {
          for (int e = lane; e < 256; e += 32) {
            const int rr = e >> 4, cc = e & 15;
            Xi[(c0 + rr) * kTS + c0 + cc] = cc <= rr ? XT16[cc * kX16Stride + rr] : 0.0;
          }
        }
      }
    }
    FCLK(s, 3);
    __syncthreads();
    // ---- P3 (rows >= c0+16:  D(:, >= c0+16) -= P P^T on the lower fragments,  Xi(:, < c0+16) -= P X(c0..c0+15, :))
    //      overlapped with P1 of the NEXT step: warp 0 updates the three fragments of the next 16x16 diagonal block first
    //      and runs its pivot chain while warps 1..7 do the rest of the update, then the side job of the next step ----
    if (s < 3) {
      const int rt0 = (c0 + 16) >> 3;
      if (warp == 0) {
        {  // the three lower fragments of the next diagonal block, three independent accumulator chains
          double* cp0 = D + (8 * rt0 + g) * kTS + 8 * rt0 + 2 * q;
          double* cp1 = cp0 + 8 * kTS;      // (rt0 + 1, rt0)
          double* cp2 = cp1 + 8;            // (rt0 + 1, rt0 + 1)
          double2 v0 = *reinterpret_cast<const double2*>(cp0), v1 = *reinterpret_cast<const double2*>(cp1),
                  v2 = *reinterpret_cast<const double2*>(cp2);
          const double* pp = Pt + q * kTS + 8 * rt0 + g;
#pragma unroll
          for (int kk = 0; kk < 4; ++kk) {
            const double p0 = pp[4 * kk * kTS], p1 = pp[4 * kk * kTS + 8];
            const double a0 = -p0, a1 = -p1;
            asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};"
                         : "+d"(v0.x), "+d"(v0.y) : "d"(a0), "d"(p0));
            asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};"
                         : "+d"(v1.x), "+d"(v1.y) : "d"(a1), "d"(p0));
            asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};"
                         : "+d"(v2.x), "+d"(v2.y) : "d"(a1), "d"(p1));
          }
          *reinterpret_cast<double2*>(cp0) = v0;
          *reinterpret_cast<double2*>(cp1) = v1;
          *reinterpret_cast<double2*>(cp2) = v2;
        }
        __syncwarp();
        factor_p1_warp(D, L16t, XT16, rdiag, s_bad, c0 + 16, lane);
      } else {
        // fragment column = warp (warp 7 also takes column 0); fragment rows start at max(ct, rt0); the look-ahead
        // fragments (rt0, rt0), (rt0+1, rt0), (rt0+1, rt0+1) are warp 0's.  (Keeping warp 4 - same scheduler as the
        // pivot warp - out of the tensor-core work was measured to change nothing: the pivot chain runs slower
        // while the other warps' DMMAs are in flight whichever scheduler issues them, i.e. the fp64 pipe behaves as
        // one SM-wide resource; the overlap still hides about half of P3.)
        const int ct = warp;
        int first = ct > rt0 ? ct : rt0;
        if (ct == rt0 || ct == rt0 + 1) first = rt0 + 2;
        if (first < 8) factor_p3_column(D, Xi, Pt, c0, C, ct, first, g, q);
        if (warp == 7) factor_p3_column(D, Xi, Pt, c0, C, 0, rt0, g, q);
        side(s + 1);
      }
    }
    FCLK(s, 5);
    __syncthreads();
  }
  // XiT = Xi^T (B operand of the panel GEMMs)
  for (int e = tid; e < kCholNB * kCholNB; e += 256) {
    const int r = e >> 6, c = e & 63;
    XiT[c * kTS + r] = Xi[r * kTS + c];
  }
  __syncthreads();
  return *s_bad == 0;
}

// ---- factor WITHOUT the 64x64 inverse, publishing per 16-column step (tile-DAG kernel, chol_dag.cu) ----
// Packet of step s (row stride kPS, 16 rows m = column 16 s + m of the block):
//   cols  0..63  Pt_s[m][row] = L[row][16 s + m]  for row >= 16 (s + 1)   (the panel below the 16x16 diagonal block)
//   cols 64..79  XT16_s[m][k] = X16_s[k][m],  X16_s = (16x16 diagonal block of L)^-1
// Everything a consumer needs for the right-looking triangular solve of ITS tile against this block column, step by
// step:  P_s = T[:, 16 s ..] X16_s' ;  T[:, > 16 (s + 1)] -= P_s Pt_s(rows below)' .  The 64x64 inverse of r1 (P2b and
// half of P3 of factor_and_invert_64) is gone from the serial chain, and consumers start after the FIRST 16 columns.
constexpr int kPS = 84;                  // packet row stride in shared memory (84 = 4 mod 16: fragment loads conflict-free)
constexpr int kPacket = 16 * kPS;        // doubles per packet in shared memory
constexpr int kPacketG = 16 * 80;        // doubles per packet in global memory (dense rows of 80)

// pub(s): called by the threads of warps 1..7 (tid >= 32) right after the panel of step s is complete (s < 3), i.e.
//         while warp 0 runs the look-ahead + pivot chain of step s + 1;
// pub_last(): called by ALL threads when the last pivot chain (step 3, no panel below) is done;
// side(s): as in factor_and_invert_64.
template <class Pub, class PubLast, class Side>
__device__ __forceinline__ bool factor_64_pipe(double* D, double* Pk, double* L16t, double* rdiag, int* s_bad, Pub pub,
                                               PubLast pub_last, Side side) {
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int g = lane >> 2, q = lane & 3;
  if (tid == 0) *s_bad = 0;
  __syncthreads();
  if (warp == 0) factor_p1_warp<kPS>(D, L16t, Pk + 64, rdiag, s_bad, 0, lane);
  else side(0);
  __syncthreads();
#pragma unroll 1
  for (int s = 0; s < 3; ++s) {
    const int c0 = 16 * s;
    FCLK(s, 0);
    double* Pt = Pk + s * kPacket;        // [16][kPS]: cols 0..63 panel (transposed), cols 64..79 XT16_s
    const double* XT16 = Pt + 64;
    {
      // P2a: panel rows below the diagonal block, one 8-row fragment (both 8-column fragments) per warp
      const int n_a = (48 - c0) >> 3;
      if (warp < n_a) {
        const int i0 = c0 + 16 + 8 * warp;
        const double* pa = D + (i0 + g) * kTS + c0 + q;   // A[i0 + g][k0 + q]
        const double* pb = XT16 + q * kPS + g;            // B[k0 + q][n0 + g] = X16[n0 + g][k0 + q]
        double2 cl = make_double2(0.0, 0.0), ch = make_double2(0.0, 0.0);
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) {
          const double av = pa[4 * kk];
          if (kk < 2)                                      // X16 is lower triangular: k <= n
            asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};"
                         : "+d"(cl.x), "+d"(cl.y) : "d"(av), "d"(pb[4 * kk * kPS]));
          asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};"
                       : "+d"(ch.x), "+d"(ch.y) : "d"(av), "d"(pb[4 * kk * kPS + 8]));
        }
        Pt[(2 * q) * kPS + i0 + g] = cl.x;
        Pt[(2 * q + 1) * kPS + i0 + g] = cl.y;
        Pt[(8 + 2 * q) * kPS + i0 + g] = ch.x;
        Pt[(8 + 2 * q + 1) * kPS + i0 + g] = ch.y;
      }
    }
    FCLK(s, 1);
    __syncthreads();
    FCLK(s, 2);
    // P3 (D(rows >= c0+16, cols >= c0+16) -= P P', lower fragments) overlapped with the pivot chain of the next step:
    // warp 0 updates the three fragments of the next 16x16 diagonal block first and starts P1 at once; the other warps
    // publish the packet (consumers are waiting for it), finish the update, then run the side job.
    const int rt0 = (c0 + 16) >> 3;
    if (warp == 0) {
      double* cp0 = D + (8 * rt0 + g) * kTS + 8 * rt0 + 2 * q;
      double* cp1 = cp0 + 8 * kTS;      // (rt0 + 1, rt0)
      double* cp2 = cp1 + 8;            // (rt0 + 1, rt0 + 1)
      double2 v0 = *reinterpret_cast<const double2*>(cp0), v1 = *reinterpret_cast<const double2*>(cp1),
              v2 = *reinterpret_cast<const double2*>(cp2);
      const double* pp = Pt + q * kPS + 8 * rt0 + g;
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) {
        const double p0 = pp[4 * kk * kPS], p1 = pp[4 * kk * kPS + 8];
        const double a0 = -p0, a1 = -p1;
        asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};"
                     : "+d"(v0.x), "+d"(v0.y) : "d"(a0), "d"(p0));
        asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};"
                     : "+d"(v1.x), "+d"(v1.y) : "d"(a1), "d"(p0));
        asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};"
                     : "+d"(v2.x), "+d"(v2.y) : "d"(a1), "d"(p1));
      }
      *reinterpret_cast<double2*>(cp0) = v0;
      *reinterpret_cast<double2*>(cp1) = v1;
      *reinterpret_cast<double2*>(cp2) = v2;
      __syncwarp();
      factor_p1_warp<kPS>(D, L16t, Pk + (s + 1) * kPacket + 64, rdiag, s_bad, c0 + 16, lane);
    } else {
      pub(s);
      FCLK(s, 4);
      // fragment column ct = warp (warp 7 also column 0 ... only columns >= rt0 hold D entries to update)
      for (int ct = rt0 + (warp - 1); ct < 8; ct += 7) {
        int first = ct;  // lower fragments: rt >= ct
        if (ct == rt0 || ct == rt0 + 1) first = rt0 + 2;  // (rt0,rt0), (rt0+1,rt0), (rt0+1,rt0+1) are warp 0's
        if (first >= 8) continue;
        const double* pb = Pt + q * kPS + 8 * ct + g;
        double bv[4];
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) bv[kk] = pb[4 * kk * kPS];
        for (int rt = first; rt < 8; ++rt) {
          double* cp = D + (8 * rt + g) * kTS + 8 * ct + 2 * q;
          double2 cv = *reinterpret_cast<const double2*>(cp);
          const double* pa = Pt + q * kPS + 8 * rt + g;
#pragma unroll
          for (int kk = 0; kk < 4; ++kk) {
            const double a0 = -pa[4 * kk * kPS];
            asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};"
                         : "+d"(cv.x), "+d"(cv.y) : "d"(a0), "d"(bv[kk]));
          }
          *reinterpret_cast<double2*>(cp) = cv;
        }
      }
      side(s + 1);
    }
    FCLK(s, 3);
    __syncthreads();
  }
  FCLK(3, 0);
  pub_last();
  FCLK(3, 1);
  return *s_bad == 0;
}

// x = L^-1 v (forward, FWD) or x = L^-T v (backward) for the factored 64x64 block kept as its four packets:
// 16-wide substitution with the explicit 16x16 inverses.  v (shared, 64) is overwritten by x.  All 256 threads call.
template <bool FWD>
__device__ __forceinline__ void block_solve_packets(const double* Pk, double* v, double* x16, int tid) {
  const int lane4 = tid & 3, r4 = tid >> 2;  // 4 lanes per output
#pragma unroll 1
  for (int it = 0; it < 4; ++it) {
    const int s = FWD ? it : 3 - it;
    const double* Pt = Pk + s * kPacket;
    const double* XT = Pt + 64;
    if (tid < 64) {
      // x_s[n] : FWD  sum_{k <= n} X16[n][k] v[16 s + k] = sum_k XT[k][n] v[..]
      //          BWD  sum_{m >= n} X16[m][n] v[16 s + m] = sum_m XT[n][m] v[..]
      const int n = r4;
      double acc = 0.0;
#pragma unroll
      for (int k = lane4; k < 16; k += 4) {
        const double xe = FWD ? (k <= n ? XT[k * kPS + n] : 0.0) : (k >= n ? XT[n * kPS + k] : 0.0);
        acc = fma(xe, v[16 * s + k], acc);
      }
      acc += __shfl_xor_sync(0xffffffffu, acc, 1);
      acc += __shfl_xor_sync(0xffffffffu, acc, 2);
      if (lane4 == 0) x16[n] = acc;
    }
    __syncthreads();
    if (FWD) {
      // v[row] -= sum_k L[row][16 s + k] x_s[k]   for row >= 16 (s + 1)
      const int row = r4;
      double acc = 0.0;
      if (row >= 16 * (s + 1)) {
#pragma unroll
        for (int k = lane4; k < 16; k += 4) acc = fma(Pt[k * kPS + row], x16[k], acc);
      }
      acc += __shfl_xor_sync(0xffffffffu, acc, 1);
      acc += __shfl_xor_sync(0xffffffffu, acc, 2);
      if (lane4 == 0) {
        if (row >= 16 * (s + 1)) v[row] -= acc;
        else if (row >= 16 * s) v[row] = x16[row - 16 * s];
      }
    } else {
      // v[16 s' + k] -= sum_{row in block s} L[row][16 s' + k] x_s[row - 16 s]   for every earlier block s' < s
      // (L[row][16 s' + k] = Pt_{s'}[k][row]);  64 outputs c = 16 s' + k, 4 lanes each over the 16 rows
      const int c = r4;
      double acc = 0.0;
      if (c < 16 * s) {
        const double* Pc = Pk + (c >> 4) * kPacket + (c & 15) * kPS + 16 * s;
#pragma unroll
        for (int m = lane4; m < 16; m += 4) acc = fma(Pc[m], x16[m], acc);
      }
      acc += __shfl_xor_sync(0xffffffffu, acc, 1);
      acc += __shfl_xor_sync(0xffffffffu, acc, 2);
      if (lane4 == 0) {
        if (c < 16 * s) v[c] -= acc;
        else if (c < 16 * (s + 1)) v[c] = x16[c - 16 * s];
      }
    }
    __syncthreads();
  }
}

// Xi = L^-1 (lower triangular, row-major, row stride kTS, upper part zeroed) of the factored 64x64 block kept as its four
// packets.  16x16 blocks: X[s][s] = X16_s ;  X[s][s'] = -X16_s * sum_{t = s'}^{s-1} L[s][t] X[t][s']  (s' < s), thread
// (a, b) = one entry of a 16x16 block.  Not on the factorisation's critical chain (see the caller).
__device__ __forceinline__ void inverse_from_packets(const double* Pk, double* Xi, int tid) {
  const int a = tid >> 4, b = tid & 15;
  for (int e = tid; e < kTile; e += 256) Xi[e] = 0.0;
  __syncthreads();
#pragma unroll
  for (int s = 0; s < 4; ++s) Xi[(16 * s + a) * kTS + 16 * s + b] = b <= a ? Pk[s * kPacket + b * kPS + 64 + a] : 0.0;  // X16_s[a][b] = XT16_s[b][a]
  __syncthreads();
  __shared__ double W[16][17];
#pragma unroll 1
  for (int s = 1; s < 4; ++s)
#pragma unroll 1
    for (int sp = s - 1; sp >= 0; --sp) {
      // W[a][b] = sum_{t = sp}^{s-1} sum_k L[16 s + a][16 t + k] X[16 t + k][16 sp + b] ;  L[row][16 t + k] = Pt_t[k][row]
      double w = 0.0;
      for (int t = sp; t < s; ++t) {
        const double* Pt = Pk + t * kPacket;
#pragma unroll
        for (int k = 0; k < 16; ++k) w = fma(Pt[k * kPS + 16 * s + a], Xi[(16 * t + k) * kTS + 16 * sp + b], w);
      }
      W[a][b] = w;
      __syncthreads();
      // X[s][sp][a][b] = -sum_{k <= a} X16_s[a][k] W[k][b]
      const double* XT = Pk + s * kPacket + 64;
      double x = 0.0;
#pragma unroll
      for (int k = 0; k < 16; ++k) x = fma(k <= a ? XT[k * kPS + a] : 0.0, W[k][b], x);
      Xi[(16 * s + a) * kTS + 16 * sp + b] = -x;
      __syncthreads();
    }
}

}  // namespace ctvio
