// Blocked two-sided Jacobi eigen-solver for the priors of streaming windows (16 <= n <= ~120): replaces the
// Eigen::SelfAdjointEigenSolver calls of marginalization_factor.cpp:240-263 for those sizes.
//
// The element-wise parallel Jacobi (marginalize.cu) pays two block-wide barriers and a pass over the whole matrix for
// every round of n/2 rotations (n - 1 rounds per sweep, each bound by one SM's shared-memory
// bandwidth).  Here the matrix is cut into 8-wide index blocks; a round pairs the blocks (round-robin tournament), ONE
// WARP per pair runs 8 rounds of 8 disjoint rotations on its private 16x16 sub-matrix - every (p in I, q in J) pair
// once - and accumulates them into a 16x16 orthogonal Q; then the whole matrix is updated ONCE per block round as
// A <- Q' A Q with the fp64 tensor-core path (DMMA), block pair by block pair, lower pair-blocks only (the matrix is
// symmetric; the diagonal pair-blocks are the warps' own sub-matrices).  One "within" round per sweep covers the
// (p, q) pairs inside each 8-block, so a sweep visits every index pair exactly once, like the classical cyclic method
// (same number of sweeps), with nb + 1 block-wide phases instead of n - 1.
// Eigenvectors: the Qs are logged; `jacobi_blocked_apply_kernel` (one CTA per 8 rows of V) replays them on rows of the
// identity with DMMA (the rows of V transform independently).
// Rotation order and every sum are fixed: bit-reproducible.
#include <cuda_runtime.h>

#include <cstdint>

#include "kernels.h"
#include "marginalize.h"

namespace ctvio {
namespace {

constexpr int kLdQ = 24;    // row stride of the 16x16 Q / T scratch tiles (== 8 mod 16: conflict-free fragment loads)
constexpr int kLdS = 20;    // row stride of a pair problem's 16x16 working matrix (== 4 mod 16: the 2x2-block accesses of a
                            // half-warp, rows k = 0..3 x columns l = 0..3, hit 16 different 8-byte banks; 17 was 4-way conflicted
                            // and made the inner rounds shared-memory bound)
constexpr int kWarps = 16;  // warps of the eigenvalue kernel

// 1/sqrt(x) to working precision: hardware seed (~2^-22) + ONE third-order step (error ~ e^3)
__device__ __forceinline__ double rsqrt_seed3(double x) {
  double y;
  asm("rsqrt.approx.ftz.f64 %0, %1;" : "=d"(y) : "d"(x));
  const double e = fma(-(y * y), x, 1.0);
  return fma(fma(e, 0.375, 0.5), y * e, y);
}

// Jacobi rotation of the 2x2 problem [app apq; apq aqq]: column update  x_p' = c x_p - s x_q,  x_q' = s x_p + c x_q
// zeroes a_pq with |phi| <= pi/4.  With d = aqq - app, o = 2 apq, r = hypot(d, o):  cos 2phi = |d| / r,
// c = sqrt((1 + cos 2phi) / 2),  s = sin 2phi / (2 c) = sign(d) o / (2 r c): two reciprocal square roots, no division
// (the textbook t = sign(theta) / (|theta| + sqrt(theta^2 + 1)) form needs two divisions and two square roots on the
// serial path of every round).
__device__ __forceinline__ void rotation(double app, double aqq, double apq, double& c, double& s) {
  const double d = aqq - app, o = apq + apq;
  const double r2 = fma(d, d, o * o);
  c = 1.0;
  s = 0.0;
  if (o != 0.0 && r2 > 1e-280 && r2 < 1e280) {
    const double ir = rsqrt_seed3(r2);
    const double c2 = fma(0.5, fabs(d) * ir, 0.5);
    const double ic = rsqrt_seed3(c2);
    c = c2 * ic;
    s = copysign(0.5, d) * o * ir * ic;
  }
}

// pair k of round rr of the round-robin tournament on m (even) players, ascending
__device__ __forceinline__ void rr_pair(int m, int rr, int k, int& a, int& b) {
  int x, y;
  if (k == 0) { x = m - 1; y = rr; }
  else { x = (rr + k) % (m - 1); y = (rr + m - 1 - k) % (m - 1); }
  a = min(x, y);
  b = max(x, y);
}
// block pair k of block round `br` of a sweep: br == 0 is the "within" round (blocks 2k, 2k+1 side by side, rotations
// inside each block only), br >= 1 the tournament round br - 1
__device__ __forceinline__ void block_pair(int nb, int br, int k, int& I, int& J) {
  if (br == 0) { I = 2 * k; J = 2 * k + 1; }
  else rr_pair(nb, br - 1, k, I, J);
}
// rotation pair i (0..7) of inner round t on the 16 local indices
__device__ __forceinline__ void inner_pair(bool within, int t, int i, int& p, int& q) {
  if (within) {  // tournament on 8 inside each half: pairs 0..3 first block, 4..7 second
    int a, b;
    rr_pair(8, t, i & 3, a, b);
    const int o = (i & 4) ? 8 : 0;
    p = a + o;
    q = b + o;
  } else {
    p = i;
    q = 8 + ((i + t) & 7);
  }
}

__device__ __forceinline__ void dmma(double& c0, double& c1, double a, double b) {
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};"
               : "+d"(c0), "+d"(c1)
               : "d"(a), "d"(b));
}

// barrier of the two warps that share a pair problem
__device__ __forceinline__ void pair_barrier(int id) { asm volatile("bar.sync %0, 64;" ::"r"(id) : "memory"); }

// One pass of rotations over a 16x16 pair problem: WITHIN = the pairs inside each 8-block (7 rounds), else every
// (p in first block, q in second block) pair (8 rounds).  S: [16][kLdS] symmetric working matrix, Q: [16][kLdQ]
// accumulated rotations.  Run by two warps (half = 0 / 1).  Lane layout: rotation of pair (lane & 7); 2x2 block
// (k, l) = (lane >> 2, (lane & 3) + 4 half) of S; rows (lane >> 3) + 4 (2 half + {0, 1}) of Q for pair (lane & 7).
template <bool WITHIN>
__device__ __forceinline__ void inner_rounds(double* S, double* Q, int lane, int half, int bar_id) {
  const int i = lane & 7, k = lane >> 2, l = (lane & 3) + 4 * half;
  const int a0 = (lane >> 3) + 8 * half, a1 = a0 + 4;
#pragma unroll
  for (int t = 0; t < (WITHIN ? 7 : 8); ++t) {
    int p, q, pk, qk, pl, ql;
    inner_pair(WITHIN, t, i, p, q);
    inner_pair(WITHIN, t, k, pk, qk);
    inner_pair(WITHIN, t, l, pl, ql);
    double c, s;
    rotation(S[p * kLdS + p], S[q * kLdS + q], S[p * kLdS + q], c, s);
    const double qp0 = Q[a0 * kLdQ + p], qq0 = Q[a0 * kLdQ + q], qp1 = Q[a1 * kLdQ + p], qq1 = Q[a1 * kLdQ + q];
    const double b00 = S[pk * kLdS + pl], b01 = S[pk * kLdS + ql], b10 = S[qk * kLdS + pl], b11 = S[qk * kLdS + ql];
    const double ck = __shfl_sync(0xffffffffu, c, k), sk = __shfl_sync(0xffffffffu, s, k);
    const double cl = __shfl_sync(0xffffffffu, c, l), sl = __shfl_sync(0xffffffffu, s, l);
    const double t00 = cl * b00 - sl * b01, t01 = sl * b00 + cl * b01;
    const double t10 = cl * b10 - sl * b11, t11 = sl * b10 + cl * b11;
    const double r00 = ck * t00 - sk * t10, r10 = sk * t00 + ck * t10;
    const double r01 = ck * t01 - sk * t11, r11 = sk * t01 + ck * t11;
    pair_barrier(bar_id);  // both warps have read their rotation inputs and blocks
    Q[a0 * kLdQ + p] = c * qp0 - s * qq0;
    Q[a0 * kLdQ + q] = s * qp0 + c * qq0;
    Q[a1 * kLdQ + p] = c * qp1 - s * qq1;
    Q[a1 * kLdQ + q] = s * qp1 + c * qq1;
    const bool own = k == l;  // the rotated pair's own off-diagonal entry is zero by construction: exact zero
    S[pk * kLdS + pl] = r00;
    S[pk * kLdS + ql] = own ? 0.0 : r01;
    S[qk * kLdS + pl] = own ? 0.0 : r10;
    S[qk * kLdS + ql] = r11;
    pair_barrier(bar_id);
  }
}

}  // namespace

__device__ int g_jacobi_blocked_dbg[8];

// log layout: [0] int rounds (block rounds executed) ... 64 bytes header, then rounds x npairs x 256 doubles (Q row-major)
__global__ void __launch_bounds__(kWarps * 32) jacobi_blocked_kernel(const double* __restrict__ Ag, double* ev, double* qlog,
                                                                     int* log_rounds, int n, int nb, int max_sweeps) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int tid = threadIdx.x, nt = blockDim.x, warp = tid >> 5, lane = tid & 31;
  const int N = 8 * nb, npairs = nb / 2, lda = N + 4;
  double* A = reinterpret_cast<double*>(smem_raw);      // [N][lda], both triangles maintained
  double* Qs = A + size_t(N) * lda;                     // [npairs][16][kLdQ]
  double* Ss = Qs + size_t(npairs) * 16 * kLdQ;         // [npairs][16][kLdS] (+ pad)
  double* Ts = Ss + size_t(npairs) * (16 * kLdS);   // [kWarps][16][kLdQ]
  __shared__ double s_red[2][kWarps];
  __shared__ double s_off, s_diag, s_prev;
  __shared__ int s_pair[8][2];  // block pair (I, J) of pair-problem w in the current block round
  for (int e = tid; e < N * N; e += nt) {
    const int i = e / N, j = e - i * N;
    A[i * lda + j] = (i < n && j < n) ? Ag[size_t(i) * n + j] : 0.0;
  }
  __syncthreads();
  const int g = lane >> 2, q4 = lane & 3;
  int rounds_done = 0, sweeps_done = 0;
  long long cyc[4] = {0, 0, 0, 0};  // warp 0: inner solves | wait | update | wait (tools/eig_timing.py)
  for (int sweep = 0; sweep < max_sweeps; ++sweep) {
    // ---- convergence: off-diagonal vs diagonal mass (fixed summation order) ----
    double off = 0, dg = 0;
    for (int e = tid; e < N * N; e += nt) {
      const int i = e / N, j = e - i * N;
      const double v = A[i * lda + j];
      if (i == j) dg = fma(v, v, dg); else off = fma(v, v, off);
    }
    for (int o = 16; o > 0; o >>= 1) {
      off += __shfl_xor_sync(0xffffffffu, off, o);
      dg += __shfl_xor_sync(0xffffffffu, dg, o);
    }
    if (lane == 0) { s_red[0][warp] = off; s_red[1][warp] = dg; }
    __syncthreads();
    if (tid == 0) {
      double a = 0, b = 0;
      for (int w = 0; w < kWarps; ++w) { a += s_red[0][w]; b += s_red[1][w]; }
      s_prev = sweep > 0 ? s_off : 1e300;
      s_off = a;
      s_diag = b;
    }
    __syncthreads();
    // converged, or stagnating at the rounding floor; stopping earlier is not an option: the eps = 1e-30 pseudo-inverse
    // of the reference inverts the smallest eigenvalues, so their relative accuracy matters
    if (s_off <= 1e-60 || s_off <= 1e-30 * s_diag || (s_off <= 1e-24 * s_diag && s_off > 0.5 * s_prev)) break;
    ++sweeps_done;
    for (int br = 0; br < nb; ++br) {
      const bool within = br == 0;
      const long long c0 = clock64();
      // ---- phase 1: warps 2w, 2w+1 diagonalise (one pass over its 64 / 56 index pairs) the 16x16 sub-matrix of block
      //      pair w: both compute the 8 rotations of an inner round, each applies them to half of the 2x2 blocks of S
      //      and to half of the rows of Q; they meet at a named barrier (id 1 + w) twice per inner round ----
      if (warp < 2 * npairs) {
        const int pr = warp >> 1, half = warp & 1;
        int I, J;
        block_pair(nb, br, pr, I, J);
        if (half == 0 && lane == 0) { s_pair[pr][0] = I; s_pair[pr][1] = J; }
        double* S = Ss + size_t(pr) * (16 * kLdS);
        double* Q = Qs + size_t(pr) * 16 * kLdQ;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int e = lane + 32 * (j + 4 * half), a = e >> 4, b = e & 15;
          const int ga = a < 8 ? 8 * I + a : 8 * J + a - 8, gb = b < 8 ? 8 * I + b : 8 * J + b - 8;
          S[a * kLdS + b] = A[ga * lda + gb];
          Q[a * kLdQ + b] = a == b ? 1.0 : 0.0;
        }
        pair_barrier(1 + pr);
        if (within) inner_rounds<true>(S, Q, lane, half, 1 + pr);
        else inner_rounds<false>(S, Q, lane, half, 1 + pr);
        // results: the diagonal pair-block of A, and Q into the log
        double* ql_out = qlog + (size_t(rounds_done) * npairs + pr) * 256;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int e = lane + 32 * (j + 4 * half), a = e >> 4, b = e & 15;
          const int ga = a < 8 ? 8 * I + a : 8 * J + a - 8, gb = b < 8 ? 8 * I + b : 8 * J + b - 8;
          A[ga * lda + gb] = S[a * kLdS + b];
          ql_out[e] = Q[a * kLdQ + b];
        }
      }
      ++rounds_done;
      const long long c1 = clock64();
      __syncthreads();
      const long long c2 = clock64();
      // ---- phase 2: A[P_k, P_l] <- Q_k' A[P_k, P_l] Q_l for the pair-blocks k > l (and the mirror block) ----
      {
        double* T = Ts + size_t(warp) * 16 * kLdQ;
        const int npb = npairs * (npairs - 1) / 2;
        for (int pb = warp; pb < npb; pb += kWarps) {
          int k = 1, rem = pb;
          while (rem >= k) { rem -= k; ++k; }
          const int l = rem;  // 0 <= l < k
          const int Ik = s_pair[k][0], Jk = s_pair[k][1], Il = s_pair[l][0], Jl = s_pair[l][1];
          const double* Qk = Qs + size_t(k) * 16 * kLdQ;
          const double* Ql = Qs + size_t(l) * 16 * kLdQ;
          const int rb[2] = {8 * Ik, 8 * Jk}, cb[2] = {8 * Il, 8 * Jl};
          double av[2][4], bv[4][2], acc[2][2][2];
          // T = A[R, C] * Q_l
#pragma unroll
          for (int mt = 0; mt < 2; ++mt)
#pragma unroll
            for (int s = 0; s < 4; ++s) av[mt][s] = A[(rb[mt] + g) * lda + cb[s >> 1] + 4 * (s & 1) + q4];
#pragma unroll
          for (int s = 0; s < 4; ++s)
#pragma unroll
            for (int c = 0; c < 2; ++c) bv[s][c] = Ql[(4 * s + q4) * kLdQ + 8 * c + g];
#pragma unroll
          for (int mt = 0; mt < 2; ++mt)
#pragma unroll
            for (int c = 0; c < 2; ++c) {
              acc[mt][c][0] = acc[mt][c][1] = 0.0;
#pragma unroll
              for (int s = 0; s < 4; ++s) dmma(acc[mt][c][0], acc[mt][c][1], av[mt][s], bv[s][c]);
            }
#pragma unroll
          for (int mt = 0; mt < 2; ++mt)
#pragma unroll
            for (int c = 0; c < 2; ++c)
              *reinterpret_cast<double2*>(&T[(8 * mt + g) * kLdQ + 8 * c + 2 * q4]) = make_double2(acc[mt][c][0], acc[mt][c][1]);
          __syncwarp();
          // A' = Q_k' * T
#pragma unroll
          for (int mt = 0; mt < 2; ++mt)
#pragma unroll
            for (int s = 0; s < 4; ++s) av[mt][s] = Qk[(4 * s + q4) * kLdQ + 8 * mt + g];
#pragma unroll
          for (int s = 0; s < 4; ++s)
#pragma unroll
            for (int c = 0; c < 2; ++c) bv[s][c] = T[(4 * s + q4) * kLdQ + 8 * c + g];
#pragma unroll
          for (int mt = 0; mt < 2; ++mt)
#pragma unroll
            for (int c = 0; c < 2; ++c) {
              acc[mt][c][0] = acc[mt][c][1] = 0.0;
#pragma unroll
              for (int s = 0; s < 4; ++s) dmma(acc[mt][c][0], acc[mt][c][1], av[mt][s], bv[s][c]);
            }
#pragma unroll
          for (int mt = 0; mt < 2; ++mt)
#pragma unroll
            for (int c = 0; c < 2; ++c) {
              const int r = rb[mt] + g, cc = cb[c] + 2 * q4;
              A[r * lda + cc] = acc[mt][c][0];
              A[r * lda + cc + 1] = acc[mt][c][1];
              A[cc * lda + r] = acc[mt][c][0];
              A[(cc + 1) * lda + r] = acc[mt][c][1];
            }
          __syncwarp();  // T is reused by the next pair-block of this warp
        }
      }
      const long long c3 = clock64();
      __syncthreads();
      cyc[0] += c1 - c0; cyc[1] += c2 - c1; cyc[2] += c3 - c2; cyc[3] += clock64() - c3;
    }
  }
  for (int i = tid; i < n; i += nt) ev[i] = A[i * lda + i];
  if (tid == 0) {
    *log_rounds = rounds_done;
    g_jacobi_blocked_dbg[0] = sweeps_done;
    g_jacobi_blocked_dbg[1] = n;
    g_jacobi_blocked_dbg[2] = int(-log10(fmax(s_off / fmax(s_diag, 1e-300), 1e-300)));
    g_jacobi_blocked_dbg[3] = rounds_done;
    for (int i = 0; i < 4; ++i) g_jacobi_blocked_dbg[4 + i] = int(cyc[i] / max(rounds_done, 1));
  }
}

// V = product of the logged block rotations.  CTA b owns rows 8b .. 8b+7 of V (a slab of the identity), warp k applies
// the Q of block pair k of every round to the slab's 16 columns of that pair: slab[:, P_k] <- slab[:, P_k] Q_k
// (8x16 by 16x16: 8 DMMAs).  The next round's Q fragments are already in flight while the current ones are used.
__global__ void __launch_bounds__(256) jacobi_blocked_apply_kernel(const double* __restrict__ qlog, const int* log_rounds, int n,
                                                                   int nb, double* Vg) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int N = 8 * nb, npairs = nb / 2, ldv = N + 4;
  double* slab = reinterpret_cast<double*>(smem_raw);  // [8][ldv]
  const int tid = threadIdx.x, nt = blockDim.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, q4 = lane & 3;
  const int r0 = 8 * blockIdx.x;
  for (int e = tid; e < 8 * N; e += nt) {
    const int i = e / N, j = e - i * N;
    slab[i * ldv + j] = (r0 + i == j) ? 1.0 : 0.0;
  }
  const int rounds = *log_rounds;
  double bv[4][2], bn[4][2];
  auto load_q = [&](int round, double (&dst)[4][2]) {
    const double* Q = qlog + (size_t(round) * npairs + warp) * 256;
#pragma unroll
    for (int s = 0; s < 4; ++s)
#pragma unroll
      for (int c = 0; c < 2; ++c) dst[s][c] = __ldg(&Q[(4 * s + q4) * 16 + 8 * c + g]);
  };
  if (warp < npairs && rounds > 0) load_q(0, bv);
  __syncthreads();
  for (int round = 0; round < rounds; ++round) {
    if (warp < npairs) {
      if (round + 1 < rounds) load_q(round + 1, bn);
      int I, J;
      block_pair(nb, round % nb, warp, I, J);
      const int cb[2] = {8 * I, 8 * J};
      double av[4], acc[2][2];
#pragma unroll
      for (int s = 0; s < 4; ++s) av[s] = slab[g * ldv + cb[s >> 1] + 4 * (s & 1) + q4];
#pragma unroll
      for (int c = 0; c < 2; ++c) {
        acc[c][0] = acc[c][1] = 0.0;
#pragma unroll
        for (int s = 0; s < 4; ++s) dmma(acc[c][0], acc[c][1], av[s], bv[s][c]);
      }
      __syncwarp();
#pragma unroll
      for (int c = 0; c < 2; ++c) {
        slab[g * ldv + cb[c] + 2 * q4] = acc[c][0];
        slab[g * ldv + cb[c] + 2 * q4 + 1] = acc[c][1];
      }
#pragma unroll
      for (int s = 0; s < 4; ++s)
#pragma unroll
        for (int c = 0; c < 2; ++c) bv[s][c] = bn[s][c];
    }
    __syncthreads();
  }
  for (int e = tid; e < 8 * n; e += nt) {
    const int i = e / n, j = e - i * n;
    if (r0 + i < n) Vg[size_t(r0 + i) * n + j] = slab[i * ldv + j];
  }
}

static int blocked_nb(int n) {
  int nb = (n + 7) / 8;
  if (nb & 1) ++nb;
  return nb;
}
static size_t blocked_smem(int nb) {
  const int N = 8 * nb, npairs = nb / 2;
  return (size_t(N) * (N + 4) + size_t(npairs) * 16 * kLdQ + size_t(npairs) * (16 * kLdS) + size_t(kWarps) * 16 * kLdQ) *
         sizeof(double);
}
bool jacobi_blocked_fits(int n) { return n >= 16 && blocked_nb(n) <= 16 && blocked_smem(blocked_nb(n)) <= size_t(224) * 1024; }
size_t jacobi_blocked_log_bytes(int n, int max_sweeps) {
  if (!jacobi_blocked_fits(n)) return 0;
  const int nb = blocked_nb(n);
  return 64 + size_t(max_sweeps) * nb * (nb / 2) * 256 * sizeof(double);
}
int launch_jacobi_blocked(const double* A, double* V, double* ev, int n, void* log_buf, int max_sweeps, cudaStream_t s) {
  const int nb = blocked_nb(n);
  const size_t smem = blocked_smem(nb);
  static PerDeviceOnce once;
  if (once.first()) cudaFuncSetAttribute(jacobi_blocked_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 224 * 1024);
  int* rounds = reinterpret_cast<int*>(log_buf);
  double* qlog = reinterpret_cast<double*>(reinterpret_cast<unsigned char*>(log_buf) + 64);
  jacobi_blocked_kernel<<<1, kWarps * 32, smem, s>>>(A, ev, qlog, rounds, n, nb, max_sweeps);
  jacobi_blocked_apply_kernel<<<nb, 256, size_t(8) * (8 * nb + 4) * sizeof(double), s>>>(qlog, rounds, n, nb, V);
  return 2;
}

extern "C" int ctvio_debug_jacobi_blocked(int* out8) {
  return cudaMemcpyFromSymbol(out8, g_jacobi_blocked_dbg, sizeof(g_jacobi_blocked_dbg)) == cudaSuccess ? 0 : -1;
}

}  // namespace ctvio

// Test hook (not part of include/ctvio.h): eigen-decomposition of a host matrix through the same launcher the
// marginalization uses.  A: [n][n] symmetric row-major; V: [n][n] eigenvectors in columns; ev: [n].
extern "C" int ctvio_debug_eig(int n, const double* A, double* V, double* ev, int device) {
  if (n <= 0 || !A || !V || !ev) return -1;
  if (cudaSetDevice(device) != cudaSuccess) return -2;
  double *dA = nullptr, *dV = nullptr, *dev_ = nullptr;
  void* log = nullptr;
  const size_t nn = size_t(n) * n * sizeof(double);
  int rc = 0;
  if (cudaMalloc(&dA, nn) != cudaSuccess || cudaMalloc(&dV, nn) != cudaSuccess || cudaMalloc(&dev_, n * sizeof(double)) != cudaSuccess ||
      cudaMalloc(&log, ctvio::jacobi_log_bytes(n, 40)) != cudaSuccess)
    rc = -3;
  if (!rc) {
    cudaMemcpy(dA, A, nn, cudaMemcpyHostToDevice);
    cudaMemset(dV, 0, nn);
    ctvio::launch_jacobi_eig(dA, dV, dev_, n, log, 0);
    if (cudaGetLastError() != cudaSuccess) rc = -5;
    if (cudaDeviceSynchronize() != cudaSuccess) rc = -4;
    cudaMemcpy(V, dV, nn, cudaMemcpyDeviceToHost);
    cudaMemcpy(ev, dev_, n * sizeof(double), cudaMemcpyDeviceToHost);
  }
  cudaFree(dA); cudaFree(dV); cudaFree(dev_); cudaFree(log);
  return rc;
}
