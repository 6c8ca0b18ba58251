// K5 (fast path): tile-DAG Cholesky + both triangular solves of the reduced camera system in ONE persistent
// kernel WITHOUT grid-wide barriers.  Replaces the factor/solve half of Ceres' SPARSE_NORMAL_CHOLESKY step
// (estimator/trajectory_estimator.cpp:374; Ceres itself is not part of the reference repository) on the Schur-reduced system.
//
// Owner computes: every 64x64 tile (i, j), i >= j, of the lower triangle has ONE owner CTA that keeps the tile in
// tensor-core fragments from the first to the last update, so the trailing matrix is never re-read or re-written in HBM.
//   * diagonal CTA j: tile (j, j).  Applies the SYRK updates of the finished tiles L(j,k), factors the block 16 columns
//     at a time (pivot chain in one warp) WITHOUT forming its 64x64 inverse, and publishes a PACKET per 16 columns
//     (the panel below the 16x16 diagonal block + that block's 16x16 inverse, which the pivot warp's idle lanes get for free).
//   * tile CTA (i, j), i > j: applies its GEMM updates, then runs the right-looking triangular solve against block column
//     j IN STEP with its factorisation (one packet = 16 columns of L(i,j)); the sub-diagonal CTA (j+1, j) streams each
//     finished 16-column slab to diagonal CTA j+1, which applies it as a rank-16 update: when the last pivot of column j
//     is done, one 16x16 product, one slab hop and one rank-16 update separate it from the first pivot of column j+1.
// r2 changes vs r1: no 64x64 inverse on the chain (was ~half of the diagonal
// factor), solve pipelined with the factorisation, the chain's GEMM work split over two SMs per column (r1: one), and
// the chain's messages are SELF-VALIDATING WORDS (sentinel = not yet written) instead of store + fence + flag + acquire.
// Tiles that feed later GEMM updates still use release/acquire flags in global memory (epoch valued: never cleared).
// The forward substitution is folded in: the owner of (i,k) publishes L(i,k) x_k, the diagonal CTA i sums those
// partials in a FIXED order (bit-reproducible, required by the replicated solve of the sharded mode); the backward
// sweep reuses the tiles still resident in shared memory: owner (r,k) publishes L(r,k)^T x_r.
// Needs nb (nb + 1) / 2 <= #SMs (all CTAs co-resident: cooperative launch); launch_factor_solve falls back to the
// barrier kernel (chol_coop.cu) otherwise.
#include <algorithm>
#include <atomic>
#include <cstdlib>

#include "chol_tiles.cuh"
#include "dmma_tiles.cuh"
#include "kernels.h"

namespace ctvio {

namespace {

// ---- self-validating words: packets of the diagonal factorisations travel WITHOUT flag + fence ----
// A packet word is either the sentinel (a negative quiet NaN with a payload no arithmetic produces) or final data; 8-byte
// accesses are single-copy atomic, so a consumer spins on the data itself: ONE L2 round trip per hop instead of
// store -> fence -> flag -> acquire -> load.  Two buffers alternate by the engine's launch parity; a producer resets its
// slots of the OTHER buffer at the end of a launch (nobody reads that buffer during this launch), so the next launch
// finds sentinels.  (A NaN in the data - non-positive pivot - is the default qNaN, never the sentinel: no deadlock.)
constexpr unsigned long long kSentinel = 0xFFF8C0DEC0DE0001ull;
// ---- thread-block cluster / distributed shared memory (the two hops per block column of the critical chain) ----
// Chain positions p = 0, 1, 2, ... = diag 0, tile (1,0), diag 1, tile (2,1), ... are consecutive CTAs, so position p + 1
// sits in the same cluster unless p + 1 is a multiple of the cluster size: the producer then writes its message words
// straight into the consumer's shared memory (st.shared::cluster), the consumer spins on its OWN shared memory
// (a poll of local shared memory instead of an L2 round trip).  Same self-validating words:
// the consumer fills its receive area with sentinels, then arrives at the cluster barrier; a producer waits on that
// barrier once, before its first remote store.
__device__ __forceinline__ unsigned smem_u32(const void* p) { return static_cast<unsigned>(__cvta_generic_to_shared(p)); }
__device__ __forceinline__ unsigned mapa_u32(unsigned addr, unsigned rank) {
  unsigned r;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(addr), "r"(rank));
  return r;
}
__device__ __forceinline__ void st_cluster2(unsigned addr, double2 v) {
  asm volatile("st.shared::cluster.v2.f64 [%0], {%1, %2};" ::"r"(addr), "d"(v.x), "d"(v.y) : "memory");
}
__device__ __forceinline__ double2 ld_shared_volatile2(const double* p) {
  double2 v;
  asm volatile("ld.volatile.shared.v2.f64 {%0, %1}, [%2];" : "=d"(v.x), "=d"(v.y) : "r"(smem_u32(p)) : "memory");
  return v;
}
__device__ __forceinline__ void cluster_arrive() { asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory"); }
__device__ __forceinline__ void cluster_wait() { asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory"); }
__device__ __forceinline__ unsigned cluster_ctarank() {
  unsigned r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ unsigned cluster_nctarank() {
  unsigned r;
  asm volatile("mov.u32 %0, %%cluster_nctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ bool is_sentinel(double v) { return static_cast<unsigned long long>(__double_as_longlong(v)) == kSentinel; }
__device__ __forceinline__ double2 ld_relaxed2(const double* p) {
  double2 v;
  asm volatile("ld.relaxed.gpu.global.v2.f64 {%0, %1}, [%2];" : "=d"(v.x), "=d"(v.y) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_relaxed2(double* p, double2 v) {
  asm volatile("st.relaxed.gpu.global.v2.f64 [%0], {%1, %2};" ::"l"(p), "d"(v.x), "d"(v.y) : "memory");
}

__device__ __forceinline__ double ld_relaxed1(const double* p) {
  double v;
  asm volatile("ld.relaxed.gpu.global.f64 %0, [%1];" : "=d"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_relaxed1(double* p, double v) {
  asm volatile("st.relaxed.gpu.global.f64 [%0], %1;" ::"l"(p), "d"(v) : "memory");
}
// spin until the word has been written (self-validating message word)
__device__ __forceinline__ double ld_spin(const double* p) {
  double v = ld_relaxed1(p);
  while (is_sentinel(v)) v = ld_relaxed1(p);
  return v;
}
__device__ __forceinline__ double sentinel_value() { return __longlong_as_double(static_cast<long long>(kSentinel)); }

// all threads of the CTA: wait until *flag == epoch (thread 0 spins), then make the producer's data visible
__device__ __forceinline__ void wait_flag(const int* flag, int epoch) {
  if (threadIdx.x == 0) {
    spin_until_gpu(flag, epoch);
  }
  __syncthreads();
}
// two flags at once: two polling threads in different warps, one barrier
__device__ __forceinline__ void wait_flags2(const int* f1, const int* f2, int epoch) {
  if (threadIdx.x == 0) {
    spin_until_gpu(f1, epoch);
  } else if (threadIdx.x == 32) {
    spin_until_gpu(f2, epoch);
  }
  __syncthreads();
}
// all threads have written their part of the payload; publish it
__device__ __forceinline__ void post_flag(int* flag, int epoch) {
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    st_release_gpu(flag, epoch);
  }
}

// smem tile <- 64x64 global block with row stride ld, straight copy (16-byte accesses on both sides): final tiles
// and block inverses are PUBLISHED TRANSPOSED, i.e. already in the [k][row] operand layout
__device__ __forceinline__ void load_tile_cg(double* dst, const double* src, int ld, int tid) {
#pragma unroll
  for (int e = tid; e < kCholNB * kCholNB / 2; e += 256) {
    const int r = e >> 5, c = (e & 31) * 2;
    *reinterpret_cast<double2*>(dst + r * kTS + c) = __ldcg(reinterpret_cast<const double2*>(src + size_t(r) * ld + c));
  }
}
// smem tile (stride kTS) -> global 64x64 slot (row stride ld), straight copy with 16-byte accesses
__device__ __forceinline__ void store_tile_global(double* dst, int ld, const double* src, int tid) {
#pragma unroll
  for (int e = tid; e < kCholNB * kCholNB / 2; e += 256) {
    const int r = e >> 5, c = (e & 31) * 2;
    *reinterpret_cast<double2*>(dst + size_t(r) * ld + c) = *reinterpret_cast<const double2*>(src + r * kTS + c);
  }
}
// s[tid & 63] partial: sum over q = (tid >> 6), q + 4, ... < n of part[q * stride + (tid & 63)], combined over the
// four thread groups in a fixed order through red[4][64]; returns the total for tid < 64 (after a barrier)
// (the partials are self-validating words: every load spins until its producer has written it)
__device__ __forceinline__ double sum_partials(const double* part, int n, size_t stride, double* red, int tid) {
  const int c = tid & 63, g = tid >> 6;
  double s = 0.0;
  int q = g;
  for (; q + 12 < n; q += 16) {
    double v0 = ld_relaxed1(part + size_t(q) * stride + c), v1 = ld_relaxed1(part + size_t(q + 4) * stride + c);
    double v2 = ld_relaxed1(part + size_t(q + 8) * stride + c), v3 = ld_relaxed1(part + size_t(q + 12) * stride + c);
    while (is_sentinel(v0)) v0 = ld_relaxed1(part + size_t(q) * stride + c);
    while (is_sentinel(v1)) v1 = ld_relaxed1(part + size_t(q + 4) * stride + c);
    while (is_sentinel(v2)) v2 = ld_relaxed1(part + size_t(q + 8) * stride + c);
    while (is_sentinel(v3)) v3 = ld_relaxed1(part + size_t(q + 12) * stride + c);
    s += v0; s += v1; s += v2; s += v3;
  }
  for (; q < n; q += 4) s += ld_spin(part + size_t(q) * stride + c);
  red[g * kCholNB + c] = s;
  __syncthreads();
  return tid < kCholNB ? (red[tid] + red[kCholNB + tid]) + (red[2 * kCholNB + tid] + red[3 * kCholNB + tid]) : 0.0;
}
// out[r] = sum_c Lrm[r][c] * v[c]  (Lrm row-major smem tile; 4 lanes per row); optional shared copy of the result
__device__ __forceinline__ void tile_matvec(const double* Lrm, const double* v, double* out_global, int tid,
                                            double* out_shared = nullptr) {
  const int r = tid >> 2, pt = tid & 3;
  double s = 0.0;
#pragma unroll 4
  for (int c = pt; c < kCholNB; c += 4) s = fma(Lrm[r * kTS + c], v[c], s);
  s += __shfl_xor_sync(0xffffffffu, s, 1);
  s += __shfl_xor_sync(0xffffffffu, s, 2);
  if (pt == 0) {
    st_relaxed1(out_global + r, s);
    if (out_shared) out_shared[r] = s;
  }
}
}  // namespace

// ---- masked fragment products --------------------------------------------------------------------
// f[mt][nt] -= A_frag(mt) B_frag(nt)' over nk4 k-steps of 4, for the (mt, nt) pairs of the COMPILE-TIME mask (bit 4 mt + nt).
// Which fragments a warp has to touch is warp-uniform but only known at run time (it depends on the warp's position in
// the folded fragment grid and on the 16-column step); a run-time predicate per mma.sync makes ptxas guard EVERY DMMA with
// a WARPSYNC (which made a 64x16x64 slab update several times slower).  So the run-time value selects one of a
// handful of instantiations and the inner loop is branch free.
template <unsigned MASK>
__device__ __forceinline__ void mma_masked(Frag& f, const double* pa, int sa, const double* pb, int sb, const Lane& L, int nk4) {
#pragma unroll 4
  for (int kk = 0; kk < nk4; ++kk) {
    double av[2], bv[4];
#pragma unroll
    for (int mt = 0; mt < 2; ++mt)
      if (MASK & (0xFu << (4 * mt))) av[mt] = -pa[4 * kk * sa + 8 * L.rt[mt]];
#pragma unroll
    for (int nt = 0; nt < 4; ++nt)
      if (MASK & (0x11u << nt)) bv[nt] = pb[4 * kk * sb + 8 * L.ct[nt]];
#pragma unroll
    for (int mt = 0; mt < 2; ++mt)
#pragma unroll
      for (int nt = 0; nt < 4; ++nt)
        if ((MASK >> (4 * mt + nt)) & 1u)
          asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};"
                       : "+d"(f.c[mt][nt][0]), "+d"(f.c[mt][nt][1]) : "d"(av[mt]), "d"(bv[nt]));
  }
}
__device__ __forceinline__ void mma_dispatch(unsigned mask, Frag& f, const double* pa, int sa, const double* pb, int sb,
                                             const Lane& L, int nk4) {
  switch (mask) {  // warp-uniform
    case 0x33u: mma_masked<0x33u>(f, pa, sa, pb, sb, L, nk4); break;
    case 0xCCu: mma_masked<0xCCu>(f, pa, sa, pb, sb, L, nk4); break;
    case 0xFFu: mma_masked<0xFFu>(f, pa, sa, pb, sb, L, nk4); break;
    case 0xF1u: mma_masked<0xF1u>(f, pa, sa, pb, sb, L, nk4); break;
    case 0x73u: mma_masked<0x73u>(f, pa, sa, pb, sb, L, nk4); break;
    case 0xF0u: mma_masked<0xF0u>(f, pa, sa, pb, sb, L, nk4); break;
    default: break;
  }
}
// fragments (mt, nt) with rt[mt] >= ct[nt] (lower triangle of a diagonal tile) for the folded ownership of lane_of():
// warp (wm, wn) owns fragment rows {wm, 7 - wm} and columns {0,1,6,7} (wn = 0) / {2,3,4,5} (wn = 1)
__device__ __forceinline__ unsigned lower_mask(int warp) {
  const int wm = warp & 3, wn = warp >> 2;
  if (wn == 0) return wm == 0 ? 0xF1u : wm == 1 ? 0x73u : 0x33u;
  return wm <= 1 ? 0xF0u : wm == 2 ? 0xF1u : 0x73u;
}
// fragment-column pairs of a warp by 16-column slab: wn = 0: pair 0 (nt 0,1) = slab 0, pair 1 (nt 2,3) = slab 3;
// wn = 1: pair 0 = slab 1, pair 1 = slab 2
__device__ __forceinline__ unsigned slab_mask(int warp, int s) {
  const int wn = warp >> 2;
  if (wn == 0) return s == 0 ? 0x33u : s == 3 ? 0xCCu : 0u;
  return s == 1 ? 0x33u : s == 2 ? 0xCCu : 0u;
}
// ... and the pairs that lie in slabs > s (trailing columns of a solve step)
__device__ __forceinline__ unsigned trailing_mask(int warp, int s) {
  const int wn = warp >> 2;
  if (wn == 0) return s < 3 ? 0xCCu : 0u;
  return s == 0 ? 0xFFu : s == 1 ? 0xCCu : 0u;
}

struct CholDagArgs {
  double* M;          // [npad][npad], strictly-lower tiles overwritten with L(i,j)^T (transposed inside the tile slot)
  int npad;
  double* Lpub;       // this launch's packet buffer [nb][4][16][80] (self-validating words, see kSentinel)
  double* Lpub_other; // the other parity's buffer: reset to sentinels by the producers at the end of this launch
  double* Spub;       // [nb][nb][4][16][64] slabs P_s^T of every tile (i, k) as its solve produces them (self-validating):
                      // read by diagonal CTA i (k = i - 1) and by the tiles whose last update needs L(i,k)
  double* Spub_other;
  const double* rhs;  // [npad]
  double* y;          // [npad] solution
  double* yf;         // [npad] forward-solved right-hand side
  double* part;       // messages of the two substitution sweeps, all self-validating words (this launch's parity):
                      //   fwd_part[nb][nb][64] = L(i,k) x_k | bwd_part[nb][nb][64] = L(r,k)^T x_r | xf[nb][64] | xb[nb][64]
  double* part_other; // the other parity (reset to sentinels by the writers at the end of this launch)
  int* flags;         // tile_ready[nb*nb]: L(i,k) final and written (release / acquire, epoch valued)
  int epoch;
  LmScalars* scal;
  const int32_t* go;  // speculated LM step: null or &LmDecision::go (0: every CTA returns before touching any message)
};

#ifdef CTVIO_CHOL_TIMING
__device__ unsigned long long g_dag_stamps[32 * 16];
#define DSTAMP(j, i) do { if (threadIdx.x == 0 && (j) >= 0 && (j) < 32) { unsigned long long t_; \
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t_)); g_dag_stamps[(j) * 16 + (i)] = t_; } } while (0)
extern "C" int ctvio_debug_fac_clk(long long* out) {
  return cudaMemcpyFromSymbol(out, g_fac_clk, sizeof(g_fac_clk)) == cudaSuccess ? 0 : -1;
}
extern "C" int ctvio_debug_dag_stamps(unsigned long long* out) {
  return cudaMemcpyFromSymbol(out, g_dag_stamps, sizeof(g_dag_stamps)) == cudaSuccess ? 0 : -1;
}
#else
#define DSTAMP(j, i)
#endif

// shared memory: D | S1 | S2 | Pk (4 packets) | At | Bp (2 packets) | L16t | rdiag, vec, vec2, red[4][64], x16
constexpr size_t kCholDagSmem =
    (3 * size_t(kTile) + 4 * size_t(kPacket) + 16 * size_t(kTS) + 2 * size_t(kPacket) + 256 + 7 * kCholNB + 16) * sizeof(double);

// out[r] = sum_c St[c][r] v[c]   (St = the tile TRANSPOSED, [c][r] layout: lanes run along r, conflict free).
// 4 partial sums per output (threads r, r + 64, ...) combined in a fixed order through red[4][64].
__device__ __forceinline__ void tile_matvec_t(const double* St, const double* v, double* out_global, double* red, int tid,
                                              double* out_shared = nullptr) {
  const int r = tid & 63, part = tid >> 6;
  double s = 0.0;
#pragma unroll 4
  for (int c = part; c < kCholNB; c += 4) s = fma(St[c * kTS + r], v[c], s);
  red[part * kCholNB + r] = s;
  __syncthreads();
  if (tid < kCholNB) {
    const double t = (red[tid] + red[kCholNB + tid]) + (red[2 * kCholNB + tid] + red[3 * kCholNB + tid]);
    st_relaxed1(out_global + tid, t);
    if (out_shared) out_shared[tid] = t;
  }
}

// Right-looking triangular solve of the tile held in `acc` (fragments) against block column jc, consuming the packets
// of its diagonal-block factorisation AS THEY ARE PUBLISHED (one per 16 columns):  L(i,jc) = T L_jj^-T.
// Result: S1 = L(i,jc)^T ([c][row] layout = the operand / publication layout).  slab_out != nullptr (sub-diagonal tile):
// every finished 16-column slab P_s^T is streamed to the diagonal CTA of row i as self-validating words.
// Ua / Ub != nullptr: the LAST GEMM update of the tile (operands L(i,j-1)^T, L(j,j-1)^T in [k][row] layout) is applied
// lazily, 16 output columns at a time right before the step that needs them: the solve starts one quarter of a tile
// product after its operands arrive instead of a whole one, which keeps this CTA in step with the factorisation.
__device__ __forceinline__ void trsm_pipelined(Frag& acc, const Lane& L, double* S1, double* At, double* Bp2,
                                               const double* Lpub_col, double* slab_out, const double* Ua, const double* Ub,
                                               int tid, int jstamp, const double* pk_local = nullptr, unsigned slab_remote = 0u) {
  const int warp = tid >> 5, lane = tid & 31, g = lane >> 2, q = lane & 3;
  // packet words of this thread: e = tid, tid + 256, tid + 512 of the 640 double2 of a full packet (16 rows x 40); the
  // last packet only carries the 16x16 inverse (128 double2).  Loads of packet s + 1 are IN FLIGHT while step s computes.
  int goff[3], soff[3];
#pragma unroll
  for (int u = 0; u < 3; ++u) {
    const int e = tid + 256 * u;
    const int r = e / 40, c = (e - r * 40) * 2;
    goff[u] = e < 640 ? r * 80 + c : -1;
    soff[u] = r * kPS + c;
  }
  const int goff3 = tid < 128 ? (tid >> 3) * 80 + 64 + (tid & 7) * 2 : -1, soff3 = (tid >> 3) * kPS + 64 + (tid & 7) * 2;
  double2 pre[3];
  auto issue = [&](int s) {
    if (pk_local) return;  // the packets arrive in this CTA's shared memory
    const double* src = Lpub_col + size_t(s) * kPacketG;
    if (s < 3) {
#pragma unroll
      for (int u = 0; u < 3; ++u)
        if (goff[u] >= 0) pre[u] = ld_relaxed2(src + goff[u]);
    } else if (goff3 >= 0) {
      pre[0] = ld_relaxed2(src + goff3);
    }
  };
  auto commit = [&](int s, double* Bp) {
    if (pk_local) {  // Bp IS the receive area of packet s: wait for this thread's words
      if (s < 3) {
#pragma unroll
        for (int u = 0; u < 3; ++u)
          if (goff[u] >= 0) {
            double2 v = ld_shared_volatile2(Bp + soff[u]);
            while (is_sentinel(v.x) || is_sentinel(v.y)) v = ld_shared_volatile2(Bp + soff[u]);
          }
      } else if (goff3 >= 0) {
        double2 v = ld_shared_volatile2(Bp + soff3);
        while (is_sentinel(v.x) || is_sentinel(v.y)) v = ld_shared_volatile2(Bp + soff3);
      }
      return;
    }
    const double* src = Lpub_col + size_t(s) * kPacketG;
    if (s < 3) {
#pragma unroll
      for (int u = 0; u < 3; ++u)
        if (goff[u] >= 0) {
          while (is_sentinel(pre[u].x) || is_sentinel(pre[u].y)) pre[u] = ld_relaxed2(src + goff[u]);
          *reinterpret_cast<double2*>(Bp + soff[u]) = pre[u];
        }
    } else if (goff3 >= 0) {
      while (is_sentinel(pre[0].x) || is_sentinel(pre[0].y)) pre[0] = ld_relaxed2(src + goff3);
      *reinterpret_cast<double2*>(Bp + soff3) = pre[0];
    }
  };
  issue(0);
#pragma unroll 1
  for (int s = 0; s < 4; ++s) {
    double* Bp = pk_local ? const_cast<double*>(pk_local) + s * kPacket : Bp2 + (s & 1) * kPacket;
    // lazy last update, one slab AHEAD of the solve (slab 0 and 1 before the first packet is needed, slab s + 1 while
    // packet s is in flight), so that nothing but the 16x16 product of step 3 follows the last packet
    if (Ua) {
      if (s == 0) mma_dispatch(slab_mask(warp, 0), acc, Ua + q * kTS + g, kTS, Ub + q * kTS + g, kTS, L, kCholNB / 4);
      if (s < 3) mma_dispatch(slab_mask(warp, s + 1), acc, Ua + q * kTS + g, kTS, Ub + q * kTS + g, kTS, L, kCholNB / 4);
    }
    // a. the 16 columns of step s (as updated so far) -> At[k][row]
#pragma unroll
    for (int mt = 0; mt < 2; ++mt)
#pragma unroll
      for (int nt = 0; nt < 4; ++nt) {
        const int ct = L.ct[nt];
        if ((ct >> 1) == s) {
#pragma unroll
          for (int e = 0; e < 2; ++e) At[(8 * (ct & 1) + 2 * q + e) * kTS + L.row(mt)] = acc.c[mt][nt][e];
        }
      }
    // b. packet of step s: every thread waits for ITS words (they are their own flags), then the next packet's loads go out
    DSTAMP(16 + jstamp, 4 * s + 0);
    commit(s, Bp);
    DSTAMP(16 + jstamp, 4 * s + 1);
    if (s < 3) issue(s + 1);
    __syncthreads();
    DSTAMP(jstamp, 8 + s);
    if (s == 3) DSTAMP(jstamp, 2);
    // c. P_s = A_s X16_s'  : warp w = row fragment w, both 8-column fragments -> S1 rows 16 s .. 16 s + 15 (transposed)
    {
      const double* pa = At + q * kTS + 8 * warp + g;   // A[8 w + g][k0 + q]
      const double* pb = Bp + q * kPS + 64 + g;         // B[k0 + q][n0 + g] = X16[n0 + g][k0 + q] = XT16[k0 + q][n0 + g]
      double2 cl = make_double2(0.0, 0.0), ch = make_double2(0.0, 0.0);
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) {
        const double av = pa[4 * kk * kTS];
        if (kk < 2)
          asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};"
                       : "+d"(cl.x), "+d"(cl.y) : "d"(av), "d"(pb[4 * kk * kPS]));
        asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};"
                     : "+d"(ch.x), "+d"(ch.y) : "d"(av), "d"(pb[4 * kk * kPS + 8]));
      }
      double* dst = S1 + (16 * s) * kTS + 8 * warp + g;
      dst[(2 * q) * kTS] = cl.x;
      dst[(2 * q + 1) * kTS] = cl.y;
      dst[(8 + 2 * q) * kTS] = ch.x;
      dst[(8 + 2 * q + 1) * kTS] = ch.y;
    }
    DSTAMP(16 + jstamp, 4 * s + 2);
    __syncthreads();
    if (slab_out) {  // 16 x 64 doubles = 512 double2, two per thread, straight out of S1's rows 16 s ..
#pragma unroll
      for (int u = 0; u < 2; ++u) {
        const int e = tid + 256 * u, r = e >> 5, c = (e & 31) * 2;
        const double2 v = *reinterpret_cast<const double2*>(S1 + (16 * s + r) * kTS + c);
        if (slab_remote) st_cluster2(slab_remote + unsigned(((16 * s + r) * kTS + c) * sizeof(double)), v);  // diagonal CTA's S1
        st_relaxed2(slab_out + size_t(s) * 16 * 64 + r * 64 + c, v);
      }
    }
    // d. trailing columns of the tile:  T[:, c] -= sum_k P_s[:, k] L_jj[c][16 s + k]  for c >= 16 (s + 1)
    if (s < 3)  // A = P_s^T rows (S1), B = Pt_s (packet): K = 16
      mma_dispatch(trailing_mask(warp, s), acc, S1 + (16 * s + q) * kTS + g, kTS, Bp + q * kPS + g, kPS, L, 4);
    // (Bp is double buffered and At / S1 rows are rewritten only after the next step's barrier)
    DSTAMP(16 + jstamp, 4 * s + 3);
  }
}

__global__ void __launch_bounds__(256, 1) chol_dag_kernel(CholDagArgs a) {
  extern __shared__ __align__(16) unsigned char dag_smem[];
  double* D = reinterpret_cast<double*>(dag_smem);  // column CTA: diagonal tile (row-major), destroyed by the factor
  double* S1 = D + kTile;                            // operand A ([k][row]); later the owned final tile, transposed
  double* S2 = S1 + kTile;                           // operand B ([k][row])
  double* Pk = S2 + kTile;                           // column CTA: the four packets of its own factorisation
  double* At = Pk + 4 * kPacket;                     // [16][kTS] current 16-column slab of the tile being solved
  double* Bp = At + 16 * kTS;                        // [2][16][kPS] packets being consumed (double buffered)
  double* L16t = Bp + 2 * kPacket;                   // [16][16] scratch of the pivot chain
  double* rdiag = L16t + 256;                        // [64]
  double* vec = rdiag + kCholNB;                     // [64]
  double* vec2 = vec + kCholNB;                      // [64]
  double* red = vec2 + kCholNB;                      // [4][64]
  double* x16 = red + 4 * kCholNB;                   // [16]
  __shared__ int s_bad;
  const int tid = threadIdx.x;
  const Lane L = lane_of(tid);
  const int npad = a.npad, nb = npad / kCholNB, epoch = a.epoch;
  int* tile_ready = a.flags;
  const size_t nn = size_t(nb) * nb * kCholNB;
  double* fwd_part = a.part;            // [i][k][64] = L(i,k) x_k
  double* bwd_part = a.part + nn;       // [k][r][64] = L(r,k)^T x_r
  double* xf_pub = a.part + 2 * nn;     // [j][64] forward-solved x_j
  double* xb_pub = xf_pub + size_t(nb) * kCholNB;  // [j][64] solution x_j
  const double sv = sentinel_value();
  // (go is written two launches back: read before the wait)
  const bool go = !a.go || *a.go != 0;

  // chain order: position p = blockIdx.x: p even < 2 nb - 1: diagonal CTA p / 2; p odd: sub-diagonal tile
  // ((p + 1) / 2, (p - 1) / 2); then the other tiles (i >= j + 2) column by column; then fillers (grid padded to the
  // cluster size).  Consecutive chain positions share a cluster (see the helpers above).
  const int pos = blockIdx.x, nchain = 2 * nb - 1;
  const unsigned crank = cluster_ctarank(), csize = cluster_nctarank();
  const bool dsm = csize > 1;
  const bool is_diag = pos < nchain && (pos & 1) == 0;
  const bool recv_local = dsm && pos < nchain && pos > 0 && crank != 0;        // my predecessor on the chain is in my cluster
  const bool send_remote = dsm && pos + 1 < nchain && crank + 1 < csize;       // my successor on the chain is in my cluster
  if (dsm) {
    // receive areas <- sentinels (diagonal CTA: the four slabs in S1; sub-diagonal tile: the four packets in Pk), then arrive
    if (recv_local) {
      double* area = is_diag ? S1 : Pk;
      const int n2 = (is_diag ? kTile : 4 * kPacket) / 2;
      for (int e = tid; e < n2; e += 256) *reinterpret_cast<double2*>(area + 2 * e) = make_double2(sv, sv);
    }
    __syncthreads();
    cluster_arrive();
  }
  // everything above touches this CTA's shared memory only; M and rhs come from reduced_system_kernel
  pdl_wait();
  pdl_launch_dependents();
  // speculated step behind a rejected / terminating one: nothing has been sent or reset yet, and the host takes the
  // launch out of its parity count (engine.cu)
  if (!go || (dsm && pos >= nb * (nb + 1) / 2)) {  // (or a filler CTA)
    if (dsm) cluster_wait();
    return;
  }
  if (!is_diag) {
    // ======================= tile (i, j), i > j =======================
    int i, j;
    if (pos < nchain) {
      i = (pos + 1) >> 1;
      j = i - 1;
    } else {
      int t = pos - nchain;
      j = 0;
      while (t >= nb - 2 - j) { t -= nb - 2 - j; ++j; }
      i = j + 2 + t;
    }
    const bool sub = i == j + 1;  // sub-diagonal tile: feeds the diagonal CTA of row i slab by slab
    double* slot = a.M + size_t(i) * kCholNB * npad + j * kCholNB;
    Frag acc;
    frag_load_global(acc, slot, npad, L);
    for (int k = 0; k + 1 < j; ++k) {
      wait_flags2(tile_ready + i * nb + k, tile_ready + j * nb + k, epoch);
      load_tile_cg(S1, a.M + size_t(i) * kCholNB * npad + k * kCholNB, npad, tid);
      load_tile_cg(S2, a.M + size_t(j) * kCholNB * npad + k * kCholNB, npad, tid);
      __syncthreads();
      tile_gemm_dmma<true>(S1, S2, acc, L);
      __syncthreads();
    }
    if (j >= 1) {
      // The last update T -= L(i,j-1) L(j,j-1)' is STREAMED: both operand tiles arrive 16 columns (k) at a time, as
      // self-validating slabs, straight from the CTAs (i, j-1) and (j, j-1) that are still solving them, and are applied as
      // rank-16 updates.  (Waiting for the finished tiles - flag, 2 x 32 KB from L2, four lazy slab products inside the
      // solve - left this CTA behind the packets of column j at every column of the critical chain.)
      const double* srcA = a.Spub + (size_t(i) * nb + (j - 1)) * 4096;
      const double* srcB = a.Spub + (size_t(j) * nb + (j - 1)) * 4096;
      const int r0 = tid >> 5, c0 = (tid & 31) * 2;  // thread's two double2 of a slab: rows r0, r0 + 8
      double2 pa[2], pb[2];
      auto issue = [&](int s) {
#pragma unroll
        for (int u = 0; u < 2; ++u) {
          pa[u] = ld_relaxed2(srcA + size_t(s) * 1024 + (r0 + 8 * u) * 64 + c0);
          pb[u] = ld_relaxed2(srcB + size_t(s) * 1024 + (r0 + 8 * u) * 64 + c0);
        }
      };
      issue(0);
#pragma unroll 1
      for (int s = 0; s < 4; ++s) {
#pragma unroll
        for (int u = 0; u < 2; ++u) {
          const size_t o = size_t(s) * 1024 + (r0 + 8 * u) * 64 + c0;
          while (is_sentinel(pa[u].x) || is_sentinel(pa[u].y)) pa[u] = ld_relaxed2(srcA + o);
          while (is_sentinel(pb[u].x) || is_sentinel(pb[u].y)) pb[u] = ld_relaxed2(srcB + o);
          *reinterpret_cast<double2*>(D + (16 * s + r0 + 8 * u) * kTS + c0) = pa[u];
          *reinterpret_cast<double2*>(S2 + (16 * s + r0 + 8 * u) * kTS + c0) = pb[u];
        }
        if (s < 3) issue(s + 1);
        __syncthreads();
        mma_dispatch(0xFFu, acc, D + (16 * s + L.q) * kTS + L.g, kTS, S2 + (16 * s + L.q) * kTS + L.g, kTS, L, 4);
      }
    }
    // L(i,j) = T L_jj^-T, 16 columns at a time behind the factorisation of block column j; every finished slab is
    // published (diagonal CTA i if this is the sub-diagonal tile, the tiles (r, i), r > i, and (i, j+1) otherwise)
    unsigned slab_remote = 0u;
    if (dsm) {
      cluster_wait();  // every CTA of the cluster has prepared its receive area (long ago by now)
      if (sub && send_remote) slab_remote = mapa_u32(smem_u32(S1), crank + 1);
    }
    trsm_pipelined(acc, L, S1, At, Bp, a.Lpub + size_t(j) * 4 * kPacketG, a.Spub + (size_t(i) * nb + j) * 4096, nullptr, nullptr, tid,
                   sub ? i : -100, (sub && recv_local) ? Pk : nullptr, slab_remote);
    __syncthreads();
    store_tile_global(slot, npad, S1, tid);  // published transposed
    post_flag(tile_ready + i * nb + j, epoch);  // the updates of row i / column i wait for it
    if (!sub) {  // (the diagonal CTA of row i holds a copy of the sub-diagonal tile and forms these two products itself)
      if (tid < kCholNB) vec[tid] = ld_spin(xf_pub + j * kCholNB + tid);
      __syncthreads();
      tile_matvec_t(S1, vec, fwd_part + (size_t(i) * nb + j) * kCholNB, red, tid);
      // backward sweep: L(i,j)^T x_i   (S1 row-major = L^T)
      if (tid < kCholNB) vec[tid] = ld_spin(xb_pub + i * kCholNB + tid);
      __syncthreads();
      tile_matvec(S1, vec, bwd_part + (size_t(j) * nb + i) * kCholNB, tid);
      // next launch of this engine: this CTA's message slots of the other buffer must read as "not yet written"
      if (tid < kCholNB) {
        a.part_other[(size_t(i) * nb + j) * kCholNB + tid] = sv;
        a.part_other[nn + (size_t(j) * nb + i) * kCholNB + tid] = sv;
      }
    }
    {
      double* o = a.Spub_other + (size_t(i) * nb + j) * 4096;
      for (int e = tid; e < 4096 / 2; e += 256) *reinterpret_cast<double2*>(o + 2 * e) = make_double2(sv, sv);
    }
    return;
  }

  // ======================= diagonal CTA j: tile (j, j) =======================
  const int j = pos >> 1;
  DSTAMP(j, 0);
  Frag accD;
  frag_load_global(accD, a.M + size_t(j) * kCholNB * npad + j * kCholNB, npad, L);
  for (int k = 0; k + 1 < j; ++k) {
    wait_flag(tile_ready + j * nb + k, epoch);
    load_tile_cg(S2, a.M + size_t(j) * kCholNB * npad + k * kCholNB, npad, tid);
    __syncthreads();
    mma_dispatch(lower_mask(tid >> 5), accD, S2 + L.q * kTS + L.g, kTS, S2 + L.q * kTS + L.g, kTS, L, kCholNB / 4);
    __syncthreads();
  }
  DSTAMP(j, 1);
  {  // right-hand side of block j for the forward substitution: the partials of the other owners, fixed
    // summation order; this CTA's own partial L(j,j-1) x_{j-1} is added after the factorisation (side job below)
    const double sp = sum_partials(fwd_part + size_t(j) * nb * kCholNB, j >= 1 ? j - 1 : 0, kCholNB, red, tid);
    if (tid < kCholNB) vec[tid] = a.rhs[j * kCholNB + tid] - sp;
  }
  if (j >= 1) {
    // the sub-diagonal tile arrives 16 columns at a time from CTA (j, j-1): S1 rows 16 s .. = P_s^T, accD -= P_s P_s'
    const double* src = a.Spub + (size_t(j) * nb + (j - 1)) * 4096;
    const int r0 = tid >> 5, c0 = (tid & 31) * 2;  // thread's two double2 of a slab: rows r0, r0 + 8
    double2 pre[2];
    auto issue = [&](int s) {
      pre[0] = ld_relaxed2(src + size_t(s) * 1024 + r0 * 64 + c0);
      pre[1] = ld_relaxed2(src + size_t(s) * 1024 + (r0 + 8) * 64 + c0);
    };
    if (!recv_local) issue(0);
#pragma unroll 1
    for (int s = 0; s < 4; ++s) {
      if (recv_local) {  // the slabs land in S1 itself (written by the sub-diagonal CTA through the cluster's shared memory)
#pragma unroll
        for (int u = 0; u < 2; ++u) {
          const double* w = S1 + (16 * s + r0 + 8 * u) * kTS + c0;
          double2 v = ld_shared_volatile2(w);
          while (is_sentinel(v.x) || is_sentinel(v.y)) v = ld_shared_volatile2(w);
        }
      } else {
#pragma unroll
        for (int u = 0; u < 2; ++u) {
          const double* w = src + size_t(s) * 1024 + (r0 + 8 * u) * 64 + c0;
          while (is_sentinel(pre[u].x) || is_sentinel(pre[u].y)) pre[u] = ld_relaxed2(w);
          *reinterpret_cast<double2*>(S1 + (16 * s + r0 + 8 * u) * kTS + c0) = pre[u];
        }
        if (s < 3) issue(s + 1);
      }
      __syncthreads();
      DSTAMP(j, 8 + s);
      if (s == 3) DSTAMP(j, 2);
      mma_dispatch(lower_mask(tid >> 5), accD, S1 + (16 * s + L.q) * kTS + L.g, kTS, S1 + (16 * s + L.q) * kTS + L.g, kTS, L, 4);
    }
    DSTAMP(j, 3);
  }
  frag_store(D, accD, L);
  __syncthreads();
  DSTAMP(j, 4);
  // While warp 0 runs the pivot chains, warps 1..7 publish the packets of this factorisation and form the forward
  // partial of the sub-diagonal tile (a copy of L(j,j-1)^T sits in S1: the four slabs).
  double* own = red;  // [64] L(j,j-1) x_{j-1}   (red is free until the backward sweep)
  double* gpk = a.Lpub + size_t(j) * 4 * kPacketG;
  unsigned rpk = 0u;  // the sub-diagonal tile's packet area, when that CTA is the next one of this cluster
  if (send_remote) rpk = mapa_u32(smem_u32(Pk), crank + 1);
  // (the cluster barrier is waited on by the publishing warps right before their first remote store - by then every CTA
  //  of the cluster has long arrived - so that the pivot chain of this block starts without it)
  auto side = [&](int step) {
    if (j == 0) return;
    const int tt = tid - 32;  // 0..223
    if (step == 1 && tt < kCholNB) {
      // x_{j-1} was published shortly after the last packet of column j-1: long ago by now
      vec2[tt] = ld_spin(xf_pub + (j - 1) * kCholNB + tt);
    } else if (step == 2 && tt < 128) {
      // own[r] = sum_c L(j,j-1)[r][c] x[c] = sum_c S1[c][r] x[c]; two lanes per row
      const int r = tt >> 1, pt = tt & 1;
      double acc = 0.0;
#pragma unroll 8
      for (int c = pt; c < kCholNB; c += 2) acc = fma(S1[c * kTS + r], vec2[c], acc);
      acc += __shfl_xor_sync(0xffffffffu, acc, 1);
      if (pt == 0) own[r] = acc;
    }
  };
  auto pub = [&](int s) {  // warps 1..7: packet s (panel + 16x16 inverse) -> global; the words validate themselves
    if (dsm && s == 0) cluster_wait();
    const int tt = tid - 32;
    const double* src = Pk + s * kPacket;
    double* dst = gpk + size_t(s) * kPacketG;
    for (int e = tt; e < 16 * 40; e += 224) {
      const int r = e / 40, c = (e - r * 40) * 2;
      double2 v = *reinterpret_cast<const double2*>(src + r * kPS + c);
      if (c < 16 * (s + 1) && c < 64) v = make_double2(0.0, 0.0);  // rows of the panel above the diagonal block: unused
      if (rpk) st_cluster2(rpk + unsigned((s * kPacket + r * kPS + c) * sizeof(double)), v);  // the chain's consumer first
      st_relaxed2(dst + r * 80 + c, v);
    }
  };
  auto pub_last = [&]() {  // all threads: the last 16x16 inverse
    if (dsm && tid < 32) cluster_wait();  // (warp 0 has not published anything yet)
    if (tid < 128) {
      const int r = tid >> 3, c = 64 + (tid & 7) * 2;
      const double2 v = *reinterpret_cast<const double2*>(Pk + 3 * kPacket + r * kPS + c);
      if (rpk) st_cluster2(rpk + unsigned((3 * kPacket + r * kPS + c) * sizeof(double)), v);
      st_relaxed2(gpk + size_t(3) * kPacketG + r * 80 + c, v);
    }
  };
  if (!factor_64_pipe(D, Pk, L16t, rdiag, &s_bad, pub, pub_last, side) && tid == 0) a.scal->chol_fail = 1;
  DSTAMP(j, 5);
  // forward substitution of block j: x_j = L_jj^-1 (rhs_j - sum_k L(j,k) x_k)
  if (j >= 1 && tid < kCholNB) vec[tid] -= own[tid];
  __syncthreads();
  block_solve_packets<true>(Pk, vec, x16, tid);
  if (tid < kCholNB) {
    st_relaxed1(xf_pub + j * kCholNB + tid, vec[tid]);  // the tile owners of column j spin on these words
    a.yf[j * kCholNB + tid] = vec[tid];
    vec2[tid] = vec[tid];
  }
  DSTAMP(j, 6);
  if (j == nb - 1) {
    // last block: the backward sweep starts here, with nothing to wait for - substitute straight from the packets
    // (forming the explicit inverse first, as the other columns do off the chain, would put that work ON it)
    __syncthreads();
    block_solve_packets<false>(Pk, vec, x16, tid);  // vec = yf_j on entry (set above), x_j on exit
    if (tid < kCholNB) {
      st_relaxed1(xb_pub + j * kCholNB + tid, vec[tid]);  // tile owners (j, k) spin on xb_pub
      vec2[tid] = vec[tid];
    }
  } else {
    // explicit inverse of the diagonal block (into D, free since the factorisation): off the critical chain - the
    // backward sweep arrives here much later - and it turns the backward solve of this block into one 64x64 product
    inverse_from_packets(Pk, D, tid);
    // backward sweep: x_j = L_jj^-T (yf_j - sum_{r > j} L(r,j)^T x_r); the partials are self-validating words
    {
      const double sp = sum_partials(bwd_part + (size_t(j) * nb + j + 1) * kCholNB, nb - 1 - j, kCholNB, red, tid);
      if (tid < kCholNB) vec[tid] = vec2[tid] - sp;
    }
    __syncthreads();
    tile_matvec_t(D, vec, xb_pub + j * kCholNB, red, tid, vec2);  // x_j = Xi^T v ; tile owners (j, k) spin on xb_pub
  }
  __syncthreads();
  if (j >= 1) {
    // own sub-diagonal tile: L(j,j-1)^T x_j for diagonal CTA j-1, the next link of the backward chain
    tile_matvec(S1, vec2, bwd_part + (size_t(j - 1) * nb + j) * kCholNB, tid);  // S1 row-major = L(j,j-1)^T
  }
  if (tid < kCholNB) a.y[j * kCholNB + tid] = vec2[tid];
  DSTAMP(j, 7);
  {  // next launch of this engine uses the other buffers: leave this CTA's slots there as sentinels
    double* o = a.Lpub_other + size_t(j) * 4 * kPacketG;
    for (int e = tid; e < 4 * kPacketG / 2; e += 256) *reinterpret_cast<double2*>(o + 2 * e) = make_double2(sv, sv);
    if (tid < kCholNB) {
      a.part_other[2 * nn + size_t(j) * kCholNB + tid] = sv;
      a.part_other[2 * nn + size_t(nb + j) * kCholNB + tid] = sv;
      if (j >= 1) a.part_other[nn + (size_t(j - 1) * nb + j) * kCholNB + tid] = sv;
    }
  }
}

constexpr int kDagCluster = 8;
static std::atomic<long long> g_dag_cluster_launches{0};
static std::atomic<long long> g_dag_plain_launches{0};
// number of CTAs the DAG kernel needs for nb block columns
static int dag_grid(int nb) { return nb * (nb + 1) / 2; }

bool chol_dag_supported(int npad, int n_sm) { return dag_grid(npad / kCholNB) <= n_sm; }

static size_t dag_part_half(int npad) {
  const size_t nb = npad / kCholNB;
  return (2 * nb * nb + 2 * nb) * kCholNB;
}
size_t chol_dag_part_len(int npad) { return 2 * dag_part_half(npad); }
size_t chol_dag_flags_len(int npad) {
  const size_t nb = npad / kCholNB;
  return nb * nb;
}
// [barrier kernel's block inverses npad x 64 | packets parity 0 | packets parity 1 | slabs parity 0 | slabs parity 1]
static size_t dag_pub_len(int npad) {
  const size_t nb = npad / kCholNB;
  return nb * 4 * kPacketG + nb * nb * 4096;  // packets of the diagonal CTAs + slabs of every tile (i, k)
}
size_t chol_dag_lpub_len(int npad) { return size_t(npad) * kCholNB + 2 * dag_pub_len(npad); }

__global__ void fill_sentinel_kernel(double* p, size_t n) {
  const size_t i = size_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i < n) p[i] = __longlong_as_double(static_cast<long long>(kSentinel));
}
// both packet buffers start as sentinels (call once after (re)allocating the buffer, on the engine stream)
int launch_chol_dag_init(double* linv_buf, double* part_buf, int npad, cudaStream_t s) {
  const size_t n = 2 * dag_pub_len(npad), m = chol_dag_part_len(npad);
  fill_sentinel_kernel<<<unsigned((n + 255) / 256), 256, 0, s>>>(linv_buf + size_t(npad) * kCholNB, n);
  fill_sentinel_kernel<<<unsigned((m + 255) / 256), 256, 0, s>>>(part_buf, m);
  return 2;
}

int launch_chol_dag(const LinearLaunch& l, cudaStream_t s, bool* tile_dag) {
  static PerDeviceOnce once;
  static std::atomic<unsigned> epoch_src{0};
  if (once.first()) cudaFuncSetAttribute(chol_dag_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, int(kCholDagSmem));
  CholDagArgs a;
  const size_t half = size_t(l.npad / kCholNB) * 4 * kPacketG;
  const unsigned parity = l.chol_seq ? ((*l.chol_seq)++ & 1u) : 0u;
  a.M = l.M; a.npad = l.npad;
  const size_t shalf = size_t(l.npad / kCholNB) * size_t(l.npad / kCholNB) * 4096;
  double* pk = l.Linv + size_t(l.npad) * kCholNB;
  a.Lpub = pk + parity * half;
  a.Lpub_other = pk + (parity ^ 1u) * half;
  a.Spub = pk + 2 * half + parity * shalf;
  a.Spub_other = pk + 2 * half + (parity ^ 1u) * shalf;
  a.part = l.chol_part + parity * dag_part_half(l.npad);
  a.part_other = l.chol_part + (parity ^ 1u) * dag_part_half(l.npad);
  a.rhs = l.rhs; a.y = l.y; a.yf = l.yf;
  a.flags = l.chol_flags; a.scal = l.scal; a.go = l.go;
  // process-wide unique, never 0 (flag buffers start zeroed); a wrap after 2^31 launches would need the flags of a
  // buffer to hold exactly the value 2^31 launches old: not a practical concern
  a.epoch = int(epoch_src.fetch_add(1, std::memory_order_relaxed) % 0x7ffffffeu) + 1;
  // first choice: clusters of 8 consecutive CTAs (the chain's hops go through distributed shared memory), still a
  // cooperative launch (every CTA resident: the CTAs spin on each other's messages)
  static std::atomic<int> cluster_state{-1};  // -1 untested, 0 unavailable on this system, 1 in use
  bool want_cluster = cluster_state.load(std::memory_order_relaxed) != 0;
  if (const char* v = std::getenv("CTVIO_CHOL_CLUSTER"))  // re-read on every call (tests switch it)
    if (v[0] == '0') want_cluster = false;
  // Nsight Compute can not replay a cooperative CLUSTER launch: the driver reports LaunchFailed and the tool shuts the
  // process down (measured).  Under an injected profiler (these variables are set by ncu / nsys in the target's
  // environment) the kernel is launched without clusters - same arithmetic, messages through L2.
  if (std::getenv("NV_COMPUTE_PROFILER_PERFWORKS_DIR") || std::getenv("NV_NSIGHT_INJECTION_TRANSPORT_TYPE") ||
      std::getenv("CUDA_INJECTION64_PATH") || std::getenv("NSYS_PROFILING_SESSION_ID"))
    want_cluster = false;
  const int total = dag_grid(l.npad / kCholNB);
  if (want_cluster) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(unsigned((total + kDagCluster - 1) / kDagCluster * kDagCluster));
    cfg.blockDim = dim3(256);
    cfg.dynamicSmemBytes = kCholDagSmem;
    cfg.stream = s;
    cudaLaunchAttribute at[3];
    at[0].id = cudaLaunchAttributeClusterDimension;
    at[0].val.clusterDim.x = kDagCluster; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
    at[1].id = cudaLaunchAttributeCooperative;
    at[1].val.cooperative = 1;
    at[2].id = cudaLaunchAttributeProgrammaticStreamSerialization;  // pipelined driver (launch_chained, kernels.h)
    at[2].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = at;
    cfg.numAttrs = l.pdl ? 3 : 2;
    cudaError_t cerr = cudaLaunchKernelEx(&cfg, chol_dag_kernel, a);
    if (cerr != cudaSuccess && l.pdl) {  // the three attributes refused together: the plain cluster launch
      cudaGetLastError();
      cfg.numAttrs = 2;
      cerr = cudaLaunchKernelEx(&cfg, chol_dag_kernel, a);
    }
    if (cerr == cudaSuccess) {
      cluster_state.store(1, std::memory_order_relaxed);
      g_dag_cluster_launches.fetch_add(1, std::memory_order_relaxed);
      if (tile_dag) *tile_dag = true;
      return 1;
    }
    cudaGetLastError();
    if (cluster_state.load(std::memory_order_relaxed) < 0) cluster_state.store(0, std::memory_order_relaxed);  // never worked here
  }
  void* args[] = {&a};
  const cudaError_t err = cudaLaunchCooperativeKernel(reinterpret_cast<void*>(chol_dag_kernel), dim3(total),
                                                      dim3(256), args, kCholDagSmem, s);
  if (err != cudaSuccess) {
    // the flag protocol needs every CTA resident; if the runtime cannot promise that (MIG slice, fewer usable SMs than
    // reported, ...) the barrier kernel with its own, smaller grid is the safe path
    cudaGetLastError();
    if (tile_dag) *tile_dag = false;
    return launch_chol_coop(l, s);
  }
  g_dag_plain_launches.fetch_add(1, std::memory_order_relaxed);
  if (tile_dag) *tile_dag = true;
  return 1;
}

const double* chol_dag_last_packets(const double* linv_buf, int npad, unsigned chol_seq) {
  // launch_chol_dag used parity (chol_seq - 1) & 1 and then advanced the counter; nothing resets those packets until the
  // next launch of the other parity has ended
  const size_t half = size_t(npad / kCholNB) * 4 * kPacketG;
  return linv_buf + size_t(npad) * kCholNB + ((chol_seq - 1u) & 1u) * half;
}

// test / tools hook: launches of the tile-DAG kernel that ran with thread-block clusters so far
extern "C" long long ctvio_debug_chol_cluster_launches() { return g_dag_cluster_launches.load(); }
// ... and without clusters (plain cooperative launch)
extern "C" long long ctvio_debug_chol_plain_launches() { return g_dag_plain_launches.load(); }

}  // namespace ctvio
