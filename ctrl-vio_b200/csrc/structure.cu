// The engine's two structure builds of an image-factor set, bit for bit the same arrays of the same factors in the same
// caller order: frame-pair groups, K1 work items, landmark knot ranges, the compact W layout, the K4 per-tile landmark
// lists, the landmark part of the active mask and the knot bitmask of the factors' padded windows.  The device build
// takes a set whose descriptors live on the device (ctvio_add_image_features_from_table, and slot-named factors added
// next to them), the host build a set of host records.  Each has its half of ctvio_marginalize's block discovery.
// Also the sharded mode's owned flags and the structure probe.
//
// structure_kernel runs as ONE CTA: a table window has at most 15 x 1024 factors and 16 distinct frame times, and every
// step is a scan, a stable radix sort or an order-independent atomic min / max / or, so the result does not depend on
// scheduling.  Its counts (plus a knot bitmask) come back in one small block; then schur_lists_kernel fills the K4
// lists, one CTA per tile of the reduced system, into buffers sized from those counts.
#include "engine_state.h"

namespace ctvio {
namespace {

constexpr int kStructThreads = 1024;
constexpr int kRadixBits = 8, kRadix = 1 << kRadixBits;
constexpr int kListThreads = 256;
constexpr int kMaxSlots = kKeyframeMaxSlots;

// count block written by structure_kernel, read back by the host in one copy: kHdrWords header words, then the knot
// bitmask of the image factors' padded windows (bit k of word k / 32: knot k)
enum StructCount { kErr, kItems, kSchurItems, kEntries, kPart, kActiveLm, kWLenLo, kWLenHi, kHdrWords };

struct StructureArgs {
  int n, nK, nL, n_sm, T, frame_cap;
  int64_t t0, dt, pad;
  const FactorDesc* in;     // caller order
  const int64_t* frame_t;   // [kMaxSlots]
  FactorDesc* desc;         // sorted
  int32_t* orig;            // sorted position -> caller index
  VisualItem* items;        // <= n
  int32_t *lo, *hi;
  int64_t* woff;            // [nL + 1]
  uint8_t* active_lm;       // d_active + np: [nL]
  uint64_t* key;            // scratch [max(n, nL)]
  int32_t *ia, *ib;         // scratch [max(n, nL)] each
  int32_t* gstart;          // scratch [n + 1]: first sorted position of each frame-pair group
  int32_t* lm_list;         // [nL]: landmarks with a factor, in (lo, hi, l) order
  int32_t* tiles;           // [3][T (T + 1) / 2]: landmark count | entry offset | item offset per tile
  uint32_t* counts;         // kHdrWords + ceil(nK / 32)
};

// padded knot window [first, last] of an evaluation time: engine.cu's knot_window, on the device
__device__ bool knot_window_dev(int64_t t, int64_t t0, int64_t dt, int64_t pad, int nK, int& first, int& last) {
  const int64_t maxt = t0 + int64_t(nK - 3) * dt;
  if (t < t0 || t >= maxt) return false;
  const int s1 = int((t - t0) / dt);
  const int64_t t2 = t + pad;
  const int s2 = (t2 >= maxt) ? nK - 4 : int((t2 - t0) / dt);
  if (s2 > s1 + 1) return false;
  first = s1;
  last = min(s2 + 3, nK - 1);
  return true;
}

__device__ __forceinline__ int bit_length(uint64_t x) { return x ? 64 - __clzll(x) : 0; }

// exclusive prefix sum of v over the block (blockDim.x threads, a multiple of 32) in thread order; `total` receives the
// block sum.  s: 32 T of shared memory.  Synchronises the block.
template <class T>
__device__ T block_scan(T v, T* s, T& total) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = blockDim.x >> 5;
  T x = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const T y = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= o) x += y;
  }
  if (lane == 31) s[w] = x;
  __syncthreads();
  if (w == 0) {
    T t = lane < nw ? s[lane] : T(0);
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const T y = __shfl_up_sync(0xffffffffu, t, o);
      if (lane >= o) t += y;
    }
    s[lane] = t;
  }
  __syncthreads();
  const T before = (w ? s[w - 1] : T(0)) + x - v;
  total = s[nw - 1];
  __syncthreads();
  return before;
}

struct RadixShared {
  int32_t wcnt[kStructThreads / 32][kRadix];  // per-warp digit counts of one tile, then their output offsets
  int32_t base[kRadix];                       // running output offset of each digit
};

// Stable LSD radix sort of the items a[0, n) by key[item] (its low `bits` bits), 8 bits per pass; a and b ping-pong.
// Each pass walks the items in tiles of one per thread: a warp ranks its lanes among equal digits with a match, and the
// per-warp counts are turned into offsets in (digit, warp) order - so equal keys keep their input order.  Returns the
// buffer that holds the sorted items.
__device__ int32_t* radix_sort(int32_t* a, int32_t* b, int n, const uint64_t* key, int bits, RadixShared& sm) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  for (int shift = 0; shift < bits; shift += kRadixBits) {
    for (int d = tid; d < kRadix; d += kStructThreads) sm.base[d] = 0;
    for (int k = tid; k < (kStructThreads / 32) * kRadix; k += kStructThreads) (&sm.wcnt[0][0])[k] = 0;
    __syncthreads();
    for (int i = tid; i < n; i += kStructThreads) atomicAdd(&sm.base[(key[a[i]] >> shift) & (kRadix - 1)], 1);
    __syncthreads();
    if (warp == 0) {  // exclusive scan of the digit histogram, kRadix / 32 digits per lane
      constexpr int per = kRadix / 32;
      int loc[per], sum = 0;
#pragma unroll
      for (int j = 0; j < per; ++j) { loc[j] = sum; sum += sm.base[lane * per + j]; }
      int x = sum;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int y = __shfl_up_sync(0xffffffffu, x, o);
        if (lane >= o) x += y;
      }
      const int before = x - sum;
#pragma unroll
      for (int j = 0; j < per; ++j) sm.base[lane * per + j] = before + loc[j];
    }
    __syncthreads();
    for (int t0 = 0; t0 < n; t0 += kStructThreads) {
      const int i = t0 + tid;
      const bool valid = i < n;
      const int item = valid ? a[i] : 0;
      const int d = valid ? int((key[item] >> shift) & (kRadix - 1)) : kRadix;
      const unsigned peers = __match_any_sync(0xffffffffu, d);
      const int rank = __popc(peers & ((1u << lane) - 1u));
      if (valid && rank == 0) sm.wcnt[warp][d] = __popc(peers);
      __syncthreads();
      for (int dd = tid; dd < kRadix; dd += kStructThreads) {
        int run = sm.base[dd];
        for (int w = 0; w < kStructThreads / 32; ++w) {
          const int c = sm.wcnt[w][dd];
          sm.wcnt[w][dd] = run;
          run += c;
        }
        sm.base[dd] = run;
      }
      __syncthreads();
      if (valid) b[sm.wcnt[warp][d] + rank] = item;
      __syncthreads();
      for (int k = tid; k < (kStructThreads / 32) * kRadix; k += kStructThreads) (&sm.wcnt[0][0])[k] = 0;
      __syncthreads();
    }
    int32_t* t = a; a = b; b = t;
  }
  return a;
}

__global__ void __launch_bounds__(kStructThreads) structure_kernel(StructureArgs a) {
  __shared__ RadixShared rs;
  __shared__ int s_first[kMaxSlots], s_last[kMaxSlots], s_ok[kMaxSlots];
  __shared__ int s_err, s_cap;
  __shared__ unsigned s_used;
  __shared__ int s_scan[32];
  __shared__ long long s_scan64[32];
  __shared__ unsigned long long s_sum;
  const int tid = threadIdx.x, n = a.n, nK = a.nK, nL = a.nL;
  if (tid < kMaxSlots) {
    int f = 0, l = 0;
    s_ok[tid] = knot_window_dev(a.frame_t[tid], a.t0, a.dt, a.pad, nK, f, l) ? 1 : 0;
    s_first[tid] = f; s_last[tid] = l;
  }
  if (tid == 0) { s_err = INT_MAX; s_used = 0u; }
  for (int l = tid; l < nL; l += kStructThreads) { a.lo[l] = INT_MAX; a.hi[l] = 0; }
  __syncthreads();
  // ---- windows, landmark ranges, sort keys; the first failing factor in caller order decides the error (a time
  //      outside the spline before a landmark out of range, as the host's loop checks them) ----
  const int lbits = bit_length(uint64_t(max(nL - 1, 0)));
  for (int k = tid; k < n; k += kStructThreads) {
    const FactorDesc d = a.in[k];
    const int si = d.slot_i / a.frame_cap, sj = d.slot_j / a.frame_cap;
    if (!s_ok[si] || !s_ok[sj]) { atomicMin(&s_err, 2 * k); continue; }
    if (d.lm < 0 || d.lm >= nL) { atomicMin(&s_err, 2 * k + 1); continue; }
    const int f0 = s_first[si], f1 = s_first[sj];
    atomicMin(&a.lo[d.lm], 6 * min(f0, f1));
    atomicMax(&a.hi[d.lm], 6 * (max(s_last[si], s_last[sj]) + 1));
    atomicOr(&s_used, (1u << si) | (1u << sj));
    a.key[k] = (uint64_t(f0 * nK + f1) << lbits) | uint64_t(d.lm);
    a.ia[k] = k;
  }
  __syncthreads();
  if (s_err != INT_MAX) {
    if (tid == 0) a.counts[kErr] = 1u + uint32_t(s_err);  // 1 + 2 k (+ 1 for the landmark)
    return;
  }
  // ---- order (frame-pair group, landmark, caller position) ----
  const int gbits = bit_length(uint64_t(nK) * uint64_t(nK) - 1);
  const int32_t* sorted = radix_sort(a.ia, a.ib, n, a.key, gbits + lbits, rs);
  for (int s = tid; s < n; s += kStructThreads) {
    const int k = sorted[s];
    a.orig[s] = k;
    a.desc[s] = a.in[k];
  }
  __syncthreads();
  // ---- frame-pair groups (first knots of the two windows) ----
  int n_groups = 0;
  for (int c = 0; c < n; c += kStructThreads) {
    const int s = c + tid;
    const bool head = s < n && (s == 0 || (a.key[a.orig[s]] >> lbits) != (a.key[a.orig[s - 1]] >> lbits));
    int tot;
    const int ex = block_scan(int(head), s_scan, tot);
    if (head) a.gstart[n_groups + ex] = s;
    n_groups += tot;
  }
  if (tid == 0) a.gstart[n_groups] = n;
  __syncthreads();
  // ---- K1 work items: the cap halved while the SMs still hold every chunk, each group cut into equal chunks ----
  if (tid == 0) s_cap = kVisObsPerRound;
  __syncthreads();
  for (;;) {
    const int half = s_cap / 2;
    if (half < kVisMinChunk) break;
    if (tid == 0) s_sum = 0ull;
    __syncthreads();
    unsigned long long m = 0;
    for (int g = tid; g < n_groups; g += kStructThreads) m += (a.gstart[g + 1] - a.gstart[g] + half - 1) / half;
    atomicAdd(&s_sum, m);
    __syncthreads();
    const bool finer = s_sum <= (unsigned long long)a.n_sm;
    __syncthreads();
    if (!finer) break;
    if (tid == 0) s_cap = half;
    __syncthreads();
  }
  const int cap = s_cap;
  int n_items = 0;
  for (int c = 0; c < n_groups; c += kStructThreads) {
    const int g = c + tid;
    int cnt = 0, per = 1, ni = 0;
    if (g < n_groups) {
      cnt = a.gstart[g + 1] - a.gstart[g];
      const int nchunks = (cnt + cap - 1) / cap;
      per = (cnt + nchunks - 1) / nchunks;
      ni = (cnt + per - 1) / per;
    }
    int tot;
    const int ex = block_scan(ni, s_scan, tot);
    if (g < n_groups) {
      const int g0 = a.gstart[g], g1 = a.gstart[g + 1];
      const int gk = int(a.key[a.orig[g0]] >> lbits);
      const int wi0 = gk / nK, wj0 = gk % nK;
      int o = n_items + ex;
      for (int s = g0; s < g1; s += per) a.items[o++] = VisualItem{s, min(per, g1 - s), wi0, wj0};
    }
    n_items += tot;
  }
  // ---- landmark layout: a landmark without a factor gets lo = hi = 0; woff is the scan of hi - lo ----
  long long w_run = 0;
  int n_act = 0;
  for (int c = 0; c < nL; c += kStructThreads) {
    const int l = c + tid;
    int h = 0, lo = 0;
    if (l < nL) {
      h = a.hi[l];
      lo = h == 0 ? 0 : a.lo[l];
    }
    long long tot;
    const long long ex = block_scan((long long)(h - lo), s_scan64, tot);
    int atot;
    const int aex = block_scan(int(h > 0), s_scan, atot);
    if (l < nL) {
      a.lo[l] = lo;
      a.woff[l] = w_run + ex;
      a.active_lm[l] = h > 0 ? 1 : 0;
      if (h > 0) {
        a.ia[n_act + aex] = l;
        a.key[n_act + aex] = uint64_t(lo / 6) * uint64_t(nK + 1) + uint64_t(h / 6);
      }
    }
    w_run += tot;
    n_act += atot;
  }
  if (tid == 0) a.woff[nL] = w_run;
  __syncthreads();
  // ---- K4: the landmarks with a factor in (lo, hi, l) order, counted into every tile pair of the blocks they span
  //      (at most 63 blocks) ----
  for (int k = tid; k < n_act; k += kStructThreads) a.ib[k] = k;  // sort positions into the compacted list
  __syncthreads();
  {
    const int kbits = bit_length(uint64_t(nK + 1) * uint64_t(nK + 1) - 1);
    // (ia holds the landmark of each compacted position; gstart is free again and serves as the second buffer)
    const int32_t* ord = radix_sort(a.ib, a.gstart, n_act, a.key, kbits, rs);
    for (int r = tid; r < n_act; r += kStructThreads) a.lm_list[r] = a.ia[ord[r]];
  }
  const int n_tiles = a.T * (a.T + 1) / 2;
  for (int t = tid; t < n_tiles; t += kStructThreads) a.tiles[t] = 0;
  __syncthreads();
  for (int r = tid; r < n_act; r += kStructThreads) {
    const int l = a.lm_list[r];
    const int b0 = a.lo[l] / kCholNB, b1 = min((a.hi[l] - 1) / kCholNB, b0 + 62);
    for (int x = b0; x <= b1; ++x)
      for (int y = b0; y <= x; ++y) atomicAdd(&a.tiles[x * (x + 1) / 2 + y], 1);
  }
  __syncthreads();
  int total = 0;
  for (int c = 0; c < n_tiles; c += kStructThreads) {
    const int t = c + tid;
    int tot;
    const int ex = block_scan(t < n_tiles ? a.tiles[t] : 0, s_scan, tot);
    if (t < n_tiles) a.tiles[n_tiles + t] = total + ex;
    total += tot;
  }
  const int part = max(32, int((total / (2 * a.n_sm) + 31) / 32) * 32);
  int n_schur = 0;
  for (int c = 0; c < n_tiles; c += kStructThreads) {
    const int t = c + tid;
    const int cnt = t < n_tiles ? a.tiles[t] : 0;
    int tot;
    const int ex = block_scan((cnt + part - 1) / part, s_scan, tot);
    if (t < n_tiles) a.tiles[2 * n_tiles + t] = n_schur + ex;
    n_schur += tot;
  }
  // ---- the knots inside the padded windows of the frames the factors use ----
  const int words = (nK + 31) / 32;
  for (int w = tid; w < words; w += kStructThreads) {
    uint32_t bits = 0;
    for (int s = 0; s < kMaxSlots; ++s) {
      if (!(s_used >> s & 1u)) continue;
      for (int k = max(s_first[s], 32 * w); k <= min(s_last[s], 32 * w + 31); ++k) bits |= 1u << (k - 32 * w);
    }
    a.counts[kHdrWords + w] = bits;
  }
  if (tid == 0) {
    a.counts[kErr] = 0;
    a.counts[kItems] = uint32_t(n_items);
    a.counts[kSchurItems] = uint32_t(n_schur);
    a.counts[kEntries] = uint32_t(total);
    a.counts[kPart] = uint32_t(part);
    a.counts[kActiveLm] = uint32_t(n_act);
    a.counts[kWLenLo] = uint32_t(uint64_t(w_run));
    a.counts[kWLenHi] = uint32_t(uint64_t(w_run) >> 32);
  }
}

struct SchurListArgs {
  int T, n_act, part;
  const int32_t *lm_list, *lo, *hi, *tiles;
  const int64_t* woff;
  SchurEntry* entries;
  SchurTileItem* items;
};

// one CTA per tile (ti >= tj): its landmarks in lm_list order, then its items of `part` landmarks each
__global__ void __launch_bounds__(kListThreads) schur_lists_kernel(SchurListArgs a) {
  __shared__ int s_scan[32];
  const int tile = blockIdx.x, n_tiles = a.T * (a.T + 1) / 2;
  int ti = 0;
  while ((ti + 1) * (ti + 2) / 2 <= tile) ++ti;
  const int tj = tile - ti * (ti + 1) / 2;
  const int cnt = a.tiles[tile], first = a.tiles[n_tiles + tile], item0 = a.tiles[2 * n_tiles + tile];
  int run = 0;
  for (int c = 0; c < a.n_act; c += kListThreads) {
    const int r = c + threadIdx.x;
    int l = -1;
    bool in = false;
    if (r < a.n_act) {
      l = a.lm_list[r];
      const int b0 = a.lo[l] / kCholNB, b1 = min((a.hi[l] - 1) / kCholNB, b0 + 62);
      in = b0 <= tj && ti <= b1;
    }
    int tot;
    const int ex = block_scan(int(in), s_scan, tot);
    if (in) a.entries[first + run + ex] = SchurEntry{l, a.lo[l], a.hi[l], 0, a.woff[l]};
    run += tot;
  }
  for (int i = threadIdx.x; i * a.part < cnt; i += kListThreads)
    a.items[item0 + i] = SchurTileItem{ti, tj, first + i * a.part, min(cnt - i * a.part, a.part)};
}

struct MargDiscoverArgs {
  int n, nK, nL, frame_cap;
  int64_t t0, dt, pad;
  const FactorDesc* desc;   // sorted
  const int64_t* frame_t;
  int32_t* marg_img;        // sorted positions of the flagged factors, ascending
  int32_t* pos_lm;          // rank of each landmark among the flagged factors' landmarks (-1: none)
  uint32_t* counts;         // n_marg, n_rho, knot bitmask
};

// the image part of ctvio_marginalize's block discovery (one CTA)
__global__ void __launch_bounds__(kStructThreads) marg_discover_kernel(MargDiscoverArgs a) {
  __shared__ int s_first[kMaxSlots], s_last[kMaxSlots];
  __shared__ unsigned s_used;
  __shared__ int s_scan[32];
  const int tid = threadIdx.x;
  if (tid < kMaxSlots) {
    int f = 0, l = -1;
    if (!knot_window_dev(a.frame_t[tid], a.t0, a.dt, a.pad, a.nK, f, l)) { f = 0; l = -1; }
    s_first[tid] = f; s_last[tid] = l;
  }
  if (tid == 0) s_used = 0u;
  for (int l = tid; l < a.nL; l += kStructThreads) a.pos_lm[l] = 0;
  __syncthreads();
  int n_marg = 0;
  for (int c = 0; c < a.n; c += kStructThreads) {
    const int s = c + tid;
    const bool m = s < a.n && a.desc[s].marg != 0;
    int tot;
    const int ex = block_scan(int(m), s_scan, tot);
    if (m) {
      const FactorDesc d = a.desc[s];
      a.marg_img[n_marg + ex] = s;
      a.pos_lm[d.lm] = 1;
      atomicOr(&s_used, (1u << (d.slot_i / a.frame_cap)) | (1u << (d.slot_j / a.frame_cap)));
    }
    n_marg += tot;
  }
  __syncthreads();
  int n_rho = 0;
  for (int c = 0; c < a.nL; c += kStructThreads) {
    const int l = c + tid;
    const bool f = l < a.nL && a.pos_lm[l] != 0;
    int tot;
    const int ex = block_scan(int(f), s_scan, tot);
    if (l < a.nL) a.pos_lm[l] = f ? n_rho + ex : -1;
    n_rho += tot;
  }
  const int words = (a.nK + 31) / 32;
  for (int w = tid; w < words; w += kStructThreads) {
    uint32_t bits = 0;
    for (int s = 0; s < kMaxSlots; ++s) {
      if (!(s_used >> s & 1u)) continue;
      for (int k = max(s_first[s], 32 * w); k <= min(s_last[s], 32 * w + 31); ++k) bits |= 1u << (k - 32 * w);
    }
    a.counts[2 + w] = bits;
  }
  if (tid == 0) { a.counts[0] = uint32_t(n_marg); a.counts[1] = uint32_t(n_rho); }
}

__global__ void offset_positions_kernel(int32_t* pos, int n, int base) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n && pos[i] >= 0) pos[i] += base;
}

// sharded mode: owned flags of the landmarks with a factor on this rank (hi > 0), as doubles and as bytes
__global__ void owned_flags_kernel(const int32_t* hi, int nL, double* as_double, uint8_t* as_byte) {
  const int l = blockIdx.x * blockDim.x + threadIdx.x;
  if (l >= nL) return;
  if (as_double) as_double[l] = hi[l] > 0 ? 1.0 : 0.0;
  if (as_byte) as_byte[l] = hi[l] > 0 ? 1 : 0;
}

}  // namespace
}  // namespace ctvio

namespace ctvio::host {

// the SoA payload of the n sorted descriptors in d_img_desc, gathered from the resident frame tables
int gather_factors(ctvio_engine* e, int n) {
  CUDA_OK(e->d_img_t.reserve(n)); CUDA_OK(e->d_img_pi.reserve(n)); CUDA_OK(e->d_img_pj.reserve(n)); CUDA_OK(e->d_img_meta.reserve(n));
  ctvio::GatherFactorsArgs ga;
  ga.n = n; ga.desc = e->d_img_desc.p; ga.table = e->d_frames.p; ga.frame_t = e->d_frame_t.p;
  ga.frame_cap = ctvio_engine::kFrameCap;
  ga.t = e->d_img_t.p; ga.pi = e->d_img_pi.p; ga.pj = e->d_img_pj.p; ga.meta = e->d_img_meta.p;
  e->launches += ctvio::launch_gather_factors(ga, e->stream);
  return CTVIO_OK;
}

int structure_build_device(ctvio_engine* e, int T) {
  cudaStream_t st = e->stream;
  const int n = e->n_img_dev, nL = e->nL, nK = e->nK;
  const ProblemDims d = e->dims();
  const size_t m = size_t(std::max(n, nL)) + 1;
  const int n_tiles = T * (T + 1) / 2;
  const int words = (nK + 31) / 32;
  CUDA_OK(e->d_img_desc.reserve(n)); CUDA_OK(e->d_img_orig.reserve(n)); CUDA_OK(e->d_items.reserve(n));
  CUDA_OK(e->d_lo.reserve(nL)); CUDA_OK(e->d_hi.reserve(nL)); CUDA_OK(e->d_woff.reserve(size_t(nL) + 1));
  CUDA_OK(e->d_active.reserve(size_t(d.np) + nL));
  CUDA_OK(e->sb_key.reserve(m));
  CUDA_OK(e->sb_idx.reserve(3 * m + size_t(nL) + 3 * size_t(n_tiles)));
  CUDA_OK(e->sb_counts.reserve(kHdrWords + words));
  StructureArgs a;
  a.n = n; a.nK = nK; a.nL = nL; a.n_sm = device_sm_count(); a.T = T; a.frame_cap = ctvio_engine::kFrameCap;
  a.t0 = e->cfg.t0_ns; a.dt = e->cfg.dt_ns; a.pad = e->cfg.rs_padding_ns;
  a.in = e->d_img_in.p; a.frame_t = e->d_frame_t.p;
  a.desc = e->d_img_desc.p; a.orig = e->d_img_orig.p; a.items = e->d_items.p;
  a.lo = e->d_lo.p; a.hi = e->d_hi.p; a.woff = e->d_woff.p; a.active_lm = e->d_active.p + d.np;
  a.key = e->sb_key.p;
  a.ia = e->sb_idx.p; a.ib = a.ia + m; a.gstart = a.ib + m; a.lm_list = a.gstart + m; a.tiles = a.lm_list + nL;
  a.counts = e->sb_counts.p;
  structure_kernel<<<1, kStructThreads, 0, st>>>(a);
  e->launches += 1;
  std::vector<uint32_t>& c = e->h_struct_counts;
  c.assign(kHdrWords + words, 0);
  CUDA_OK(cudaMemcpyAsync(c.data(), a.counts, c.size() * sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
  CUDA_OK(stream_sync(st));
  e->d2h_bytes += c.size() * sizeof(uint32_t);
  if (c[kErr]) {
    const uint32_t code = c[kErr] - 1u;
    if (code & 1u) return fail(CTVIO_ERR_INVALID, "landmark index out of range");
    return fail(CTVIO_ERR_TIME_RANGE, "image factor time (+ rolling-shutter padding) outside the spline");
  }
  e->n_items = int(c[kItems]);
  e->n_schur_items = int(c[kSchurItems]);
  e->n_schur_entries = int(c[kEntries]);
  e->w_len = int64_t(uint64_t(c[kWLenLo]) | (uint64_t(c[kWLenHi]) << 32));
  e->img_knots.assign(c.begin() + kHdrWords, c.end());
  e->h_active.assign(d.np, 0);  // the landmark part of the active mask is in d_active already
  return gather_factors(e, n);
}

int schur_lists_device(ctvio_engine* e, int T) {
  const int n_tiles = T * (T + 1) / 2;
  const size_t m = size_t(std::max(e->n_img_dev, e->nL)) + 1;
  CUDA_OK(e->d_schur_list.reserve(size_t(e->n_schur_entries)));
  CUDA_OK(e->d_schur_items.reserve(size_t(e->n_schur_items)));
  SchurListArgs a;
  a.T = T; a.n_act = int(e->h_struct_counts[kActiveLm]); a.part = int(e->h_struct_counts[kPart]);
  a.lm_list = e->sb_idx.p + 3 * m; a.tiles = a.lm_list + e->nL;
  a.lo = e->d_lo.p; a.hi = e->d_hi.p; a.woff = e->d_woff.p;
  a.entries = e->d_schur_list.p; a.items = e->d_schur_items.p;
  if (n_tiles > 0) {
    schur_lists_kernel<<<n_tiles, kListThreads, 0, e->stream>>>(a);
    e->launches += 1;
  }
  return CTVIO_OK;
}

int structure_build_host(ctvio_engine* e) {
  cudaStream_t st = e->stream;
  const ProblemDims d = e->dims();
  // ---- image factors: padded knot windows, landmark knot ranges, the knot bitmask ----
  const int n = int(e->img.size());
  std::vector<int32_t> wi0(n), wj0(n);
  e->h_lo.assign(e->nL, INT32_MAX);
  e->h_hi.assign(e->nL, 0);
  e->img_knots.assign((size_t(e->nK) + 31) / 32, 0u);
  // the image factors of a window carry a dozen distinct frame times: the padded knot window of a time (two 64-bit
  // divisions) is looked up in a small direct-mapped cache.  Every window handed out was computed by a fill, so the
  // fills mark the bitmask.
  struct WinCache { int64_t t = INT64_MIN; int f = 0, l = 0; bool ok = false; } wc[64];
  auto window_of = [&](int64_t t, int& f, int& l) {
    WinCache& c = wc[size_t(uint64_t(t) * 0x9E3779B97F4A7C15ull >> 58)];
    if (c.t != t) {
      c.t = t;
      c.ok = knot_window(e, t, c.f, c.l);
      for (int k = c.f; c.ok && k <= c.l; ++k) e->img_knots[size_t(k) / 32] |= 1u << (k % 32);
    }
    f = c.f; l = c.l;
    return c.ok;
  };
  for (int k = 0; k < n; ++k) {
    const HostImage& o = e->img[k];
    int f0, l0, f1, l1;
    if (!window_of(o.ti, f0, l0) || !window_of(o.tj, f1, l1))
      return fail(CTVIO_ERR_TIME_RANGE, "image factor time (+ rolling-shutter padding) outside the spline");
    if (o.lm < 0 || o.lm >= e->nL) return fail(CTVIO_ERR_INVALID, "landmark index out of range");
    wi0[k] = f0; wj0[k] = f1;
    e->h_lo[o.lm] = std::min(e->h_lo[o.lm], 6 * std::min(f0, f1));
    e->h_hi[o.lm] = std::max(e->h_hi[o.lm], 6 * (std::max(l0, l1) + 1));
  }
  e->img_order.resize(n);
  // order: (frame-pair group, landmark, position).  The reference's feature loop hands the factors over landmark by
  // landmark (trajectory_manager.cpp:360-385), so they usually arrive sorted by landmark already: then a STABLE
  // counting sort by group is the whole job (O(n), this runs once per window inside the end-to-end time); any other
  // input order takes the general key sort.
  bool lm_sorted = true;
  for (int k = 1; k < n && lm_sorted; ++k) lm_sorted = e->img[k - 1].lm <= e->img[k].lm;
  const size_t nKk = size_t(e->nK) + 1;
  if (lm_sorted && nKk * nKk <= (size_t(1) << 22)) {
    std::vector<int32_t> start(nKk * nKk + 1, 0);
    for (int k = 0; k < n; ++k) ++start[size_t(wi0[k]) * nKk + size_t(wj0[k]) + 1];
    for (size_t g = 1; g < start.size(); ++g) start[g] += start[g - 1];
    for (int k = 0; k < n; ++k) e->img_order[start[size_t(wi0[k]) * nKk + size_t(wj0[k])]++] = k;
  } else {
    std::vector<uint64_t> key(n);
    const uint64_t nLl = uint64_t(std::max(e->nL, 1));
    if (uint64_t(nKk) * nKk * nLl < (uint64_t(1) << 40) && uint64_t(n) < (uint64_t(1) << 24)) {
      for (int k = 0; k < n; ++k)
        key[k] = (((uint64_t(wi0[k]) * nKk + uint64_t(wj0[k])) * nLl + uint64_t(e->img[k].lm)) << 24) | uint64_t(k);
      std::sort(key.begin(), key.end());
      for (int k = 0; k < n; ++k) e->img_order[k] = int32_t(key[k] & 0xffffffu);
    } else {
      for (int k = 0; k < n; ++k) e->img_order[k] = k;
      std::stable_sort(e->img_order.begin(), e->img_order.end(), [&](int a, int b) {
        if (wi0[a] != wi0[b]) return wi0[a] < wi0[b];
        if (wj0[a] != wj0[b]) return wj0[a] < wj0[b];
        return e->img[a].lm < e->img[b].lm;
      });
    }
  }
  std::vector<longlong2> ht(n);
  std::vector<double2> hpi(n), hpj(n);
  std::vector<int4> hm(n);
  for (int k = 0; k < n; ++k) {
    const HostImage& o = e->img[e->img_order[k]];
    ht[k] = make_longlong2(o.ti, o.tj);
    hpi[k] = make_double2(o.pi[0], o.pi[1]);
    hpj[k] = make_double2(o.pj[0], o.pj[1]);
    hm[k] = make_int4(o.rowi, o.rowj, o.lm, o.marg);
  }
  // work items: chunks of one group, one evaluation round (<= 128 observations, a lane pair each) per CTA.  The
  // round is latency bound whatever its fill, so a group is cut into EQUAL chunks (263 observations -> 3 x 88, not
  // 128 + 128 + 7) and every chunk gets its own CTA.  A window with fewer chunks than SMs has its groups cut finer
  // (the cap halved down to kVisMinChunk) as long as all chunks still run at once: each CTA then has fewer rows to
  // evaluate and to reduce in its SYRK, on SMs that would otherwise idle.  A window that fills the SMs keeps full
  // rounds (finer chunks would only add flushes).
  std::vector<int2> groups;  // [first, end) in sorted order
  for (int k = 0; k < n;) {
    const int a = e->img_order[k];
    int end = k;
    while (end < n && wi0[e->img_order[end]] == wi0[a] && wj0[e->img_order[end]] == wj0[a]) ++end;
    groups.push_back(make_int2(k, end));
    k = end;
  }
  auto n_chunks = [&](int c) {
    size_t m = 0;
    for (const int2& g : groups) m += (g.y - g.x + c - 1) / c;
    return m;
  };
  int cap = kVisObsPerRound;
  const size_t n_sm = size_t(device_sm_count());
  while (cap / 2 >= kVisMinChunk && n_chunks(cap / 2) <= n_sm) cap /= 2;
  std::vector<VisualItem> items;
  for (const int2& g : groups) {
    const int a = e->img_order[g.x];
    const int cnt = g.y - g.x;
    const int nchunks = (cnt + cap - 1) / cap;
    const int per = (cnt + nchunks - 1) / nchunks;
    for (int s = g.x; s < g.y; s += per) items.push_back(VisualItem{s, std::min(per, g.y - s), wi0[a], wj0[a]});
  }
  e->n_items = int(items.size());
  if (!e->img_desc.empty()) {
    // slot-named factors: only the sorted 16-byte descriptors go up, the SoA payload is gathered on the device
    std::vector<ctvio::FactorDesc> sd(n);
    for (int k = 0; k < n; ++k) sd[k] = e->img_desc[e->img_order[k]];
    CUDA_OK(e->d_img_desc.upload(sd, st));
    if (const int rc = gather_factors(e, n)) return rc;
  } else {
    CUDA_OK(e->d_img_t.upload(ht, st));
    CUDA_OK(e->d_img_pi.upload(hpi, st));
    CUDA_OK(e->d_img_pj.upload(hpj, st));
    CUDA_OK(e->d_img_meta.upload(hm, st));
  }
  CUDA_OK(e->d_img_orig.upload(e->img_order, st));
  CUDA_OK(e->d_items.upload(items, st));

  // ---- landmark layout; a landmark with a factor is active (the landmark part of the active mask) ----
  e->h_woff.assign(e->nL + 1, 0);
  e->h_active.assign(size_t(d.np) + e->nL, 0);
  for (int l = 0; l < e->nL; ++l) {
    if (e->h_hi[l] == 0) e->h_lo[l] = 0;
    e->h_woff[l + 1] = e->h_woff[l] + (e->h_hi[l] - e->h_lo[l]);
    e->h_active[d.np + l] = e->h_hi[l] > 0 ? 1 : 0;
  }
  CUDA_OK(e->d_lo.upload(e->h_lo, st));
  CUDA_OK(e->d_hi.upload(e->h_hi, st));
  CUDA_OK(e->d_woff.upload(e->h_woff, st));
  e->w_len = e->h_woff[e->nL];
  return CTVIO_OK;
}

int schur_lists_host(ctvio_engine* e, int T) {
  // per 64x64 tile (ti >= tj) of the reduced system the landmarks whose knot-dim range [lo, hi) touches both blocks,
  // cut into parts of `part` landmarks so that about two waves of CTAs exist whatever the window size (the line-delay
  // row / column is a matrix-vector product done by the diagonal tiles)
  std::vector<std::vector<int32_t>> lists(size_t(T) * (T + 1) / 2);
  std::vector<int32_t> order;
  for (int l = 0; l < e->nL; ++l)
    if (e->h_hi[l] > 0) order.push_back(l);
  std::stable_sort(order.begin(), order.end(), [&](int a, int b) {
    if (e->h_lo[a] != e->h_lo[b]) return e->h_lo[a] < e->h_lo[b];
    return e->h_hi[a] < e->h_hi[b];
  });
  size_t total = 0;
  for (int l : order) {
    int blocks[64], nbk = 0;
    const int b0 = e->h_lo[l] / kCholNB, b1 = (e->h_hi[l] - 1) / kCholNB;
    for (int b = b0; b <= b1 && nbk < 63; ++b) blocks[nbk++] = b;
    for (int x = 0; x < nbk; ++x)
      for (int y = 0; y <= x; ++y) {
        lists[size_t(blocks[x]) * (blocks[x] + 1) / 2 + blocks[y]].push_back(l);
        ++total;
      }
  }
  const int part = std::max(32, int((total / size_t(2 * device_sm_count()) + 31) / 32) * 32);
  std::vector<SchurTileItem> items;
  std::vector<SchurEntry> flat;
  flat.reserve(total);
  for (int ti = 0; ti < T; ++ti)
    for (int tj = 0; tj <= ti; ++tj) {
      const std::vector<int32_t>& v = lists[size_t(ti) * (ti + 1) / 2 + tj];
      for (size_t s0 = 0; s0 < v.size(); s0 += part)
        items.push_back(SchurTileItem{ti, tj, int32_t(flat.size() + s0), int32_t(std::min(v.size() - s0, size_t(part)))});
      for (int32_t l : v) flat.push_back(SchurEntry{l, e->h_lo[l], e->h_hi[l], 0, e->h_woff[l]});
    }
  e->n_schur_items = int(items.size());
  e->n_schur_entries = int(flat.size());
  CUDA_OK(e->d_schur_list.upload(flat, e->stream));
  CUDA_OK(e->d_schur_items.upload(items, e->stream));
  return CTVIO_OK;
}

int marg_discover_host(ctvio_engine* e, std::vector<uint32_t>& knots, int& n_marg, int& n_rho,
                       std::vector<int32_t>& marg_img, std::vector<int32_t>& pos_lm) {
  knots.assign((size_t(e->nK) + 31) / 32, 0u);
  marg_img.clear();
  pos_lm.assign(size_t(std::max(e->nL, 1)), -1);
  for (size_t k = 0; k < e->img_order.size(); ++k) {
    const HostImage& o = e->img[e->img_order[k]];
    if (!o.marg) continue;
    marg_img.push_back(int32_t(k));
    pos_lm[o.lm] = 0;
    for (const int64_t t : {o.ti, o.tj}) {
      int f = 0, l = -1;
      knot_window(e, t, f, l);  // checked by the structure build
      for (int kk = f; kk <= l; ++kk) knots[size_t(kk) / 32] |= 1u << (kk % 32);
    }
  }
  n_marg = int(marg_img.size());
  n_rho = 0;
  for (int32_t& p : pos_lm)
    if (p == 0) p = n_rho++;
  return CTVIO_OK;
}

int marg_discover_device(ctvio_engine* e, std::vector<uint32_t>& knots, int& n_marg, int& n_rho) {
  cudaStream_t st = e->stream;
  const int n = e->n_img_dev, words = (e->nK + 31) / 32;
  ctvio_engine::MargWs& ws = e->mws;
  CUDA_OK(ws.marg_img.reserve(size_t(std::max(n, 1))));
  CUDA_OK(ws.pos_lm.reserve(size_t(std::max(e->nL, 1))));
  CUDA_OK(e->sb_counts.reserve(size_t(2 + words)));
  MargDiscoverArgs a;
  a.n = n; a.nK = e->nK; a.nL = e->nL; a.frame_cap = ctvio_engine::kFrameCap;
  a.t0 = e->cfg.t0_ns; a.dt = e->cfg.dt_ns; a.pad = e->cfg.rs_padding_ns;
  a.desc = e->d_img_desc.p; a.frame_t = e->d_frame_t.p;
  a.marg_img = ws.marg_img.p; a.pos_lm = ws.pos_lm.p; a.counts = e->sb_counts.p;
  marg_discover_kernel<<<1, kStructThreads, 0, st>>>(a);
  e->launches += 1;
  std::vector<uint32_t> c(2 + words);
  CUDA_OK(cudaMemcpyAsync(c.data(), a.counts, c.size() * sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
  CUDA_OK(stream_sync(st));
  e->d2h_bytes += c.size() * sizeof(uint32_t);
  n_marg = int(c[0]);
  n_rho = int(c[1]);
  knots.assign(c.begin() + 2, c.end());
  return CTVIO_OK;
}

int offset_pos_lm_device(ctvio_engine* e, int base) {
  if (e->nL <= 0 || base == 0) return CTVIO_OK;
  offset_positions_kernel<<<(e->nL + 127) / 128, 128, 0, e->stream>>>(e->mws.pos_lm.p, e->nL, base);
  e->launches += 1;
  return CTVIO_OK;
}

int owned_flags_device(ctvio_engine* e, double* as_double, uint8_t* as_byte) {
  if (e->nL <= 0) return CTVIO_OK;
  owned_flags_kernel<<<(e->nL + 127) / 128, 128, 0, e->stream>>>(e->d_hi.p, e->nL, as_double, as_byte);
  e->launches += 1;
  return CTVIO_OK;
}

}  // namespace ctvio::host

extern "C" int ctvio_debug_structure(ctvio_handle e, int64_t* out, int64_t* len) {
  if (!e || !len) return fail(CTVIO_ERR_INVALID, "null argument");
  cudaSetDevice(e->cfg.device);
  if (const int rc = prepare(e)) return rc;
  const ProblemDims d = e->dims();
  const size_t n = e->n_img(), nL = size_t(e->nL), np = size_t(d.np);
  const size_t n_desc = (e->n_img_dev > 0 || !e->img_desc.empty()) ? n : 0;
  const size_t ni = size_t(e->n_items), nsi = size_t(e->n_schur_items), ne = size_t(e->n_schur_entries);
  const size_t nm = e->n_marg_img >= 0 ? size_t(e->n_marg_img) : 0;
  const size_t marg_len = e->n_marg_img >= 0 ? np + nL + nm : 0;
  const size_t nii = size_t(e->n_imu_items);
  const size_t need = 16 + 4 * n_desc + n + 4 * ni + 3 * nL + 1 + 4 * nsi + 5 * ne + np + nL + marg_len + 4 * nii;
  const int64_t cap = *len;
  *len = int64_t(need);
  if (!out) return CTVIO_OK;
  if (cap < int64_t(need)) return fail(CTVIO_ERR_INVALID, "output slab too small");
  cudaStream_t st = e->stream;
  std::vector<ctvio::FactorDesc> desc(n_desc);
  std::vector<int32_t> orig(n), lo(nL), hi(nL), pos_cam(marg_len ? np : 0), pos_lm(marg_len ? nL : 0), marg(nm);
  std::vector<VisualItem> items(ni);
  std::vector<int64_t> woff(nL + 1);
  std::vector<SchurTileItem> sitems(nsi);
  std::vector<SchurEntry> entries(ne);
  std::vector<uint8_t> active(np + nL);
  std::vector<ImuItem> imu_items(nii);
  auto get = [&](auto& v, const void* src) {
    return v.empty() ? cudaSuccess : cudaMemcpyAsync(v.data(), src, v.size() * sizeof(v[0]), cudaMemcpyDeviceToHost, st);
  };
  CUDA_OK(get(desc, e->d_img_desc.p)); CUDA_OK(get(orig, e->d_img_orig.p)); CUDA_OK(get(items, e->d_items.p));
  CUDA_OK(get(lo, e->d_lo.p)); CUDA_OK(get(hi, e->d_hi.p)); CUDA_OK(get(woff, e->d_woff.p));
  CUDA_OK(get(sitems, e->d_schur_items.p)); CUDA_OK(get(entries, e->d_schur_list.p)); CUDA_OK(get(active, e->d_active.p));
  CUDA_OK(get(pos_cam, e->mws.pos_cam.p)); CUDA_OK(get(pos_lm, e->mws.pos_lm.p)); CUDA_OK(get(marg, e->mws.marg_img.p));
  CUDA_OK(get(imu_items, e->d_imu_items.p));
  CUDA_OK(stream_sync(st));
  std::memset(out, 0, 16 * sizeof(int64_t));
  out[0] = int64_t(n); out[1] = int64_t(n_desc); out[2] = int64_t(ni); out[3] = int64_t(nL); out[4] = int64_t(nsi);
  out[5] = int64_t(ne); out[6] = int64_t(np); out[7] = e->n_marg_img; out[8] = int64_t(nii);
  int64_t* o = out + 16;
  for (const auto& x : desc) { *o++ = x.slot_i; *o++ = x.slot_j; *o++ = x.lm; *o++ = x.marg; }
  for (int32_t x : orig) *o++ = x;
  for (const auto& x : items) { *o++ = x.start; *o++ = x.count; *o++ = x.wi0; *o++ = x.wj0; }
  for (int32_t x : lo) *o++ = x;
  for (int32_t x : hi) *o++ = x;
  for (int64_t x : woff) *o++ = x;
  for (const auto& x : sitems) { *o++ = x.ti; *o++ = x.tj; *o++ = x.first; *o++ = x.count; }
  for (const auto& x : entries) { *o++ = x.l; *o++ = x.lo; *o++ = x.hi; *o++ = x.pad; *o++ = x.woff; }
  for (uint8_t x : active) *o++ = x;
  for (int32_t x : pos_cam) *o++ = x;
  for (int32_t x : pos_lm) *o++ = x;
  for (int32_t x : marg) *o++ = x;
  for (const auto& x : imu_items) { *o++ = x.start; *o++ = x.count; *o++ = x.s; *o++ = x.node; }
  return CTVIO_OK;
}
