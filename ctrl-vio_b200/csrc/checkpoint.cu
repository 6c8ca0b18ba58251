// Checkpoint and restore of the per-image odometry cycle's run (include/ctvio.h: ctvio_odometry_checkpoint,
// ctvio_odometry_restore): everything a later ctvio_process_image reads, in one self-describing blob.
//
// Blob layout (little-endian): CkptHeader (magic, format version, ABI version, length, checksum, section table), then
// the sections in CkptSection order, each at an 8-byte aligned offset and zero-padded to 8 bytes.  The first two
// sections (the counts and the host bookkeeping; the prior's block lists) are written by the host, the others are
// gathered on the device by checkpoint_pack_kernel.  The checksum covers every byte after the header: the sum modulo
// 2^64 of mix(word k, k) over its 8-byte words, mix a bijection of the word for each k, so one changed byte always
// changes it and the sum does not depend on how the words are split between CTAs, the host and the device.
#include <cstddef>

#include "engine_state.h"

namespace ctvio {
namespace {

constexpr uint64_t kCkptMagic = 0x504B434F49565443ull;  // "CTVIOCKP"
constexpr uint32_t kCkptFormat = 1;
constexpr int kSlots = kKeyframeMaxSlots;
constexpr int kCkptThreads = 256, kCkptMaxBlocks = 264, kMaxSeg = 40;

enum CkptSection : int {
  kMeta, kPriorBlocks,                                    // host-written
  kKnotQ, kKnotP, kBias, kRho, kLineDelay,                // the state
  kPriorJ, kPriorR, kPriorX0,                             // the active prior
  kImuT, kImuGa, kImuCarry,                               // the resident IMU table with its dt^2 prefix
  kFtId, kFtAnchor, kFtMask, kFtLm, kFtRho, kFtKey, kFtIdx,  // the feature table's live entries
  kClouds,                                                // the held slots' clouds, in slot order
  kSections
};
constexpr int kFirstDeviceSection = kKnotQ;

struct SectionEntry { uint64_t offset, bytes; };
struct CkptHeader {
  uint64_t magic;
  uint32_t format_version, abi_version;
  uint64_t length;     // of the whole blob
  uint64_t checksum;   // of the bytes after the header
  uint32_t n_sections, reserved;
  SectionEntry section[kSections];
};
// the counts and the host-side bookkeeping of the run; nK, nB, nL lead so that a binding can read them
struct CkptMeta {
  int32_t nK, nB, nL, prior_n, prior_nb, prior_enabled;
  int32_t n_imu, n_entries;
  uint32_t held;
  int32_t ft_n_lm, ft_n_obs, ft_oldest_slot;
  int32_t n_frames, reserved;
  int64_t t0_ns, next_frame;
  int32_t slot[kSlots];     // the cycle's window: frame slot and time of each position
  int64_t t[kSlots];
  int32_t frame_n[kSlots];  // per frame slot: the cloud's point count and time (0 for a slot the table does not hold)
  int64_t frame_t[kSlots];
  ctvio_config cfg;         // device and reserved 0, t0_ns as the slides have moved it
  ctvio_cycle_options opt;
};
static_assert(sizeof(CkptHeader) % 8 == 0 && sizeof(CkptMeta) % 8 == 0, "the sections start 8-byte aligned");

// kCopy: the bytes as they are; kIdx: the feature table's per-slot indices of the live entries (see the pack kernel);
// kPositions: the knot positions without the padding element of their kPStride layout (written 0 by a restore);
// kCloud: FrameFeature records with their padding word stored as 0 (the unpacking kernel leaves it unwritten)
enum SegKind : int32_t { kCopy = 0, kIdx = 1, kPositions = 2, kCloud = 3 };
// a device section, or one slot's part of kClouds: bytes at blob offset `off` <-> ptr
struct CkptSeg {
  unsigned char* ptr;
  uint64_t off, bytes;
  int32_t kind, pad;
};
struct CkptArgs {
  unsigned char* blob;           // device staging, in the blob's layout
  uint64_t begin, end;           // the bytes this launch covers (8-byte aligned)
  uint64_t body;                 // offset of checksum word 0 (the end of the header)
  int32_t n_seg;
  int32_t n_entries;             // kIdx: entries per slot
  const uint32_t* mask;          // kIdx, pack: the entries' slot masks
  unsigned long long* partial;   // [gridDim.x]
  int32_t* ticket;
  int32_t* verdict;              // verify: 0 passed, 1 section table, 2 checksum (mapped host memory)
  uint64_t expect[kSections];    // verify: the section sizes the host derived from the counts
  CkptSeg seg[kMaxSeg];          // sorted by off, none empty
};

__host__ __device__ __forceinline__ unsigned long long ckpt_mix(unsigned long long w, unsigned long long k) {
  unsigned long long z = w + (k + 1) * 0x9E3779B97F4A7C15ull;  // splitmix64's finalizer: a bijection of w
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}

__host__ __device__ __forceinline__ uint64_t align8(uint64_t x) { return (x + 7) & ~uint64_t(7); }

// the segment holding blob offset o: the last one with off <= o
__device__ __forceinline__ int find_seg(const CkptSeg* s, int n, uint64_t o) {
  int lo = 0, hi = n - 1;
  while (lo < hi) {
    const int m = (lo + hi + 1) >> 1;
    if (s[m].off <= o) lo = m;
    else hi = m - 1;
  }
  return lo;
}

// The block's sum into partial[blockIdx.x]; the last block to finish (ticket) adds the partial sums in block order into
// *total (thread 0 only) and resets the ticket.  Returns true in that block.
__device__ bool block_sum_last(unsigned long long v, const CkptArgs& a, unsigned long long* total) {
  __shared__ unsigned long long s_warp[kCkptThreads / 32];
  __shared__ bool s_last;
  for (int d = 16; d; d >>= 1) v += __shfl_down_sync(0xffffffffu, v, d);
  if ((threadIdx.x & 31) == 0) s_warp[threadIdx.x >> 5] = v;
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned long long b = 0;
    for (int k = 0; k < kCkptThreads / 32; ++k) b += s_warp[k];
    a.partial[blockIdx.x] = b;
    __threadfence();
    s_last = atomicAdd(a.ticket, 1) == int(gridDim.x) - 1;
  }
  __syncthreads();
  if (!s_last) return false;
  if (threadIdx.x == 0) {
    __threadfence();
    unsigned long long t = 0;
    for (unsigned k = 0; k < gridDim.x; ++k) t += reinterpret_cast<volatile unsigned long long*>(a.partial)[k];
    *total = t;
    *a.ticket = 0;
  }
  return true;
}

__device__ __forceinline__ void load_segments(const CkptArgs& a, CkptSeg* seg) {
  for (int k = threadIdx.x; k < a.n_seg; k += blockDim.x) seg[k] = a.seg[k];
  __syncthreads();
}

// Gathers the device sections into the staging blob (the feature table compacted to its live entries, each entry's
// index in a slot it is not observed in written as -1; the clouds cut to their point counts) and writes their part of
// the checksum into the header's checksum field.
__global__ void __launch_bounds__(kCkptThreads) checkpoint_pack_kernel(const CkptArgs a) {
  __shared__ CkptSeg seg[kMaxSeg];
  load_segments(a, seg);
  unsigned long long sum = 0;
  const uint64_t step = 8ull * gridDim.x * blockDim.x;
  for (uint64_t o = a.begin + 8ull * (uint64_t(blockIdx.x) * blockDim.x + threadIdx.x); o < a.end; o += step) {
    const CkptSeg& s = seg[find_seg(seg, a.n_seg, o)];
    const uint64_t rel = o - s.off;
    unsigned long long w = 0;
    if (s.kind == kIdx) {
      const uint64_t n = uint64_t(a.n_entries) * kSlots;
      for (int h = 0; h < 2; ++h) {
        const uint64_t j = rel / 4 + h;
        if (j >= n) break;
        const int slot = int(j / a.n_entries), ent = int(j % a.n_entries);
        const int32_t v = (a.mask[ent] >> slot & 1u)
                              ? reinterpret_cast<const int32_t*>(s.ptr)[size_t(slot) * kFeatureTableMaxEntries + ent] : -1;
        w |= (unsigned long long)(uint32_t)v << (32 * h);
      }
    } else if (s.kind == kPositions) {
      const uint64_t j = rel / 8;
      w = reinterpret_cast<const unsigned long long*>(s.ptr)[kPStride * (j / 3) + j % 3];
    } else if (s.kind == kCloud) {
      static_assert(sizeof(FrameFeature) == 32, "four words per feature, the last one padding");
      w = (rel / 8) % 4 == 3 ? 0ull : *reinterpret_cast<const unsigned long long*>(s.ptr + rel);
    } else if (rel + 8 <= s.bytes) {
      w = *reinterpret_cast<const unsigned long long*>(s.ptr + rel);
    } else {
      w = *reinterpret_cast<const uint32_t*>(s.ptr + rel);  // a 4-byte tail: every section is a multiple of 4 bytes
    }
    *reinterpret_cast<unsigned long long*>(a.blob + o) = w;
    sum += ckpt_mix(w, (o - a.body) >> 3);
  }
  unsigned long long total = 0;
  if (block_sum_last(sum, a, &total) && threadIdx.x == 0) reinterpret_cast<CkptHeader*>(a.blob)->checksum = total;
}

// kCommit = false: the checksum of the whole body and the section table against the header, into *verdict; nothing
// but the scratch is written.  kCommit = true (after a passing verdict): the device sections scattered into the
// engine's buffers.
template <bool kCommit>
__global__ void __launch_bounds__(kCkptThreads) checkpoint_unpack_kernel(const CkptArgs a) {
  __shared__ CkptSeg seg[kMaxSeg];
  const uint64_t step = 8ull * gridDim.x * blockDim.x;
  const uint64_t first = 8ull * (uint64_t(blockIdx.x) * blockDim.x + threadIdx.x);
  if (kCommit) {
    load_segments(a, seg);
    for (uint64_t o = a.begin + first; o < a.end; o += step) {
      const CkptSeg& s = seg[find_seg(seg, a.n_seg, o)];
      const uint64_t rel = o - s.off;
      const unsigned long long w = *reinterpret_cast<const unsigned long long*>(a.blob + o);
      if (s.kind == kIdx) {
        const uint64_t n = uint64_t(a.n_entries) * kSlots;
        for (int h = 0; h < 2; ++h) {
          const uint64_t j = rel / 4 + h;
          if (j >= n) break;
          const int slot = int(j / a.n_entries), ent = int(j % a.n_entries);
          reinterpret_cast<int32_t*>(s.ptr)[size_t(slot) * kFeatureTableMaxEntries + ent] = int32_t(uint32_t(w >> (32 * h)));
        }
      } else if (s.kind == kPositions) {
        const uint64_t j = rel / 8;
        unsigned long long* p = reinterpret_cast<unsigned long long*>(s.ptr) + kPStride * (j / 3);
        p[j % 3] = w;
        if (j % 3 == 2) p[3] = 0;
      } else if (rel + 8 <= s.bytes) {
        *reinterpret_cast<unsigned long long*>(s.ptr + rel) = w;
      } else {
        *reinterpret_cast<uint32_t*>(s.ptr + rel) = uint32_t(w);
      }
    }
    return;
  }
  unsigned long long sum = 0;
  for (uint64_t o = a.begin + first; o < a.end; o += step)
    sum += ckpt_mix(*reinterpret_cast<const unsigned long long*>(a.blob + o), (o - a.body) >> 3);
  unsigned long long total = 0;
  if (block_sum_last(sum, a, &total) && threadIdx.x == 0) {
    const CkptHeader& h = *reinterpret_cast<const CkptHeader*>(a.blob);
    bool table_ok = h.n_sections == kSections && h.length == a.end;
    uint64_t at = sizeof(CkptHeader);
    for (int k = 0; k < kSections && table_ok; ++k) {
      const SectionEntry& s = h.section[k];
      table_ok = s.offset == at && s.bytes == a.expect[k] && s.offset + s.bytes <= h.length;
      at = align8(s.offset + s.bytes);
    }
    table_ok = table_ok && at == h.length;
    *a.verdict = !table_ok ? 1 : (total != h.checksum ? 2 : 0);
  }
}

}  // namespace
}  // namespace ctvio

namespace {

using ctvio::CkptArgs;
using ctvio::CkptHeader;
using ctvio::CkptMeta;
using ctvio::CkptSeg;
using ctvio::align8;
using ctvio::kSections;

struct Layout {
  uint64_t off[kSections], bytes[kSections];
  uint64_t length;
};

// the sections' sizes and offsets implied by the counts (validated counts: no overflow)
Layout layout_of(const CkptMeta& m) {
  Layout L;
  uint64_t* b = L.bytes;
  const uint64_t ne = uint64_t(m.n_entries), nb = uint64_t(m.prior_nb), n = uint64_t(m.prior_n);
  b[ctvio::kMeta] = sizeof(CkptMeta);
  b[ctvio::kPriorBlocks] = 12 * nb;
  b[ctvio::kKnotQ] = 32 * uint64_t(m.nK);
  b[ctvio::kKnotP] = 24 * uint64_t(m.nK);
  b[ctvio::kBias] = 48 * uint64_t(m.nB);
  b[ctvio::kRho] = 8 * uint64_t(m.nL);
  b[ctvio::kLineDelay] = 8;
  b[ctvio::kPriorJ] = 8 * n * n;
  b[ctvio::kPriorR] = 8 * n;
  b[ctvio::kPriorX0] = 32 * nb;
  b[ctvio::kImuT] = 16 * uint64_t(m.n_imu);
  b[ctvio::kImuGa] = 48 * uint64_t(m.n_imu);
  b[ctvio::kImuCarry] = 24;
  b[ctvio::kFtId] = b[ctvio::kFtAnchor] = b[ctvio::kFtMask] = b[ctvio::kFtLm] = 4 * ne;
  b[ctvio::kFtRho] = b[ctvio::kFtKey] = 8 * ne;
  b[ctvio::kFtIdx] = 4 * ne * ctvio::kSlots;
  uint64_t pts = 0;
  for (int s = 0; s < ctvio::kSlots; ++s)
    if (m.held >> s & 1u) pts += uint64_t(m.frame_n[s]);
  b[ctvio::kClouds] = sizeof(ctvio::FrameFeature) * pts;
  uint64_t at = sizeof(CkptHeader);
  for (int k = 0; k < kSections; ++k) {
    L.off[k] = at;
    at = align8(at + b[k]);
  }
  L.length = at;
  return L;
}

// the checksum terms of the body bytes [from, to) of a host-side blob
unsigned long long host_sum(const unsigned char* blob, uint64_t from, uint64_t to) {
  unsigned long long s = 0;
  for (uint64_t o = from; o < to; o += 8) {
    unsigned long long w;
    std::memcpy(&w, blob + o, 8);
    s += ctvio::ckpt_mix(w, (o - sizeof(CkptHeader)) >> 3);
  }
  return s;
}

// the device sections' segments: src (pack) or dst (commit) pointers into the engine's buffers, in blob order
int make_segments(ctvio_engine* e, const CkptMeta& m, const Layout& L, CkptArgs& a) {
  auto& t = e->ft;
  DevState& x = e->x[e->cur];
  auto u8 = [](const void* p) { return const_cast<unsigned char*>(static_cast<const unsigned char*>(p)); };
  unsigned char* ptr[kSections] = {};
  ptr[ctvio::kKnotQ] = u8(x.q.p); ptr[ctvio::kKnotP] = u8(x.p.p); ptr[ctvio::kBias] = u8(x.bias.p); ptr[ctvio::kRho] = u8(x.rho.p);
  ptr[ctvio::kLineDelay] = u8(x.ld.p);
  ptr[ctvio::kPriorJ] = u8(e->d_prior_J.p); ptr[ctvio::kPriorR] = u8(e->d_prior_r.p); ptr[ctvio::kPriorX0] = u8(e->d_prior_x0.p);
  ptr[ctvio::kImuT] = u8(e->d_imu_tab_t.p); ptr[ctvio::kImuGa] = u8(e->d_imu_tab_ga.p); ptr[ctvio::kImuCarry] = u8(e->cyc.imu_carry.p);
  ptr[ctvio::kFtId] = u8(t.id.p); ptr[ctvio::kFtAnchor] = u8(t.anchor.p); ptr[ctvio::kFtMask] = u8(t.mask.p);
  ptr[ctvio::kFtLm] = u8(t.lm.p); ptr[ctvio::kFtRho] = u8(t.rho.p); ptr[ctvio::kFtKey] = u8(t.key[t.cur_key].p);
  ptr[ctvio::kFtIdx] = u8(t.idx.p);
  a.n_seg = 0;
  auto add = [&](unsigned char* p, uint64_t off, uint64_t bytes, int32_t kind) {
    if (!bytes) return;
    CkptSeg& s = a.seg[a.n_seg++];
    s.ptr = p; s.off = off; s.bytes = bytes; s.kind = kind; s.pad = 0;
  };
  for (int k = ctvio::kFirstDeviceSection; k < ctvio::kClouds; ++k)
    add(ptr[k], L.off[k], L.bytes[k], k == ctvio::kFtIdx ? ctvio::kIdx : k == ctvio::kKnotP ? ctvio::kPositions : ctvio::kCopy);
  uint64_t at = L.off[ctvio::kClouds];
  for (int s = 0; s < ctvio::kSlots; ++s) {
    if (!(m.held >> s & 1u)) continue;
    const uint64_t bytes = sizeof(ctvio::FrameFeature) * uint64_t(m.frame_n[s]);
    add(u8(e->d_frames.p + size_t(s) * ctvio_engine::kFrameCap), at, bytes, ctvio::kCloud);
    at += bytes;
  }
  for (int k = 0; k < a.n_seg; ++k)
    if (!a.seg[k].ptr) return fail(CTVIO_ERR_STATE, "a buffer of the run is not allocated");
  a.n_entries = m.n_entries;
  a.mask = t.mask.p;
  return CTVIO_OK;
}

// scratch of one blob of `length` bytes: device and pinned staging, partial sums, ticket, verdict
int reserve_scratch(ctvio_engine* e, uint64_t length) {
  auto& w = e->ckpt;
  CUDA_OK(w.stage.reserve(length));
  CUDA_OK(w.partial.reserve(ctvio::kCkptMaxBlocks));
  if (!w.ticket.p) {
    CUDA_OK(w.ticket.reserve(1));
    CUDA_OK(cudaMemsetAsync(w.ticket.p, 0, sizeof(int32_t), e->stream));
  }
  if (w.h_cap < length) {
    if (w.h_stage) cudaFreeHost(w.h_stage);
    w.h_stage = nullptr;
    w.h_cap = 0;
    if (cudaHostAlloc(reinterpret_cast<void**>(&w.h_stage), length + length / 4, cudaHostAllocDefault) != cudaSuccess) {
      cudaGetLastError();
      return fail(CTVIO_ERR_CUDA, "could not allocate the pinned checkpoint buffer");
    }
    w.h_cap = length + length / 4;
  }
  if (!w.h_verdict) {
    if (cudaHostAlloc(reinterpret_cast<void**>(&w.h_verdict), sizeof(int32_t), cudaHostAllocMapped) != cudaSuccess) {
      cudaGetLastError();
      return fail(CTVIO_ERR_CUDA, "could not allocate the mapped verdict");
    }
  }
  return CTVIO_OK;
}

int grid_for(uint64_t bytes) {
  const uint64_t words = bytes / 8;
  return int(std::max<uint64_t>(1, std::min<uint64_t>(ctvio::kCkptMaxBlocks, (words + ctvio::kCkptThreads - 1) / ctvio::kCkptThreads)));
}

// the run's counts and host bookkeeping
CkptMeta meta_of(const ctvio_engine* e) {
  CkptMeta m;
  std::memset(&m, 0, sizeof(m));
  const auto& c = e->cyc;
  const auto& t = e->ft;
  m.nK = e->nK; m.nB = e->nB; m.nL = e->nL;
  m.prior_n = std::max(e->prior.n, 0);
  m.prior_nb = m.prior_n > 0 ? int32_t(e->prior.type.size()) : 0;
  m.prior_enabled = e->prior_enabled ? 1 : 0;
  m.n_imu = int32_t(e->h_imu_tab_t.size());
  m.n_entries = t.n_entries; m.held = t.held;
  m.ft_n_lm = t.n_lm; m.ft_n_obs = t.n_obs; m.ft_oldest_slot = t.oldest_slot;
  m.n_frames = c.n_frames;
  m.t0_ns = e->cfg.t0_ns;
  m.next_frame = c.next_frame;
  for (int k = 0; k < c.n_frames; ++k) { m.slot[k] = c.slot[k]; m.t[k] = c.t[k]; }
  for (int s = 0; s < ctvio::kSlots; ++s)
    if (t.held >> s & 1u) { m.frame_n[s] = e->h_frame_n[s]; m.frame_t[s] = e->h_frame_t[s]; }
  m.cfg = e->cfg;
  m.cfg.device = 0;
  m.cfg.reserved = 0;
  m.opt = c.opt;
  return m;
}

bool same_bits(const void* a, const void* b, size_t n) { return std::memcmp(a, b, n) == 0; }

// the configuration fields that must match (all but t0_ns, which the run moves, device and reserved)
bool same_config(const ctvio_config& a, const ctvio_config& b) {
  return a.dt_ns == b.dt_ns && same_bits(a.q_CtoI, b.q_CtoI, sizeof(a.q_CtoI)) && same_bits(a.p_CinI, b.p_CinI, sizeof(a.p_CinI)) &&
         same_bits(&a.image_weight, &b.image_weight, 8) && same_bits(a.gravity, b.gravity, sizeof(a.gravity)) &&
         same_bits(a.imu_info, b.imu_info, sizeof(a.imu_info)) && a.rs_padding_ns == b.rs_padding_ns &&
         same_bits(&a.cauchy_solve, &b.cauchy_solve, 8) && same_bits(&a.cauchy_marg, &b.cauchy_marg, 8);
}

int bad(const std::string& why) { return fail(CTVIO_ERR_INVALID, "ctvio_odometry_restore: " + why); }

// Everything of the blob the host can check before the device sees it: header, counts, bookkeeping, configuration,
// the prior's block lists, the section table.
int parse_blob(const ctvio_engine* e, const unsigned char* b, int64_t len, CkptHeader& h, CkptMeta& m, Layout& L) {
  if (len < int64_t(sizeof(CkptHeader) + sizeof(CkptMeta))) return bad("the blob is shorter than its header");
  std::memcpy(&h, b, sizeof(h));
  if (h.magic != ctvio::kCkptMagic) return bad("not a checkpoint (bad magic number)");
  if (h.format_version != ctvio::kCkptFormat)
    return bad("format version " + std::to_string(h.format_version) + " (this library reads version 1 only)");
  if (h.abi_version != CTVIO_ABI_VERSION) return bad("written by C-ABI version " + std::to_string(h.abi_version));
  if (h.length != uint64_t(len)) return bad("the length differs from the blob's own (truncated or padded)");
  if (h.n_sections != uint32_t(kSections)) return bad("bad section table");
  std::memcpy(&m, b + sizeof(CkptHeader), sizeof(m));
  if (!same_config(m.cfg, e->cfg)) return bad("the configuration differs from the engine's");
  if ((m.t0_ns - e->cfg.t0_ns) % e->cfg.dt_ns != 0) return bad("the time origin is off the engine's knot grid");
  const bool counts_ok = m.nK >= 4 && m.nK <= (1 << 24) && m.nB >= 1 && m.nB <= (1 << 16) && m.nL >= 0 &&
                         m.nL <= ctvio::kFeatureTableMaxEntries && m.prior_n >= 0 && m.prior_n <= (1 << 14) &&
                         m.prior_nb >= 0 && m.prior_nb <= (1 << 14) && (m.prior_n > 0) == (m.prior_nb > 0) &&
                         (m.prior_enabled == 0 || m.prior_enabled == 1) && m.n_imu >= 0 && m.n_imu <= (1 << 26) &&
                         m.n_entries >= 0 && m.n_entries <= ctvio::kFeatureTableMaxEntries && (m.held >> ctvio::kSlots) == 0 &&
                         m.ft_n_lm == m.nL && m.ft_n_obs >= 0 && m.ft_oldest_slot >= 0 && m.ft_oldest_slot < ctvio::kSlots &&
                         m.n_frames >= 1 && m.n_frames <= ctvio::kSlots && m.next_frame >= m.n_frames;
  if (!counts_ok) return bad("counts out of range");
  uint32_t listed = 0;
  for (int k = 0; k < m.n_frames; ++k) {
    const int s = m.slot[k];
    if (s < 0 || s >= ctvio::kSlots || (listed >> s & 1u)) return bad("bad frame slot list");
    listed |= 1u << s;
  }
  if (listed != m.held) return bad("the window's frame slots are not the slots the feature table holds");
  for (int s = 0; s < ctvio::kSlots; ++s) {
    const bool held = m.held >> s & 1u;
    if (m.frame_n[s] < 0 || m.frame_n[s] > ctvio_engine::kFrameCap || (!held && (m.frame_n[s] || m.frame_t[s])))
      return bad("bad frame slot counts");
  }
  if (check_cycle_options(&m.opt)) return bad("bad cycle options (" + g_err + ")");
  L = layout_of(m);
  if (L.length != h.length) return bad("the length differs from the one the counts give");
  for (int k = 0; k < kSections; ++k)
    if (h.section[k].offset != L.off[k] || h.section[k].bytes != L.bytes[k]) return bad("bad section table");
  // the prior's blocks: types, indices and columns as ctvio_set_prior and the solve's preparation check them
  // (a prior never holds an inverse depth: block_base rejects it with the out-of-range types and indices)
  std::vector<int32_t> blk(3 * size_t(m.prior_nb));  // type | index | col
  if (!blk.empty()) std::memcpy(blk.data(), b + L.off[ctvio::kPriorBlocks], blk.size() * sizeof(int32_t));
  const int32_t *type = blk.data(), *index = type + m.prior_nb, *col = index + m.prior_nb;
  for (int k = 0; k < m.prior_nb; ++k)
    if (ctvio::block_base(type[k], index[k], m.nK, m.nB) < 0) return bad("bad prior block");
  if (ctvio::prior_tiling_error(m.prior_n, m.prior_nb, type, col)) return bad("bad prior block");
  return CTVIO_OK;
}

}  // namespace

extern "C" {

int ctvio_odometry_checkpoint(ctvio_handle e, void* buf, int64_t capacity, int64_t* len) {
  if (!len) return fail(CTVIO_ERR_INVALID, "null len");
  if (capacity < 0) return fail(CTVIO_ERR_INVALID, "capacity must be >= 0");
  if (!e) return fail(CTVIO_ERR_INVALID, "null handle");
  if (e->world > 1) return fail(CTVIO_ERR_STATE, "the odometry cycle runs on a single engine, not sharded");
  if (!e->cyc.started)
    return fail(CTVIO_ERR_STATE, "no run to checkpoint: ctvio_odometry_start has not run, or the last cycle stopped on an error");
  if (e->prior.n > 0 && !e->prior_on_device)
    return fail(CTVIO_ERR_STATE, "the active prior was set by ctvio_set_prior, not by the cycle");
  const CkptMeta m = meta_of(e);
  const Layout L = layout_of(m);
  *len = int64_t(L.length);
  if (!buf) return CTVIO_OK;
  if (capacity < int64_t(L.length)) return fail(CTVIO_ERR_INVALID, "capacity is smaller than the checkpoint");
  cudaSetDevice(e->cfg.device);
  if (const int rc = reserve_scratch(e, L.length)) return rc;
  auto& w = e->ckpt;
  CkptArgs a;
  std::memset(&a, 0, sizeof(a));
  if (const int rc = make_segments(e, m, L, a)) return rc;
  a.blob = w.stage.p;
  a.begin = L.off[ctvio::kFirstDeviceSection];
  a.end = L.length;
  a.body = sizeof(CkptHeader);
  a.partial = w.partial.p;
  a.ticket = w.ticket.p;
  const int grid = grid_for(a.end - a.begin);
  ctvio::checkpoint_pack_kernel<<<grid, ctvio::kCkptThreads, 0, e->stream>>>(a);
  CUDA_OK(cudaGetLastError());
  ++e->launches;
  CUDA_OK(cudaMemcpyAsync(w.h_stage, w.stage.p, L.length, cudaMemcpyDeviceToHost, e->stream));
  CUDA_OK(stream_sync(e->stream));
  e->d2h_bytes += L.length;
  // the host-written part: header, counts and bookkeeping, the prior's block lists; then the whole checksum
  unsigned char* b = w.h_stage;
  unsigned long long dev_sum;
  std::memcpy(&dev_sum, b + offsetof(CkptHeader, checksum), 8);
  std::memset(b, 0, L.off[ctvio::kFirstDeviceSection]);
  std::memcpy(b + L.off[ctvio::kMeta], &m, sizeof(m));
  int32_t* blk = reinterpret_cast<int32_t*>(b + L.off[ctvio::kPriorBlocks]);
  const size_t nb = size_t(m.prior_nb);
  if (nb) {
    std::memcpy(blk, e->prior.type.data(), 4 * nb);
    std::memcpy(blk + nb, e->prior.index.data(), 4 * nb);
    std::memcpy(blk + 2 * nb, e->prior.col.data(), 4 * nb);
  }
  CkptHeader h;
  std::memset(&h, 0, sizeof(h));
  h.magic = ctvio::kCkptMagic;
  h.format_version = ctvio::kCkptFormat;
  h.abi_version = CTVIO_ABI_VERSION;
  h.length = L.length;
  h.n_sections = kSections;
  for (int k = 0; k < kSections; ++k) h.section[k] = ctvio::SectionEntry{L.off[k], L.bytes[k]};
  h.checksum = dev_sum + host_sum(b, sizeof(CkptHeader), L.off[ctvio::kFirstDeviceSection]);
  std::memcpy(b, &h, sizeof(h));
  std::memcpy(buf, b, L.length);
  return CTVIO_OK;
}

int ctvio_odometry_restore(ctvio_handle e, const void* buf, int64_t len) {
  if (len < 0) return fail(CTVIO_ERR_INVALID, "len must be >= 0");
  if (!buf && len > 0) return fail(CTVIO_ERR_INVALID, "null buffer");
  if (!e) return fail(CTVIO_ERR_INVALID, "null handle");
  if (e->world > 1) return fail(CTVIO_ERR_STATE, "the odometry cycle runs on a single engine, not sharded");
  const unsigned char* src = static_cast<const unsigned char*>(buf);
  CkptHeader h;
  CkptMeta m;
  Layout L;
  if (const int rc = parse_blob(e, src, len, h, m, L)) return rc;
  cudaSetDevice(e->cfg.device);
  if (const int rc = reserve_scratch(e, L.length)) return rc;
  auto& w = e->ckpt;
  // one copy up, then the device's checks into the scratch: the engine's run is untouched until they pass
  std::memcpy(w.h_stage, src, L.length);
  CUDA_OK(cudaMemcpyAsync(w.stage.p, w.h_stage, L.length, cudaMemcpyHostToDevice, e->stream));
  e->h2d_bytes += L.length;
  CkptArgs a;
  std::memset(&a, 0, sizeof(a));
  a.blob = w.stage.p;
  a.begin = sizeof(CkptHeader);
  a.end = L.length;
  a.body = sizeof(CkptHeader);
  a.partial = w.partial.p;
  a.ticket = w.ticket.p;
  a.verdict = w.h_verdict;
  for (int k = 0; k < kSections; ++k) a.expect[k] = L.bytes[k];
  *w.h_verdict = -1;
  ctvio::checkpoint_unpack_kernel<false><<<grid_for(a.end - a.begin), ctvio::kCkptThreads, 0, e->stream>>>(a);
  CUDA_OK(cudaGetLastError());
  ++e->launches;
  CUDA_OK(stream_sync(e->stream));
  e->d2h_bytes += sizeof(int32_t);
  const int verdict = *reinterpret_cast<volatile int32_t*>(w.h_verdict);
  if (verdict == 1) return bad("the section table failed the device's check");
  if (verdict != 0) return bad("checksum mismatch");
  // the blob passed: it replaces the engine's run
  e->nK = m.nK; e->sp.n_knots = m.nK;
  e->nB = m.nB; e->nL = m.nL;
  e->have_knots = e->have_bias = e->have_rho = true;
  for (int b = 0; b < 2; ++b) {
    if (const int rc = alloc_state(e, e->x[b])) return rc;
    // both inverse-depth buffers at the feature table's size, as the cycle keeps them: the next window's landmarks may
    // outnumber the blob's before the predictor solves into the other buffer
    CUDA_OK(e->x[b].rho.reserve(size_t(ctvio::kFeatureTableMaxEntries) + 1));
  }
  const size_t n = size_t(m.prior_n), nb = size_t(m.prior_nb);
  if (n) {
    CUDA_OK(e->d_prior_J.reserve(n * n)); CUDA_OK(e->d_prior_r.reserve(n)); CUDA_OK(e->d_prior_x0.reserve(4 * nb));
  }
  const size_t imu_cap = 2 * size_t(m.n_imu) + 256;
  CUDA_OK(e->d_imu_tab_t.reserve(imu_cap));
  CUDA_OK(e->d_imu_tab_ga.reserve(3 * imu_cap));
  CUDA_OK(e->cyc.imu_carry.reserve(3));
  if (const int rc = ensure_feature_table(e)) return rc;
  CUDA_OK(e->d_frame_t.reserve(ctvio_engine::kFrameSlots));
  if (const int rc = make_segments(e, m, L, a)) return rc;
  a.begin = L.off[ctvio::kFirstDeviceSection];
  ctvio::checkpoint_unpack_kernel<true><<<grid_for(a.end - a.begin), ctvio::kCkptThreads, 0, e->stream>>>(a);
  CUDA_OK(cudaGetLastError());
  ++e->launches;
  // the held slots' frame times, from the counts section already on the device
  CUDA_OK(cudaMemcpyAsync(e->d_frame_t.p, w.stage.p + L.off[ctvio::kMeta] + offsetof(CkptMeta, frame_t),
                          ctvio::kSlots * sizeof(int64_t), cudaMemcpyDeviceToDevice, e->stream));
  // the host's bookkeeping
  e->cfg.t0_ns = m.t0_ns;
  e->sp.t0_ns = m.t0_ns;
  const int32_t* blk = reinterpret_cast<const int32_t*>(src + L.off[ctvio::kPriorBlocks]);
  e->prior = ctvio::PriorHost();
  e->prior.n = m.prior_n;
  e->prior.type.resize(nb); e->prior.index.resize(nb); e->prior.col.resize(nb);
  if (nb) {
    std::memcpy(e->prior.type.data(), blk, 4 * nb);
    std::memcpy(e->prior.index.data(), blk + nb, 4 * nb);
    std::memcpy(e->prior.col.data(), blk + 2 * nb, 4 * nb);
  }
  e->prior_on_device = n > 0;
  e->prior_enabled = m.prior_enabled != 0;
  e->new_prior = ctvio::PriorHost();  // ctvio_get_prior: nothing until the next marginalization
  e->new_prior_on_host = false;
  e->h_imu_tab_t.resize(size_t(m.n_imu));
  for (int k = 0; k < m.n_imu; ++k) std::memcpy(&e->h_imu_tab_t[size_t(k)], src + L.off[ctvio::kImuT] + 16 * size_t(k), 8);
  auto& t = e->ft;
  t.n_entries = m.n_entries; t.held = m.held; t.n_lm = m.ft_n_lm; t.n_obs = m.ft_n_obs; t.oldest_slot = m.ft_oldest_slot;
  t.window_current = false;
  for (int s = 0; s < ctvio::kSlots; ++s) { e->h_frame_n[s] = m.frame_n[s]; e->h_frame_t[s] = m.frame_t[s]; }
  e->h_frame_ingested = m.held;
  auto& c = e->cyc;
  c.opt = m.opt;
  c.n_frames = m.n_frames;
  c.next_frame = m.next_frame;
  for (int k = 0; k < ctvio::kSlots; ++k) { c.slot[k] = m.slot[k]; c.t[k] = m.t[k]; }
  c.started = true;
  auto& cv = c.cov;  // the last cycle's publications are not part of the run
  cv.ran = false;
  cv.requested = (m.opt.publish_pose_covariance ? 1 : 0) | (m.opt.publish_odometry_covariance ? 2 : 0) |
                 (m.opt.publish_map_covariance ? 4 : 0);
  cv.available = 0;
  cv.status = CTVIO_ERR_STATE;
  cv.rcond = NAN;
  cv.n_frames = cv.n_lm = cv.n_map = cv.n_map_nan = 0;
  cv.pending = false;
  cv.why = "no odometry cycle has run since ctvio_odometry_restore";
  // derived data is rebuilt by the next call
  ctvio_clear_factors(e);
  e->structure_dirty = e->masks_dirty = e->prior_dirty = true;
  e->table_valid = false;
  e->mirror_valid = false;
  e->n_marg_img = -1;
  return CTVIO_OK;
}

}  // extern "C"
