// The rules of a prior or marginalization parameter block (type, index), type one of CTVIO_BLK_* (include/ctvio.h):
// its tangent size, its first camera dim, its kind, whether the marginalization drops it from the old prior, and the
// check that a prior's blocks tile its columns.  Host and device; compiles with plain g++ (tests/test_param_blocks_cpu.py).
#pragma once
#include <cstdint>
#include <vector>

#include "../../include/ctvio.h"
#include "device_math.cuh"  // CTVIO_HD

namespace ctvio {

// tangent size: 3, or 1 for the line delay and an inverse depth
CTVIO_HD int block_dim(int type) {
  if (type == CTVIO_BLK_LD || type == CTVIO_BLK_RHO) return 1;
  return 3;
}

CTVIO_HD bool block_is_knot(int type) { return type == CTVIO_BLK_ROT || type == CTVIO_BLK_POS; }
CTVIO_HD bool block_is_bias(int type) { return type == CTVIO_BLK_BG || type == CTVIO_BLK_BA; }

// first camera dim of a block (np = 6 nK + 6 nB + 1: rot, pos per knot, then bg, ba per bias node, then the line delay),
// -1 if it has none (an inverse depth) or its index is out of range.  For blocks in range, the order of their first
// camera dims is the marginalization's block order.
CTVIO_HD int block_base(int type, int index, int nK, int nB) {
  const bool knot = index >= 0 && index < nK, node = index >= 0 && index < nB;
  switch (type) {
    case CTVIO_BLK_ROT: return knot ? 6 * index : -1;
    case CTVIO_BLK_POS: return knot ? 6 * index + 3 : -1;
    case CTVIO_BLK_BG: return node ? 6 * nK + 6 * index : -1;
    case CTVIO_BLK_BA: return node ? 6 * nK + 6 * index + 3 : -1;
    case CTVIO_BLK_LD: return 6 * nK + 6 * nB;
    default: return -1;
  }
}

// the old prior's blocks the marginalization drops (trajectory_manager.cpp:166-203): the knots [now, later) that leave
// the window and the oldest bias node
CTVIO_HD bool prior_block_dropped(int type, int index, int now, int later) {
  return (block_is_knot(type) && index >= now && index < later) || (block_is_bias(type) && index == 0);
}

// nullptr if the nb blocks tile the n columns of a prior exactly (col[b] + c indexes host tables and device scratch),
// else the first failure: a type out of range, a block outside [0, n), an overlap, a column no block covers
inline const char* prior_tiling_error(int n, int nb, const int32_t* type, const int32_t* col) {
  std::vector<uint8_t> covered(size_t(n), 0);
  for (int b = 0; b < nb; ++b) {
    if (type[b] < CTVIO_BLK_ROT || type[b] > CTVIO_BLK_RHO) return "prior block type out of range";
    const int dim = block_dim(type[b]);
    if (col[b] < 0 || col[b] + dim > n) return "prior block column outside [0, n)";
    for (int c = 0; c < dim; ++c) {
      if (covered[size_t(col[b] + c)]) return "prior blocks overlap";
      covered[size_t(col[b] + c)] = 1;
    }
  }
  for (int c = 0; c < n; ++c)
    if (!covered[size_t(c)]) return "prior blocks do not cover all n columns";
  return nullptr;
}

}  // namespace ctvio
