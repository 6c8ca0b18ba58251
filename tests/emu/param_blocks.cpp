// TEST INFRASTRUCTURE: compiles the engine's parameter-block rules (ctrl-vio_b200/csrc/param_blocks.h) with plain g++
// so that tests/test_param_blocks_cpu.py can check them without a GPU.  Not linked into the product library.
#include "../../ctrl-vio_b200/csrc/param_blocks.h"

extern "C" {

int pb_block_dim(int type) { return ctvio::block_dim(type); }
int pb_block_base(int type, int index, int nK, int nB) { return ctvio::block_base(type, index, nK, nB); }
int pb_block_is_knot(int type) { return ctvio::block_is_knot(type); }
int pb_block_is_bias(int type) { return ctvio::block_is_bias(type); }
int pb_prior_block_dropped(int type, int index, int now, int later) {
  return ctvio::prior_block_dropped(type, index, now, later);
}
const char* pb_prior_tiling_error(int n, int nb, const int32_t* type, const int32_t* col) {
  return ctvio::prior_tiling_error(n, nb, type, col);
}

}  // extern "C"
