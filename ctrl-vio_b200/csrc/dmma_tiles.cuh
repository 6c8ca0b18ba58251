// 64x64 fp64 tiles on the Hopper tensor cores' fp64 path (mma.sync.m8n8k4.f64; wgmma has no fp64 kind):
// shared by the dense Cholesky (K5) and the Schur complement (K4).
#pragma once
#include "chol_tiles.cuh"

namespace ctvio {

// ---- fp64 tensor-core tiles (mma.sync.m8n8k4.f64: about the DFMA rate on H100, measured by
// ctvio_measure_fp64_tensor_tflops, at a fraction of the shared-memory operand traffic of a 4x4 register-tiled DFMA
// loop) ----
// The 64x64 tile is an 8x8 grid of m8n8 fragments.  Warp (wm, wn) = (warp & 3, warp >> 2) owns the fragment rows
// {wm, 7 - wm} and the fragment columns {0, 1, 6, 7} (wn = 0) / {2, 3, 4, 5} (wn = 1): with this folding every warp
// has the same amount of work when only the lower triangle of the product is needed (SYRK of a diagonal tile: at most
// 5 of 8 fragments per warp) or when the B operand is lower triangular (panel * Linv^T: 144 of 256 k-columns per
// warp), so those two GEMMs of the Cholesky's critical chain cost ~60 % of a full tile product.
// Lane (g, q) = (lane >> 2, lane & 3) holds C[8 rt + g][8 ct + 2 q + {0, 1}] of each fragment (rt, ct).
struct Frag {
  double c[2][4][2];
};
struct Lane {
  int rt[2], ct[4];  // fragment rows / columns of the warp
  int g, q;          // lane coordinates
  __device__ __forceinline__ int row(int mt) const { return 8 * rt[mt] + g; }
  __device__ __forceinline__ int col(int nt) const { return 8 * ct[nt] + 2 * q; }
};
__device__ __forceinline__ Lane lane_of(int tid) {
  const int warp = tid >> 5, lane = tid & 31;
  const int wm = warp & 3, wn = warp >> 2;
  Lane L;
  L.rt[0] = wm; L.rt[1] = 7 - wm;
  L.ct[0] = 2 * wn; L.ct[1] = 2 * wn + 1; L.ct[2] = wn ? 4 : 6; L.ct[3] = wn ? 5 : 7;
  L.g = lane >> 2; L.q = lane & 3;
  return L;
}
__device__ __forceinline__ void frag_zero(Frag& f) {
#pragma unroll
  for (int mt = 0; mt < 2; ++mt)
#pragma unroll
    for (int nt = 0; nt < 4; ++nt) f.c[mt][nt][0] = f.c[mt][nt][1] = 0.0;
}
enum GemmShape {
  kGemmFull = 0,
  kGemmLowerOut = 1,  // only fragments with rt >= ct are computed (C = A A^T of a diagonal tile; the rest is left as is)
  kGemmLowerB = 2,    // B is lower triangular (B[j][k] = 0 for k > j): k runs to the end of fragment column ct only
};
// k-range [k_lo, k_hi) of  f (+|-)= A * B^T  restricted to the fragment columns nt >= NT0 (branch-free inner loop)
template <bool SUB, int NT0, bool LOWER_OUT>
__device__ __forceinline__ void tile_gemm_dmma_range(const double* pa, const double* pb, Frag& f, const Lane& L, int k_lo, int k_hi) {
  bool on[2][4];
#pragma unroll
  for (int mt = 0; mt < 2; ++mt)
#pragma unroll
    for (int nt = 0; nt < 4; ++nt) on[mt][nt] = !LOWER_OUT || L.rt[mt] >= L.ct[nt];  // loop invariant, warp-uniform
#pragma unroll 4
  for (int k0 = k_lo; k0 < k_hi; k0 += 4) {
    double av[2], bv[4];
#pragma unroll
    for (int mt = 0; mt < 2; ++mt) av[mt] = SUB ? -pa[k0 * kTS + 8 * L.rt[mt]] : pa[k0 * kTS + 8 * L.rt[mt]];
#pragma unroll
    for (int nt = NT0; nt < 4; ++nt) bv[nt] = pb[k0 * kTS + 8 * L.ct[nt]];
#pragma unroll
    for (int mt = 0; mt < 2; ++mt)
#pragma unroll
      for (int nt = NT0; nt < 4; ++nt) {
        if (LOWER_OUT && !on[mt][nt]) continue;
        asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};"
                     : "+d"(f.c[mt][nt][0]), "+d"(f.c[mt][nt][1])
                     : "d"(av[mt]), "d"(bv[nt]));
      }
  }
}
// f (+|-)= A * B^T with both operands in [k][row] layout in smem (At[k][i] = A[i][k], Bt[k][j] = B[j][k])
template <bool SUB, int K = kCholNB, int SHAPE = kGemmFull>
__device__ __forceinline__ void tile_gemm_dmma(const double* At, const double* Bt, Frag& f, const Lane& L) {
  const double* pa = At + L.q * kTS + L.g;
  const double* pb = Bt + L.q * kTS + L.g;
  if (SHAPE == kGemmLowerB) {
    // fragment column ct needs k < 8 (ct + 1); the warp's columns are ascending: four k-segments, each with one
    // fragment column fewer
    const int e0 = 8 * (L.ct[0] + 1), e1 = 8 * (L.ct[1] + 1), e2 = 8 * (L.ct[2] + 1), e3 = 8 * (L.ct[3] + 1);
    tile_gemm_dmma_range<SUB, 0, false>(pa, pb, f, L, 0, e0);
    tile_gemm_dmma_range<SUB, 1, false>(pa, pb, f, L, e0, e1);
    tile_gemm_dmma_range<SUB, 2, false>(pa, pb, f, L, e1, e2);
    tile_gemm_dmma_range<SUB, 3, false>(pa, pb, f, L, e2, e3 < K ? e3 : K);
  } else {
    tile_gemm_dmma_range<SUB, 0, SHAPE == kGemmLowerOut>(pa, pb, f, L, 0, K);
  }
}
// fragments <- global tile (row-major, row stride npad; L2 path: another SM may have produced it)
__device__ __forceinline__ void frag_load_global(Frag& f, const double* tile, int npad, const Lane& L) {
#pragma unroll
  for (int mt = 0; mt < 2; ++mt)
#pragma unroll
    for (int nt = 0; nt < 4; ++nt) {
      const double2 v = __ldcg(reinterpret_cast<const double2*>(tile + size_t(L.row(mt)) * npad + L.col(nt)));
      f.c[mt][nt][0] = v.x; f.c[mt][nt][1] = v.y;
    }
}
// fragments -> smem row-major (dst[r][c])
__device__ __forceinline__ void frag_store(double* dst, const Frag& f, const Lane& L) {
#pragma unroll
  for (int mt = 0; mt < 2; ++mt)
#pragma unroll
    for (int nt = 0; nt < 4; ++nt)
      *reinterpret_cast<double2*>(dst + L.row(mt) * kTS + L.col(nt)) = make_double2(f.c[mt][nt][0], f.c[mt][nt][1]);
}
}  // namespace ctvio
