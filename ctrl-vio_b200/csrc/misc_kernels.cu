// Gram matrix of the prior Jacobian (once per prior) and the line-search directional derivative.
#include "marginalize.h"

namespace ctvio {

__global__ void gram_kernel(const double* J, int rows, int cols, double* G) {
  const int i = blockIdx.y * 16 + threadIdx.y, j = blockIdx.x * 16 + threadIdx.x;
  if (i >= cols || j >= cols) return;
  double s = 0;
  for (int r = 0; r < rows; ++r) s = fma(J[size_t(r) * cols + i], J[size_t(r) * cols + j], s);
  G[size_t(i) * cols + j] = s;
}
int launch_gram(const double* J, int rows, int cols, double* G, cudaStream_t s) {
  if (cols <= 0) return 0;
  dim3 grid((cols + 15) / 16, (cols + 15) / 16), block(16, 16);
  gram_kernel<<<grid, block, 0, s>>>(J, rows, cols, G);
  return 1;
}

__global__ void dot_gradient_kernel(LinearLaunch a) {
  __shared__ double red[8];
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const int np = a.dims.np, nL = a.dims.nL;
  double v = 0;
  if (i < np) v = a.ne.gc[i] * a.dc[i];
  else if (i < np + nL) v = a.ne.gl[i - np] * a.dl[i - np];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  if (threadIdx.x == 0) {
    double s = 0;
    for (int w = 0; w < 8; ++w) s += red[w];
    if (s != 0.0) atomicAdd(&a.scal->gd, s);
  }
}
int launch_dot_gradient(const LinearLaunch& a, cudaStream_t s) {
  cudaMemsetAsync(&a.scal->gd, 0, sizeof(double), s);
  const int n = a.dims.np + a.dims.nL;
  dot_gradient_kernel<<<(n + 255) / 256, 256, 0, s>>>(a);
  return 1;
}

// sharded mode helpers
// buf =[rho masked by ownership (nL) | owned (nL)] before the all-reduce, rho <- sum / count afterwards
__global__ void rho_pack_kernel(const double* rho, const uint8_t* owned, double* buf, int nL) {
  const int l = blockIdx.x * blockDim.x + threadIdx.x;
  if (l >= nL) return;
  buf[l] = owned[l] ? rho[l] : 0.0;
  buf[nL + l] = owned[l] ? 1.0 : 0.0;
}
__global__ void rho_unpack_kernel(double* rho, const double* buf, int nL) {
  const int l = blockIdx.x * blockDim.x + threadIdx.x;
  if (l >= nL) return;
  if (buf[nL + l] > 0.0) rho[l] = buf[l] / buf[nL + l];
}
int launch_rho_pack(const double* rho, const uint8_t* owned, double* buf, int nL, cudaStream_t s) {
  if (nL <= 0) return 0;
  rho_pack_kernel<<<(nL + 255) / 256, 256, 0, s>>>(rho, owned, buf, nL);
  return 1;
}
int launch_rho_unpack(double* rho, const double* buf, int nL, cudaStream_t s) {
  if (nL <= 0) return 0;
  rho_unpack_kernel<<<(nL + 255) / 256, 256, 0, s>>>(rho, buf, nL);
  return 1;
}

// fp64 FMA micro-benchmark: 8 independent DFMA chains per thread, enough CTAs to fill every SM.
__global__ void __launch_bounds__(256) fp64_peak_kernel(double* out, int iters, double seed) {
  double a0 = seed, a1 = seed + 1, a2 = seed + 2, a3 = seed + 3, a4 = seed + 4, a5 = seed + 5, a6 = seed + 6, a7 = seed + 7;
  const double m = 1.0000001, c = 1e-9 * threadIdx.x;
  for (int i = 0; i < iters; ++i) {
    a0 = fma(a0, m, c); a1 = fma(a1, m, c); a2 = fma(a2, m, c); a3 = fma(a3, m, c);
    a4 = fma(a4, m, c); a5 = fma(a5, m, c); a6 = fma(a6, m, c); a7 = fma(a7, m, c);
  }
  out[blockIdx.x * blockDim.x + threadIdx.x] = ((a0 + a1) + (a2 + a3)) + ((a4 + a5) + (a6 + a7));
}

double measure_fp64_tflops(cudaStream_t s) {
  int dev = 0, n_sm = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, dev);
  const int ctas = n_sm * 8, iters = 1 << 15;
  double* out = nullptr;
  if (cudaMalloc(&out, size_t(ctas) * 256 * sizeof(double)) != cudaSuccess) return -1.0;
  cudaEvent_t e0, e1;
  cudaEventCreate(&e0);
  cudaEventCreate(&e1);
  float best = 1e30f;
  for (int rep = 0; rep < 5; ++rep) {
    cudaEventRecord(e0, s);
    fp64_peak_kernel<<<ctas, 256, 0, s>>>(out, iters, 1.0 + rep);
    cudaEventRecord(e1, s);
    cudaEventSynchronize(e1);
    float ms = 0;
    cudaEventElapsedTime(&ms, e0, e1);
    if (rep > 0 && ms < best) best = ms;
  }
  cudaEventDestroy(e0);
  cudaEventDestroy(e1);
  cudaFree(out);
  const double flops = 2.0 * 8.0 * double(iters) * double(ctas) * 256.0;
  return flops / (best * 1e-3) / 1e12;
}

// fp64 tensor-core micro-benchmark: every warp runs 8 independent mma.sync.m8n8k4.f64 accumulator chains (the fp64
// tensor path this library uses; wgmma has no fp64 kind).  It is a different pipe from DFMA, so the kernels built on
// DMMA (K4, K5) are measured against the rate of the instruction they issue, not against the DFMA loop above.  With
// `lat`, warp 0 of CTA 0 also times a dependent chain of 256 mma.
__device__ __forceinline__ void dmma(double& d0, double& d1, double a, double b) {
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};" : "+d"(d0), "+d"(d1) : "d"(a), "d"(b));
}
__global__ void __launch_bounds__(256) fp64_tensor_peak_kernel(double* out, int iters, double seed, long long* lat) {
  double c[8][2];
#pragma unroll
  for (int i = 0; i < 8; ++i) { c[i][0] = seed + i; c[i][1] = seed - i; }
  const double a = 1.0 + 1e-9 * threadIdx.x, b = 1e-3 + 1e-9 * threadIdx.x;
  for (int i = 0; i < iters; ++i) {
#pragma unroll
    for (int j = 0; j < 8; ++j) dmma(c[j][0], c[j][1], a, b);
  }
  double s = 0.0;
#pragma unroll
  for (int i = 0; i < 8; ++i) s += c[i][0] + c[i][1];
  if (lat && blockIdx.x == 0 && threadIdx.x < 32) {
    double d0 = s, d1 = s + 1;
    const long long t0 = clock64();
#pragma unroll 1
    for (int i = 0; i < 64; ++i) { dmma(d0, d1, a, b); dmma(d0, d1, a, b); dmma(d0, d1, a, b); dmma(d0, d1, a, b); }
    const long long t1 = clock64();
    s += d0 + d1;
    if (threadIdx.x == 0) lat[0] = t1 - t0;
  }
  out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}

double measure_fp64_tensor_tflops(cudaStream_t s, int ctas_per_sm, double* dep_latency_cycles) {
  int dev = 0, n_sm = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, dev);
  const int ctas = n_sm * ctas_per_sm, iters = 1 << 13;
  double* out = nullptr;
  long long* lat = nullptr;
  if (cudaMalloc(&out, size_t(ctas) * 256 * sizeof(double)) != cudaSuccess) return -1.0;
  if (dep_latency_cycles && cudaMalloc(&lat, sizeof(long long)) != cudaSuccess) {
    cudaFree(out);
    return -1.0;
  }
  cudaEvent_t e0, e1;
  cudaEventCreate(&e0);
  cudaEventCreate(&e1);
  float best = 1e30f;
  for (int rep = 0; rep < 5; ++rep) {
    cudaEventRecord(e0, s);
    fp64_tensor_peak_kernel<<<ctas, 256, 0, s>>>(out, iters, 1.0 + rep, lat);
    cudaEventRecord(e1, s);
    cudaEventSynchronize(e1);
    float ms = 0;
    cudaEventElapsedTime(&ms, e0, e1);
    if (rep > 0 && ms < best) best = ms;
  }
  cudaEventDestroy(e0);
  cudaEventDestroy(e1);
  if (lat) {
    long long l = 0;
    cudaMemcpy(&l, lat, sizeof(l), cudaMemcpyDeviceToHost);
    *dep_latency_cycles = double(l) / 256.0;
    cudaFree(lat);
  }
  cudaFree(out);
  if (cudaGetLastError() != cudaSuccess) return -1.0;
  // one m8n8k4 = 256 FMAs = 512 flop; 8 per warp-iteration; 8 warps per CTA
  const double flops = 512.0 * 8.0 * 8.0 * double(iters) * double(ctas);
  return flops / (best * 1e-3) / 1e12;
}


// ---- sharded mode: packed all-reduce buffer (lower-triangular tiles only: half the bytes of the dense slab) ----
size_t shard_pack_len(int npad) {
  const size_t T = npad / kCholNB;
  return T * (T + 1) / 2 * kCholNB * kCholNB + 2 * size_t(npad);
}
__global__ void shard_pack_kernel(LinearLaunch a, double* packed) {
  const int T = a.npad / kCholNB, ntile = T * (T + 1) / 2;
  const int t = blockIdx.x;
  if (t < ntile) {
    int ti = 0, rem = t;
    while (rem > ti) { rem -= ti + 1; ++ti; }
    const int tj = rem;
    const double* src = a.M + size_t(ti) * kCholNB * a.npad + tj * kCholNB;
    double* dst = packed + size_t(t) * kCholNB * kCholNB;
    for (int e = threadIdx.x; e < kCholNB * kCholNB / 2; e += blockDim.x) {
      const int r = e >> 5, c = (e & 31) * 2;
      *reinterpret_cast<double2*>(dst + r * kCholNB + c) = *reinterpret_cast<const double2*>(src + size_t(r) * a.npad + c);
    }
  } else {
    double* tail = packed + size_t(ntile) * kCholNB * kCholNB;
    for (int i = threadIdx.x; i < a.npad; i += blockDim.x) { tail[i] = a.rhs[i]; tail[a.npad + i] = a.diagA[i]; }
  }
}
__global__ void shard_unpack_kernel(LinearLaunch a, const double* packed, double radius) {
  const int T = a.npad / kCholNB, ntile = T * (T + 1) / 2;
  const int t = blockIdx.x;
  const double* tail = packed + size_t(ntile) * kCholNB * kCholNB;
  if (t < ntile) {
    int ti = 0, rem = t;
    while (rem > ti) { rem -= ti + 1; ++ti; }
    const int tj = rem;
    double* dst = a.M + size_t(ti) * kCholNB * a.npad + tj * kCholNB;
    const double* src = packed + size_t(t) * kCholNB * kCholNB;
    for (int e = threadIdx.x; e < kCholNB * kCholNB / 2; e += blockDim.x) {
      const int r = e >> 5, c = (e & 31) * 2;
      double2 v = *reinterpret_cast<const double2*>(src + r * kCholNB + c);
      if (ti == tj) {  // LM damping / identity rows on the diagonal (Ceres min/max_lm_diagonal 1e-6 / 1e32)
        const int i = ti * kCholNB + r;
        const bool live = i < a.dims.np && !a.cmask[i];
        if (c == r || c + 1 == r) {
          double& d = c == r ? v.x : v.y;
          if (live) {
            const double sd = a.sc[i] * a.sc[i] * tail[a.npad + i];
            d += fmin(fmax(sd, 1e-6), 1e32) / radius;
          } else {
            d = 1.0;
          }
        }
      }
      *reinterpret_cast<double2*>(dst + size_t(r) * a.npad + c) = v;
    }
  } else {
    for (int i = threadIdx.x; i < a.npad; i += blockDim.x) {
      const bool live = i < a.dims.np && !a.cmask[i];
      a.rhs[i] = live ? tail[i] : 0.0;
      a.diagA[i] = tail[a.npad + i];
    }
  }
}
int launch_shard_pack(const LinearLaunch& a, double* packed, cudaStream_t s) {
  const int T = a.npad / kCholNB;
  shard_pack_kernel<<<T * (T + 1) / 2 + 1, 256, 0, s>>>(a, packed);
  return 1;
}
int launch_shard_unpack(const LinearLaunch& a, const double* packed, double radius, cudaStream_t s) {
  const int T = a.npad / kCholNB;
  shard_unpack_kernel<<<T * (T + 1) / 2 + 1, 256, 0, s>>>(a, packed, radius);
  return 1;
}
__global__ void shard_scalars_pack_kernel(LmScalars* scal, double* send8) {
  send8[0] = scal->cost_eval; send8[1] = scal->gd; send8[2] = scal->dHd; send8[3] = scal->step_norm2;
  send8[4] = scal->x_norm2; send8[5] = (scal->error_flags != 0) ? 1.0 : 0.0; send8[6] = scal->gmax; send8[7] = scal->dir_max;
}
__global__ void shard_scalars_reduce_kernel(const double* g, int world, LmScalars* scal, LmPublished* pub, unsigned long long seq) {
  double sum[6] = {0, 0, 0, 0, 0, 0}, mx[2] = {0, 0};
  for (int r = 0; r < world; ++r) {  // fixed order: every rank gets bit-identical scalars
    for (int k = 0; k < 6; ++k) sum[k] += g[8 * r + k];
    mx[0] = fmax(mx[0], g[8 * r + 6]);
    mx[1] = fmax(mx[1], g[8 * r + 7]);
  }
  scal->cost_eval = sum[0]; scal->gd = sum[1]; scal->dHd = sum[2]; scal->step_norm2 = sum[3]; scal->x_norm2 = sum[4];
  scal->err_sum = sum[5]; scal->gmax = mx[0]; scal->dir_max = mx[1];
  if (pub) {
    LmScalars out = *scal;
    pub->s = out;
    __threadfence_system();
    *reinterpret_cast<volatile unsigned long long*>(&pub->seq) = seq;
  }
}
int launch_shard_scalars_pack(LmScalars* scal, double* send8, cudaStream_t s) {
  shard_scalars_pack_kernel<<<1, 1, 0, s>>>(scal, send8);
  return 1;
}
int launch_shard_scalars_reduce(const double* gathered, int world, LmScalars* scal, LmPublished* pub, unsigned long long seq,
                                cudaStream_t s) {
  shard_scalars_reduce_kernel<<<1, 1, 0, s>>>(gathered, world, scal, pub, seq);
  return 1;
}


// ResidualSummary support: out[c] = sum_k |r[k][c]| (one CTA, fixed order), and the bias random-walk residuals
__global__ void abs_column_sums_kernel(const double* r, int n, int cols, double* out) {
  __shared__ double part[32][8];
  const int c = threadIdx.x & 7, g = threadIdx.x >> 3;  // 8 column slots x 32 row groups
  double s = 0.0;
  if (c < cols)
    for (int k = g; k < n; k += 32) s += fabs(r[size_t(k) * cols + c]);
  part[g][c] = s;
  __syncthreads();
  if (threadIdx.x < cols) {
    double t = 0.0;
    for (int k = 0; k < 32; ++k) t += part[k][threadIdx.x];
    out[threadIdx.x] = t;
  }
}
int launch_abs_column_sums(const double* r, int n, int cols, double* out, cudaStream_t s) {
  if (n <= 0 || cols > 8) return 0;
  abs_column_sums_kernel<<<1, 256, 0, s>>>(r, n, cols, out);
  return 1;
}
__global__ void bias_abs_sums_kernel(const int2* ij, const double* sq, int n, const double* bias, double* out6) {
  const int c = threadIdx.x;
  if (c >= 6) return;
  double t = 0.0;
  for (int k = 0; k < n; ++k) t += fabs(sq[6 * k + c] * (bias[6 * ij[k].y + c] - bias[6 * ij[k].x + c]));
  out6[c] = t;
}
int launch_bias_abs_sums(const int2* ij, const double* sq, int n, const double* bias, double* out6, cudaStream_t s) {
  if (n <= 0) return 0;
  bias_abs_sums_kernel<<<1, 32, 0, s>>>(ij, sq, n, bias, out6);
  return 1;
}

}  // namespace ctvio
