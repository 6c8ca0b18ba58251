#!/usr/bin/env bash
# debug build: libctvio_b200_timing.so = the product objects with chol_coop.cu recompiled under -DCTVIO_CHOL_TIMING
set -euo pipefail
cd "$(dirname "$0")/../ctrl-vio_b200/csrc"
bash build.sh
NVCC=${NVCC:-/usr/local/cuda/bin/nvcc}
$NVCC -DCTVIO_CHOL_TIMING -gencode arch=compute_90a,code=sm_90a -lineinfo -O3 -std=c++17 --expt-relaxed-constexpr \
  -Xcompiler -fPIC -c chol_coop.cu -o chol_coop_timing.o
$NVCC -DCTVIO_CHOL_TIMING -gencode arch=compute_90a,code=sm_90a -lineinfo -O3 -std=c++17 --expt-relaxed-constexpr \
  -Xcompiler -fPIC -c chol_dag.cu -o chol_dag_timing.o
$NVCC -DCTVIO_CHOL_TIMING -gencode arch=compute_90a,code=sm_90a -lineinfo -O3 -std=c++17 --expt-relaxed-constexpr \
  -Xcompiler -fPIC -c kernels_residual.cu -o kernels_residual_timing.o
$NVCC -gencode arch=compute_90a,code=sm_90a -shared -o libctvio_b200_timing.so engine.o resident.o solve.o kernels_residual_timing.o \
  kernels_linear.o chol_coop_timing.o chol_dag_timing.o misc_kernels.o marginalize.o jacobi_blocked.o frontend.o comm.o -lcudart -ldl
echo "built libctvio_b200_timing.so"
