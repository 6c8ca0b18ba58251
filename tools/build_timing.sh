#!/usr/bin/env bash
# debug build: libctvio_b200_timing.so = the product objects with chol_coop.cu, chol_dag.cu and kernels_residual.cu
# recompiled under -DCTVIO_CHOL_TIMING.  The object list is build.sh's SRCS, so the two libraries link the same sources.
set -euo pipefail
cd "$(dirname "$0")/../ctrl-vio_b200/csrc"
bash build.sh
NVCC=${NVCC:-/usr/local/cuda/bin/nvcc}
TIMED="chol_coop.cu chol_dag.cu kernels_residual.cu"
for f in $TIMED; do
  $NVCC -DCTVIO_CHOL_TIMING -gencode arch=compute_90a,code=sm_90a -lineinfo -O3 -std=c++17 --expt-relaxed-constexpr \
    -Xcompiler -fPIC -c "$f" -o "${f%.cu}_timing.o"
done
SRCS=$(sed -n 's/^SRCS="\(.*\)"$/\1/p' build.sh)
[[ -n "$SRCS" ]] || { echo "build_timing.sh: no SRCS line in build.sh" >&2; exit 1; }
objs=""
for f in $SRCS; do
  if [[ " $TIMED " == *" $f "* ]]; then objs="$objs ${f%.cu}_timing.o"; else objs="$objs ${f%.cu}.o"; fi
done
$NVCC -gencode arch=compute_90a,code=sm_90a -shared -o libctvio_b200_timing.so $objs -lcudart -ldl
echo "built libctvio_b200_timing.so"
