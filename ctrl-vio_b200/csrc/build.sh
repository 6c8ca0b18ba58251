#!/usr/bin/env bash
# Build libctvio_b200.so in-tree for sm_90a (H100).  nvcc cross-compiles without a GPU.
# Every object is rebuilt when its source, ANY header of this directory, the public C-ABI header or this script is
# newer than it (the header set is globbed, so a new .cuh / .h can not be forgotten in a dependency list).
set -euo pipefail
cd "$(dirname "$0")"
OUT=libctvio_b200.so
SRCS="engine.cu kernels_residual.cu kernels_linear.cu chol_coop.cu chol_dag.cu misc_kernels.cu marginalize.cu jacobi_blocked.cu frontend.cu comm.cu"
HDRS="$(ls *.h *.cuh) ../../include/ctvio.h build.sh"
NVCC=${NVCC:-/usr/local/cuda/bin/nvcc}
# NCCL: only <nccl.h> (types) is needed at build time; the library is dlopen'ed by comm.cu on first use.
FLAGS="${CTVIO_EXTRA_NVCC_FLAGS:-} -gencode arch=compute_90a,code=sm_90a -lineinfo -O3 -std=c++17 --expt-relaxed-constexpr -Xcompiler -fPIC -Xptxas -v"
objs=""
relink=0
[[ -f "$OUT" ]] || relink=1
pids=()
for f in $SRCS; do
  o="${f%.cu}.o"
  stale=0
  [[ -n "${CTVIO_FORCE_BUILD:-}" || ! -f "$o" || "$f" -nt "$o" ]] && stale=1
  for h in $HDRS; do [[ "$h" -nt "$o" ]] && stale=1; done
  if [[ $stale -eq 1 ]]; then
    relink=1
    ( $NVCC $FLAGS -c "$f" -o "$o" 2> "${o}.log" || { cat "${o}.log"; exit 1; } ) &
    pids+=($!)
  fi
  objs="$objs $o"
done
for p in "${pids[@]:-}"; do [[ -n "$p" ]] && wait "$p"; done
for f in $SRCS; do [[ "${f%.cu}.o" -nt "$OUT" ]] && relink=1; done
if [[ $relink -eq 1 ]]; then
  $NVCC -gencode arch=compute_90a,code=sm_90a -shared -o "$OUT" $objs -lcudart -ldl
  echo "built $OUT"
fi
