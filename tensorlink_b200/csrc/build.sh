#!/usr/bin/env bash
# Build libtensorlink_b200.so in-tree for sm_90a (H100).
set -euo pipefail
here="$(cd "$(dirname "${BASH_SOURCE[0]}")" && pwd)"
out="$here/libtensorlink_b200.so"
srcs=("$here"/*.cu)
objs=()
arch=sm_90a
objdir="$here/build/$arch"     # objects of another architecture are never relinked
mkdir -p "$objdir"
pids=()
for s in "${srcs[@]}"; do
  o="$objdir/$(basename "${s%.cu}").o"
  objs+=("$o")
  if [[ ! -f "$o" || "$s" -nt "$o" || "${BASH_SOURCE[0]}" -nt "$o" || "$here/common.cuh" -nt "$o" || "$here/gemm_common.cuh" -nt "$o" || "$here/fp8.cuh" -nt "$o" || "$here/../../include/tensorlink_b200.h" -nt "$o" ]]; then
    nvcc -gencode arch=compute_90a,code=$arch -O3 -std=c++17 -lineinfo -Xcompiler -fPIC \
         ${TL_NVCC_EXTRA:-} -c "$s" -o "$o" &
    pids+=($!)
  fi
done
for p in "${pids[@]:-}"; do [[ -n "$p" ]] && wait "$p"; done
nvcc -shared -o "$out" "${objs[@]}" -lcudart
echo "built $out"
