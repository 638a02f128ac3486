#!/usr/bin/env bash
# Builds libaniportrait_b200.so (sm_90a only) in-tree next to the sources. Called by __graft_entry__.build().
set -euo pipefail
cd "$(dirname "$0")"
NVCC=${NVCC:-/usr/local/cuda/bin/nvcc}
OUT=../libaniportrait_b200.so
FLAGS=(-gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -std=c++17 -Xcompiler -fPIC -Xcompiler -Wall
       --expt-relaxed-constexpr -Xptxas -v -cudart static)
mkdir -p build
objs=()
pids=()
for src in *.cu; do
  obj=build/${src%.cu}.o
  objs+=("$obj")
  if [[ ! -f "$obj" || "$src" -nt "$obj" || ap_ptx.cuh -nt "$obj" || ap_wgmma.cuh -nt "$obj" || ap_u8.cuh -nt "$obj" || ap_host.h -nt "$obj" || ../../include/aniportrait_b200.h -nt "$obj" ]]; then
    ( "$NVCC" "${FLAGS[@]}" -c "$src" -o "$obj" > "build/${src%.cu}.log" 2>&1 || { cat "build/${src%.cu}.log"; exit 1; } ) &
    pids+=($!)
  fi
done
for p in "${pids[@]:-}"; do [[ -n "$p" ]] && wait "$p"; done
"$NVCC" -shared -cudart static -o "$OUT" "${objs[@]}"
echo "built $OUT"
