#!/usr/bin/env bash
# Build liblpb200.so (hand-written sm_90a CUDA behind a C ABI) in-tree.
set -euo pipefail
cd "$(dirname "$0")"
SRC=lightning_pose_b200/csrc
OUT=lightning_pose_b200/liblpb200.so
NVCC=${NVCC:-/usr/local/cuda/bin/nvcc}
FLAGS=(-gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -std=c++17 -Xcompiler -fPIC -Xcompiler -O3)
mkdir -p build
objs=()
pids=()
for f in $SRC/*.cu; do
  o=build/$(basename "${f%.cu}").o
  if [[ ! -f $o || $f -nt $o || -n $(find $SRC include -newer "$o" \( -name '*.cuh' -o -name '*.h' \) -print -quit) ]]; then
    echo "nvcc $f"
    rm -f "$o"  # a failed compile must break the link, never reuse a stale object
    "$NVCC" "${FLAGS[@]}" ${PTXAS_V:+-Xptxas -v} -c "$f" -o "$o" &
    pids+=($!)
  fi
  objs+=("$o")
done
for p in "${pids[@]:-}"; do
  [[ -z $p ]] || wait "$p" || { echo "build.sh: a compile failed" >&2; exit 1; }
done
"$NVCC" -shared -o "$OUT" "${objs[@]}" -lcudart
echo "built $OUT"
