#!/usr/bin/env bash
# Builds lidiff_b200/_C/liblidiff_b200.so for sm_90a (cross-compiles without a GPU).
set -euo pipefail
here="$(cd "$(dirname "$0")" && pwd)"
out="$here/../_C"
mkdir -p "$out"
NVCC=${NVCC:-/usr/local/cuda/bin/nvcc}
FLAGS=(-gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -std=c++17 -Xcompiler -fPIC -Xptxas -v)
objs=()
for f in coords spconv_ffma spconv_tc spconv_wgrad spconv_scatter dense metrics gate_grad sync_bn maps samples rng render mesh ssc api; do
  src="$here/$f.cu"; obj="$out/$f.o"
  # this script is a dependency too: a change of FLAGS (e.g. the target architecture) rebuilds every object
  if [ ! -f "$obj" ] || [ "$src" -nt "$obj" ] || [ "$here/common.cuh" -nt "$obj" ] || [ "$here/tc_common.cuh" -nt "$obj" ] || [ "$here/../../include/lidiff_b200.h" -nt "$obj" ] || [ "$here/build.sh" -nt "$obj" ]; then
    "$NVCC" "${FLAGS[@]}" -c "$src" -o "$obj" 2> "$out/$f.ptxas.log" || { cat "$out/$f.ptxas.log"; exit 1; }
  fi
  objs+=("$obj")
done
"$NVCC" -shared -gencode arch=compute_90a,code=sm_90a -o "$out/liblidiff_b200.so" "${objs[@]}" -lcudart
echo "built $out/liblidiff_b200.so"
