#!/bin/bash
# Builds libb200dsp.so (the product: CUDA kernels + C-ABI) in-tree for the H100 (sm_90a).
# nvcc cross-compiles without a GPU.
set -e
cd "$(dirname "$0")"
SRC=gstreamer_b200/csrc
OUT=gstreamer_b200/libb200dsp.so
NVCC=${NVCC:-/usr/local/cuda/bin/nvcc}
ARCH="-gencode arch=compute_90a,code=sm_90a"
FLAGS="$ARCH -lineinfo -O3 -std=c++17 -Xcompiler -fPIC,-O3,-Wall,-ffp-contract=off -Xptxas -v"
mkdir -p build
# objects compiled with other flags (another architecture) are stale whatever their time stamps say
if [ "$(cat build/flags 2>/dev/null)" != "$FLAGS" ]; then rm -f build/*.o; echo "$FLAGS" > build/flags; fi
OBJS=""
for f in $SRC/*.cu $SRC/*.cpp; do
  o=build/$(basename "$f").o
  if [ ! -f "$o" ] || [ -n "$(find $SRC include -newer "$o" \( -name '*.cu' -o -name '*.cuh' -o -name '*.h' -o -name '*.cpp' \) | head -1)" ]; then
    echo "nvcc $f"
    $NVCC $FLAGS -x cu -c "$f" -o "$o" 2> "build/$(basename "$f").ptxas.log" || { cat "build/$(basename "$f").ptxas.log"; exit 1; }
  fi
  OBJS="$OBJS $o"
done
$NVCC $ARCH -shared -o $OUT $OBJS -cudart static
echo "built $OUT"
