#!/bin/bash
# Builds libseg_b200.so (the C-ABI shared library) for sm_90a (H100), in-tree.
set -e
HERE="$(cd "$(dirname "$0")" && pwd)"
OUT="$HERE/libseg_b200.so"
NVCC="${NVCC:-/usr/local/cuda/bin/nvcc}"
FLAGS="-gencode arch=compute_90a,code=sm_90a -lineinfo -O3 -std=c++17 -Xcompiler -fPIC --expt-relaxed-constexpr"
mkdir -p "$HERE/build"
pids=()
for f in seg_api seg_conv_tc seg_conv_simt seg_elementwise seg_loss seg_comm seg_dwconv seg_lovasz seg_data seg_score; do
  if [ -f "$HERE/csrc/$f.cu" ]; then
    if [ ! -f "$HERE/build/$f.o" ] || [ "$HERE/csrc/$f.cu" -nt "$HERE/build/$f.o" ] || [ -n "$(find "$HERE/csrc" "$HERE/../include" -name '*.cuh' -newer "$HERE/build/$f.o" -o -name '*.h' -newer "$HERE/build/$f.o" 2>/dev/null)" ]; then
      $NVCC $FLAGS ${SEG_PTXAS_V:+-Xptxas -v} -c "$HERE/csrc/$f.cu" -o "$HERE/build/$f.o" &
      pids+=($!)
    fi
  fi
done
for p in "${pids[@]}"; do wait $p; done
$NVCC -shared -gencode arch=compute_90a,code=sm_90a -o "$OUT" "$HERE"/build/*.o -lcudart_static -lpthread -ldl -lrt
echo "built $OUT"
