#!/bin/bash
# Build libvtoonify_b200.so for sm_90a (cross-compiles without a GPU).
set -e
HERE="$(cd "$(dirname "$0")" && pwd)"
OUT="$HERE/../lib"
mkdir -p "$OUT"
NVCC=${NVCC:-/usr/local/cuda/bin/nvcc}
FLAGS="-gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -std=c++17 -Xcompiler -fPIC -Xcompiler -Wall --expt-relaxed-constexpr"
SRCS="api.cu upfirdn2d.cu elementwise.cu modulate.cu conv_direct.cu norm_fir.cu resample.cu frame_prep.cu conv_tc.cu conv_rs.cu conv_wgrad.cu lpips.cu augment.cu raft.cu smooth.cu align.cu"
OBJS=""
pids=()
for s in $SRCS; do
  [ -f "$HERE/$s" ] || { echo "build.sh: missing source $HERE/$s" >&2; exit 1; }
  o="$OUT/${s%.cu}.o"
  if [ ! -f "$o" ] || [ "$HERE/$s" -nt "$o" ] || [ "$HERE/common.cuh" -nt "$o" ] || [ "$HERE/../../include/vtoonify_b200.h" -nt "$o" ] || [ "$HERE/tc_common.cuh" -nt "$o" ] || [ "$HERE/wgmma_sm90.cuh" -nt "$o" ]; then
    $NVCC $FLAGS ${VT_PTXAS_V:+-Xptxas -v} -c "$HERE/$s" -o "$o" &
    pids+=($!)
  fi
  OBJS="$OBJS $o"
done
for p in "${pids[@]}"; do wait $p; done
$NVCC -shared -o "$OUT/libvtoonify_b200.so" $OBJS -lcudart
echo "built $OUT/libvtoonify_b200.so"
