#!/usr/bin/env bash
# Builds annlite_b200/lib/libannlite_b200.so for sm_90a (H100; nvcc cross-compiles without a GPU).
set -euo pipefail
HERE="$(cd "$(dirname "${BASH_SOURCE[0]}")" && pwd)"
OUT="$HERE/../lib"
mkdir -p "$OUT" "$HERE/obj"
NVCC="${NVCC:-/usr/local/cuda/bin/nvcc}"
ARCH="-gencode arch=compute_90a,code=sm_90a"
CXXFLAGS="-O3 -std=c++17 -lineinfo -Xcompiler -fPIC,-fvisibility=hidden,-Wall,-Wno-unused-function ${ANNB_EXTRA_NVCC:-}"
pids=()
for f in adc_table adc_scan hnsw_search walk_fused walk_flagged4 walk_wide gpu_build attr_filter cells capi; do
  $NVCC $ARCH $CXXFLAGS -c "$HERE/$f.cu" -o "$HERE/obj/$f.o" &
  pids+=($!)
done
# host builder: no FMA contraction so the fp32 sums match the reference's ISO-mode build
g++ -O3 -std=c++17 -fPIC -fvisibility=hidden -ffp-contract=off -march=x86-64-v3 -Wall -I/usr/local/cuda/include \
    -c "$HERE/hnsw_build.cpp" -o "$HERE/obj/hnsw_build.o" &
pids+=($!)
for p in "${pids[@]}"; do wait "$p"; done
$NVCC $ARCH -shared -o "$OUT/libannlite_b200.so" "$HERE"/obj/{adc_table,adc_scan,hnsw_search,walk_fused,walk_flagged4,walk_wide,gpu_build,attr_filter,cells,capi,hnsw_build}.o \
    -Xlinker --exclude-libs,ALL -lpthread
echo "built $OUT/libannlite_b200.so"
