#!/usr/bin/env bash
# Host-code hygiene (CPU only, no GPU needed): the CPU test-suite and two fuzzers under ASan+UBSan, and the threaded
# graph builder under TSan.  The sanitizer build of the library temporarily replaces annlite_b200/lib/…so and the
# regular build is put back at the end.   usage: bash scripts/hygiene/run.sh
set -euo pipefail
ROOT="$(cd "$(dirname "$0")/../.." && pwd)"
H="$ROOT/annlite_b200/csrc"; LIB="$ROOT/annlite_b200/lib/libannlite_b200.so"
O="$(mktemp -d)"; NVCC="${NVCC:-/usr/local/cuda/bin/nvcc}"; ARCH="-gencode arch=compute_90a,code=sm_90a"
for f in adc_table adc_scan hnsw_search walk_fused walk_flagged4 gpu_build attr_filter capi; do
  $NVCC $ARCH -O1 -g -std=c++17 -Xcompiler -fPIC,-fvisibility=hidden,-fsanitize=address,-fsanitize=undefined,-fno-omit-frame-pointer -c "$H/$f.cu" -o "$O/$f.o" &
done
g++ -O1 -g -std=c++17 -fPIC -fvisibility=hidden -ffp-contract=off -march=x86-64-v3 -fsanitize=address,undefined -fno-omit-frame-pointer \
    -I/usr/local/cuda/include -c "$H/hnsw_build.cpp" -o "$O/hnsw_build.o" &
wait
$NVCC $ARCH -shared -o "$O/asan.so" "$O"/{adc_table,adc_scan,hnsw_search,walk_fused,walk_flagged4,gpu_build,attr_filter,capi,hnsw_build}.o -Xlinker --exclude-libs,ALL -lpthread -Xcompiler -fsanitize=address,-fsanitize=undefined
cp "$LIB" "$O/good.so"; trap 'cp "$O/good.so" "$LIB"' EXIT
cp "$O/asan.so" "$LIB"
export LD_PRELOAD="$(gcc -print-file-name=libasan.so) $(gcc -print-file-name=libubsan.so)"
# alloc_dealloc_mismatch=0: the compiled REFERENCE (oracle/_ref, loaded by the oracle-vs-reference tests) frees malloc'ed
# result buffers with operator delete in its pybind11 capsules; that is its defect, not this library's.
export ASAN_OPTIONS=detect_leaks=0:halt_on_error=1:allocator_may_return_null=1:alloc_dealloc_mismatch=0 UBSAN_OPTIONS=print_stacktrace=1:halt_on_error=1
(cd "$ROOT" && python -m pytest tests -q -m "not gpu" -p no:cacheprovider -x | tail -1)
python "$ROOT/scripts/hygiene/fuzz_load.py" 2000
python "$ROOT/scripts/hygiene/fuzz_state.py" 3000
unset LD_PRELOAD
g++ -O1 -g -std=c++17 -fsanitize=thread -ffp-contract=off -march=x86-64-v3 -I"$H" -I"$ROOT/include" -I/usr/local/cuda/include \
    "$ROOT/scripts/hygiene/tsan_build_main.cpp" "$H/hnsw_build.cpp" -o "$O/tsan_build" -lpthread
TSAN_OPTIONS=halt_on_error=1 "$O/tsan_build" 60000 32
echo "hygiene: clean"
