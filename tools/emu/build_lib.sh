#!/bin/bash
# Build the WHOLE library (C ABI, host logic, every kernel) against the host stand-in for the CUDA runtime:
#   tools/emu/build_lib.sh [outdir]  ->  <outdir>/libblaze_b200_emu.so
# Test infrastructure only (tools/emu/run_gpu_suite.py loads it explicitly); the product library is blaze_b200/libblaze_b200.so.
set -e
HERE=$(cd "$(dirname "$0")" && pwd); OUT=${1:-${TMPDIR:-/tmp}/b200q_emu}
python "$HERE/build_emu.py" "$OUT" > /dev/null
SAN=""; if [ -n "$EMU_SANITIZE" ]; then SAN="-fsanitize=address,undefined -fno-omit-frame-pointer"; fi   # run python with LD_PRELOAD=$(gcc -print-file-name=libasan.so)
cd "$OUT/blaze_b200/csrc"
pids=()
for f in kernels.cu kernels_fast.cu kernels_tile.cu kernels_shuffle.cu kernels_join.cu kernels_sort.cu kernels_window.cu kernels_parquet.cu parquet_source.cu stages.cu shuffle_stage.cu join_stage.cu sort_stage.cu window_stage.cu capi.cu exchange.cu plan_decode.cc arrow_ipc.cc compile.cc lz4_frame.cc parquet_meta.cc; do
  g++ -std=c++20 -O1 -g -fPIC -pthread -w $SAN -x c++ -I"$HERE/include" -I. -c "$f" -o "${f%.*}.o" & pids+=($!)
done
for p in "${pids[@]}"; do wait "$p"; done
g++ -shared -pthread $SAN -o "$OUT/libblaze_b200_emu.so" kernels.o kernels_fast.o kernels_tile.o kernels_shuffle.o kernels_join.o kernels_sort.o kernels_window.o kernels_parquet.o parquet_source.o stages.o shuffle_stage.o join_stage.o sort_stage.o window_stage.o capi.o exchange.o plan_decode.o arrow_ipc.o compile.o lz4_frame.o parquet_meta.o
echo "$OUT/libblaze_b200_emu.so"
