#!/bin/bash
# Build the sanitizer harnesses of the host-side decoders and run a bounded fuzz: tools/fuzz/run.sh [iterations] [seed]
set -e
HERE=$(cd "$(dirname "$0")" && pwd); ROOT=$(cd "$HERE/../.." && pwd); OUT=${TMPDIR:-/tmp}/b200q_fuzz; N=${1:-100000}; SEED=${2:-1}
mkdir -p "$OUT/seeds"
python "$HERE/make_seeds.py" "$OUT/seeds"
g++ -std=c++17 -O1 -g -fsanitize=address,undefined -fno-sanitize-recover=undefined -I"$ROOT/blaze_b200/csrc" \
    "$HERE/plan_decode_fuzz.cc" "$ROOT/blaze_b200/csrc/plan_decode.cc" "$ROOT/blaze_b200/csrc/arrow_ipc.cc" -o "$OUT/plan_decode_fuzz"
"$OUT/plan_decode_fuzz" "$SEED" "$N" "$OUT"/seeds/seed*.bin
"$OUT/plan_decode_fuzz" "$SEED" "$N" --ipc "$OUT"/seeds/lit*.bin
g++ -std=c++17 -O1 -g -fsanitize=address,undefined -fno-sanitize-recover=undefined -I"$ROOT/blaze_b200/csrc" \
    "$HERE/ipc_fuzz.cc" "$ROOT/blaze_b200/csrc/lz4_frame.cc" "$ROOT/blaze_b200/csrc/ipc_records.cc" -o "$OUT/ipc_fuzz"
"$OUT/ipc_fuzz" "$SEED" "$N" --lz4 "$OUT"/seeds/lz4_*.bin
"$OUT/ipc_fuzz" "$SEED" "$N" --records "$OUT"/seeds/rec_*.bin
