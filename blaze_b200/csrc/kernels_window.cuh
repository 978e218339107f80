// Descriptors and launchers of the WindowExec kernels (kernels_window.cu): segmented prefix scans over a sorted stream.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "ir.h"
#include "vm.h"

namespace b200q {

constexpr int WIN_MAX_KEYS = WINDOW_MAX_KEYS;
constexpr int WIN_MAX_ARGS = WINDOW_MAX_COUNT_ARGS;   // COUNT arguments (the other aggregates take one)
constexpr int WIN_THREADS = 256, WIN_ITEMS = 8, WIN_TILE = WIN_THREADS * WIN_ITEMS;
constexpr int WIN_SCAN_THREADS = 512;   // the one CTA that scans the tile summaries

struct WinKey { DevCol col; uint8_t phys; uint8_t is_order; uint8_t _pad[6]; };
struct WinKeys { WinKey k[WIN_MAX_KEYS]; int nkeys, has_partition, has_order, _pad; };

// key words of the last row of the previous push (device resident: the next push compares its row 0 with them)
struct WinKeyCarry { unsigned long long lo[WIN_MAX_KEYS], hi[WIN_MAX_KEYS]; uint32_t valid_mask, has_prev; };

enum WinOp : uint8_t { WOP_RANK = 0, WOP_SUM_I64, WOP_SUM_I128, WOP_SUM_F64, WOP_MIN_I64, WOP_MAX_I64, WOP_MIN_I128, WOP_MAX_I128,
                       WOP_MIN_F, WOP_MAX_F, WOP_COUNT, WOP_AVG_F64, WOP_AVG_DEC };

// State of a segmented scan over a span of rows.  `reset`: a partition starts inside the span (the span's state then only
// depends on its rows from the last partition head on).  Rank-like functions: c = rows, d = peer-group heads, h = row number of
// the last peer-group head (valid if has_head), all counted from the span start or the last partition head, wrapping at 2^32.
// Aggregates: lo/hi = the accumulator (f64 bits, i64, i128, or the raw bits of a MIN/MAX value), valid = a valid value was
// accumulated, cnt = valid values (AVG) or counted rows (COUNT).
struct WinState {
  uint32_t reset, has_head, c, h, d, valid;
  unsigned long long lo, hi;
  long long cnt;
};

struct WinFn {
  uint8_t op, arg_phys, out_phys, nargs;
  uint32_t _pad;
  DevCol arg[WIN_MAX_ARGS];
  void* out[3];                         // WOP_RANK: row_number, rank, dense_rank (int32, each optional); aggregates: out[0]
  uint8_t* out_valid;                   // aggregates: one byte per row (packed afterwards), null when the column is never NULL
};

// flags[i] = bit 0: partition head, bit 1: order key differs from row i-1 (the carry row for i = 0); refreshes the key carry
int launch_window_flags(const WinKeys& keys, int64_t n, WinKeyCarry* d_carry, uint8_t* d_flags, cudaStream_t s);
inline int64_t window_num_tiles(int64_t n) { return (n + WIN_TILE - 1) / WIN_TILE; }
// reduce-then-scan of one function over the rows of a push; d_carry: the state after the previous push (updated in place)
// d_tile_sum / d_tile_prefix: window_num_tiles(n) states each
int launch_window_scan(const WinFn& f, const uint8_t* d_flags, int64_t n, WinState* d_carry, WinState* d_tile_sum, WinState* d_tile_prefix, cudaStream_t s);

}  // namespace b200q
