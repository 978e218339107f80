// WindowExec kernels (window/processors/*.rs of the reference, restated as segmented prefix scans).
//
// The input is sorted by (partition spec, order spec).  window_flags_kernel marks partition heads and order-key changes by
// comparing row i with row i-1 (row 0 with the key carry of the previous push).  Every window function is then a segmented
// scan with an associative state (WinState), run as reduce-then-scan over tiles of WIN_TILE rows:
//   (a) window_reduce_kernel: one summary per tile;
//   (b) window_scan_tiles_kernel: one CTA scans the summaries in order from the carry state, writes each tile's prefix and
//       the next carry (the state after the last row, kept on the device);
//   (c) window_emit_kernel: each tile rescans its rows from its prefix and writes the window column(s).
// The association of every combine is fixed by the tile and thread structure, so f64 running sums are identical from run to
// run for the same batch split.
#include "emit_device.cuh"
#include "kernels_window.cuh"
#include "vm.cuh"

namespace b200q {

namespace {

struct KeyWord { unsigned long long lo, hi; bool valid; };

__device__ __forceinline__ bool bit_at(const uint8_t* bits, uint64_t i) { return (bits[i >> 3] >> (i & 7)) & 1; }

// the value bits of row i at the column's width (equality is bit equality: -0.0 != +0.0, NaNs equal only with the same payload)
__device__ __forceinline__ KeyWord load_word(const DevCol& c, uint8_t phys, int64_t i) {
  KeyWord w{0, 0, c.validity == nullptr || bit_at(c.validity, (uint64_t)c.bit_offset + (uint64_t)i)};
  switch (phys) {
    case PH_BOOL: w.lo = bit_at((const uint8_t*)c.values, (uint64_t)c.bit_offset + (uint64_t)i); break;
    case PH_I8: w.lo = (unsigned long long)(long long)((const int8_t*)c.values)[i]; break;
    case PH_I16: w.lo = (unsigned long long)(long long)((const int16_t*)c.values)[i]; break;
    case PH_I32: w.lo = (unsigned long long)(long long)((const int32_t*)c.values)[i]; break;
    case PH_F32: w.lo = ((const uint32_t*)c.values)[i]; break;
    case PH_I64: case PH_F64: w.lo = ((const unsigned long long*)c.values)[i]; break;
    default: w.lo = ((const unsigned long long*)c.values)[2 * i]; w.hi = ((const unsigned long long*)c.values)[2 * i + 1]; break;
  }
  return w;
}

__global__ void __launch_bounds__(256) window_flags_kernel(const WinKeys keys, int64_t n, const WinKeyCarry* __restrict__ carry, uint8_t* __restrict__ flags) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    bool p = false, o = false;
    const bool first = i == 0 && !carry->has_prev;
    for (int k = 0; k < keys.nkeys && !first; k++) {
      const WinKey& wk = keys.k[k];
      const KeyWord a = load_word(wk.col, wk.phys, i);
      KeyWord b;
      if (i > 0) b = load_word(wk.col, wk.phys, i - 1);
      else { b.lo = carry->lo[k]; b.hi = carry->hi[k]; b.valid = (carry->valid_mask >> k) & 1; }
      const bool differ = a.valid != b.valid || (a.valid && (a.lo != b.lo || a.hi != b.hi));      // NULL == NULL
      if (wk.is_order) o = o || differ; else p = p || differ;
    }
    if (first) { p = keys.has_partition; o = keys.has_order; }   // the empty previous row of the reference's processors
    else p = p && keys.has_partition;
    flags[i] = (uint8_t)(p | (o << 1));
  }
}

// runs after window_flags_kernel (stream order): the last row's keys become the carry of the next push
__global__ void window_key_carry_kernel(const WinKeys keys, int64_t n, WinKeyCarry* carry) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  uint32_t vm = 0;
  for (int k = 0; k < keys.nkeys; k++) {
    const KeyWord w = load_word(keys.k[k].col, keys.k[k].phys, n - 1);
    carry->lo[k] = w.lo; carry->hi[k] = w.hi; vm |= (uint32_t)w.valid << k;
  }
  carry->valid_mask = vm; carry->has_prev = 1;
}

__device__ __forceinline__ WinState win_identity() { WinState s; s.reset = s.has_head = s.c = s.h = s.d = s.valid = 0; s.lo = s.hi = 0; s.cnt = 0; return s; }

__device__ __forceinline__ long long fkey(unsigned long long bits, uint8_t phys) {       // IEEE totalOrder of f32 / f64 bits
  if (phys == PH_F32) { const int x = (int)(uint32_t)bits; return (long long)(x ^ ((x >> 31) & 0x7FFFFFFF)); }
  return total_order_key(bits);
}

__device__ __forceinline__ WinState win_element(const WinFn& f, uint8_t flags, int64_t i) {
  WinState s = win_identity();
  s.reset = flags & 1;
  if (f.op == WOP_RANK) { s.has_head = flags != 0; s.c = 1; s.h = 1; s.d = flags != 0; return s; }
  if (f.op == WOP_COUNT) {
    bool all = true;
    for (int a = 0; a < f.nargs; a++) all = all && (f.arg[a].validity == nullptr || bit_at(f.arg[a].validity, (uint64_t)f.arg[a].bit_offset + (uint64_t)i));
    s.cnt = all; s.valid = 1;
    return s;
  }
  const KeyWord w = load_word(f.arg[0], f.arg_phys, i);
  s.valid = w.valid;
  if (w.valid) { s.lo = w.lo; s.hi = w.hi; s.cnt = 1; }
  return s;
}

// a then b (b's rows follow a's)
__device__ __forceinline__ WinState win_combine(const WinFn& f, const WinState& a, const WinState& b) {
  if (b.reset) return b;
  WinState r = a;
  if (f.op == WOP_RANK) {
    r.c = a.c + b.c; r.d = a.d + b.d;
    if (b.has_head) { r.h = a.c + b.h; r.has_head = 1; }
    return r;
  }
  r.cnt = a.cnt + b.cnt;
  if (!b.valid) return r;
  r.valid = 1;
  if (!a.valid) { r.lo = b.lo; r.hi = b.hi; return r; }
  switch (f.op) {
    case WOP_SUM_I64: r.lo = a.lo + b.lo; break;                                                         // wraps (overflow-checks = false)
    case WOP_SUM_I128: case WOP_AVG_DEC: { const i128_t v = (i128_t)((u128_t)mk128(a.lo, a.hi) + (u128_t)mk128(b.lo, b.hi)); r.lo = lo64(v); r.hi = hi64(v); break; }
    case WOP_SUM_F64: case WOP_AVG_F64: r.lo = f64_bits(as_f64(a.lo) + as_f64(b.lo)); break;
    case WOP_MIN_I64: if ((long long)b.lo < (long long)a.lo) r.lo = b.lo; break;
    case WOP_MAX_I64: if ((long long)b.lo > (long long)a.lo) r.lo = b.lo; break;
    case WOP_MIN_I128: if (mk128(b.lo, b.hi) < mk128(a.lo, a.hi)) { r.lo = b.lo; r.hi = b.hi; } break;
    case WOP_MAX_I128: if (mk128(b.lo, b.hi) > mk128(a.lo, a.hi)) { r.lo = b.lo; r.hi = b.hi; } break;
    case WOP_MIN_F: if (fkey(b.lo, f.arg_phys) < fkey(a.lo, f.arg_phys)) r.lo = b.lo; break;
    case WOP_MAX_F: if (fkey(b.lo, f.arg_phys) > fkey(a.lo, f.arg_phys)) r.lo = b.lo; break;
    default: break;
  }
  return r;
}

__device__ __forceinline__ void store_width(void* out, uint8_t phys, int64_t i, unsigned long long lo, unsigned long long hi) {
  switch (phys) {
    case PH_I8: ((int8_t*)out)[i] = (int8_t)lo; break;
    case PH_I16: ((int16_t*)out)[i] = (int16_t)lo; break;
    case PH_I32: case PH_F32: ((uint32_t*)out)[i] = (uint32_t)lo; break;
    case PH_I64: case PH_F64: ((unsigned long long*)out)[i] = lo; break;
    default: ((unsigned long long*)out)[2 * i] = lo; ((unsigned long long*)out)[2 * i + 1] = hi; break;
  }
}

// the window column(s) of row i from the inclusive state
__device__ __forceinline__ void win_emit(const WinFn& f, const WinState& s, int64_t i) {
  if (f.op == WOP_RANK) {
    if (f.out[0]) ((int32_t*)f.out[0])[i] = (int32_t)s.c;
    if (f.out[1]) ((int32_t*)f.out[1])[i] = (int32_t)s.h;
    if (f.out[2]) ((int32_t*)f.out[2])[i] = (int32_t)s.d;
    return;
  }
  unsigned long long lo = s.lo, hi = s.hi;
  bool valid = s.valid;
  if (f.op == WOP_COUNT) { lo = (unsigned long long)s.cnt; valid = true; }
  else if (f.op == WOP_AVG_F64) { valid = s.cnt != 0; lo = valid ? f64_bits(avg_f64_final(as_f64(s.lo), s.cnt)) : 0; }
  else if (f.op == WOP_AVG_DEC) { valid = s.cnt != 0; const i128_t q = valid ? avg_dec_final(mk128(s.lo, s.hi), s.cnt) : 0; lo = lo64(q); hi = hi64(q); }
  if (!valid) lo = hi = 0;
  store_width(f.out[0], f.out_phys, i, lo, hi);
  if (f.out_valid) f.out_valid[i] = valid;
}

__device__ __forceinline__ WinState thread_reduce(const WinFn& f, const uint8_t* __restrict__ flags, int64_t base, int64_t n) {
  WinState s = win_identity();
  for (int k = 0; k < WIN_ITEMS; k++) { const int64_t i = base + k; if (i < n) s = win_combine(f, s, win_element(f, flags[i], i)); }
  return s;
}

// (a) one summary per tile; a pairwise tree in shared memory keeps the row order (the combine is not commutative)
__global__ void __launch_bounds__(WIN_THREADS, 1) window_reduce_kernel(const WinFn f, const uint8_t* __restrict__ flags, int64_t n, WinState* __restrict__ tile_sum) {
  __shared__ WinState sh[WIN_THREADS];
  const int t = threadIdx.x;
  sh[t] = thread_reduce(f, flags, (int64_t)blockIdx.x * WIN_TILE + (int64_t)t * WIN_ITEMS, n);
  __syncthreads();
  for (int off = 1; off < WIN_THREADS; off <<= 1) {
    if ((t & (2 * off - 1)) == 0) sh[t] = win_combine(f, sh[t], sh[t + off]);
    __syncthreads();
  }
  if (t == 0) tile_sum[blockIdx.x] = sh[0];
}

// inclusive scan of sh[0..NT) in place (Hillis-Steele; every step reads before any thread writes)
template <int NT>
__device__ __forceinline__ void block_scan(const WinFn& f, WinState* sh) {
  const int t = threadIdx.x;
  for (int off = 1; off < NT; off <<= 1) {
    WinState v = sh[t];
    if (t >= off) v = win_combine(f, sh[t - off], v);
    __syncthreads();
    sh[t] = v;
    __syncthreads();
  }
}

// (b) one CTA: the exclusive prefix of every tile from the carry, and the next carry
__global__ void __launch_bounds__(WIN_SCAN_THREADS) window_scan_tiles_kernel(const WinFn f, int64_t ntiles, WinState* carry, const WinState* __restrict__ tile_sum, WinState* __restrict__ tile_prefix) {
  __shared__ WinState sh[WIN_SCAN_THREADS];
  const int t = threadIdx.x;
  const WinState c0 = *carry;
  const int64_t per = (ntiles + WIN_SCAN_THREADS - 1) / WIN_SCAN_THREADS, lo = (int64_t)t * per, hi = lo + per < ntiles ? lo + per : ntiles;
  WinState s = win_identity();
  for (int64_t j = lo; j < hi; j++) s = win_combine(f, s, tile_sum[j]);
  sh[t] = s;
  __syncthreads();
  block_scan<WIN_SCAN_THREADS>(f, sh);
  WinState p = t == 0 ? c0 : win_combine(f, c0, sh[t - 1]);
  for (int64_t j = lo; j < hi; j++) { tile_prefix[j] = p; p = win_combine(f, p, tile_sum[j]); }
  if (t == 0) *carry = win_combine(f, c0, sh[WIN_SCAN_THREADS - 1]);
}

// (c) rescan each tile from its prefix and write the window columns
__global__ void __launch_bounds__(WIN_THREADS) window_emit_kernel(const WinFn f, const uint8_t* __restrict__ flags, int64_t n, const WinState* __restrict__ tile_prefix) {
  __shared__ WinState sh[WIN_THREADS];
  const int t = threadIdx.x;
  const int64_t base = (int64_t)blockIdx.x * WIN_TILE + (int64_t)t * WIN_ITEMS;
  sh[t] = thread_reduce(f, flags, base, n);
  __syncthreads();
  block_scan<WIN_THREADS>(f, sh);
  const WinState tp = tile_prefix[blockIdx.x];
  WinState s = t == 0 ? tp : win_combine(f, tp, sh[t - 1]);
  for (int k = 0; k < WIN_ITEMS; k++) {
    const int64_t i = base + k;
    if (i >= n) break;
    s = win_combine(f, s, win_element(f, flags[i], i));
    win_emit(f, s, i);
  }
}

}  // namespace

int launch_window_flags(const WinKeys& keys, int64_t n, WinKeyCarry* d_carry, uint8_t* d_flags, cudaStream_t s) {
  if (n <= 0) return 0;
  const int64_t blocks = (n + 255) / 256;
  window_flags_kernel<<<(unsigned)(blocks < 65536 ? blocks : 65536), 256, 0, s>>>(keys, n, d_carry, d_flags);
  window_key_carry_kernel<<<1, 32, 0, s>>>(keys, n, d_carry);
  return 2;
}

int launch_window_scan(const WinFn& f, const uint8_t* d_flags, int64_t n, WinState* d_carry, WinState* d_tile_sum, WinState* d_tile_prefix, cudaStream_t s) {
  if (n <= 0) return 0;
  const int64_t ntiles = window_num_tiles(n);
  window_reduce_kernel<<<(unsigned)ntiles, WIN_THREADS, 0, s>>>(f, d_flags, n, d_tile_sum);
  window_scan_tiles_kernel<<<1, WIN_SCAN_THREADS, 0, s>>>(f, ntiles, d_carry, d_tile_sum, d_tile_prefix);
  window_emit_kernel<<<(unsigned)ntiles, WIN_THREADS, 0, s>>>(f, d_flags, n, d_tile_prefix);
  return 3;
}

}  // namespace b200q
