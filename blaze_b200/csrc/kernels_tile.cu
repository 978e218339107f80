// TILE form of the specialised HashAgg update kernels (round 2): the streaming front end of every shape that has
// fused FilterExec conjuncts, typed (int8..int64) or nullable inputs, or two keys.
//
// Why: the one-row-per-lane kernels of kernels_fast.cu issue one 8-byte (or narrower) load per row per column plus one
// validity-byte load per row, re-read a filter column once per conjunct, and run G shuffle + RED steps per 32 rows
// whether or not the rows survived the filter.
// Here a warp owns a TILE of 128 consecutive rows and lane l holds rows l, l + 32, l + 64 and l + 96 of it:
//   * one warp-wide load reads 32 consecutive rows of a column, i.e. whole 32-byte sectors at every width (256 bytes of
//     an int64 column, 512 of a decimal128, 32 of an int8); a validity bitmap is read as the byte that holds the lane's
//     bit (32 lanes: one 4-byte run per 32 rows);
//   * FILTER FIRST: with fused conjuncts the filter columns are read in full, and the key and argument columns (values and
//     validity) only for the rows that pass — a predicated per-row load, so a sector without a surviving row is never
//     requested (DESIGN §3.1 measures what that saves); a filter column that is also a key or argument is read once;
//   * the filter columns of the warp's NEXT tile are in flight while the current tile is compacted and reduced;
//   * the conjuncts on one column are merged on the host into one closed interval [lo, hi] (FilterExec conjuncts are
//     pre-split `col cmp literal` terms, NativeFilterBase.scala:66-87), tested with one subtract + one unsigned compare;
//   * rows that survive are COMPACTED into a per-warp shared-memory queue (ballot + popc, no atomics), and the dense
//     table is updated from the queue G lanes per entry: one RED instruction updates the G words of 32/G rows, so a
//     selectivity of 0.2 costs 0.2 x the RED issue slots and sector operations instead of 1.0 x.
// Semantics are those of agg_dense_row_kernel (same table, same entry layout, same fall-back of NULL / out-of-range
// keys to the hashed slots, same deferred-row protocol: a deferred entry is the row's launch-relative index), so the
// emit / grow / replay code is shared.
#include <cuda_runtime.h>
#include <stdint.h>

#include <algorithm>

#include "agg_device.cuh"
#include "emit_device.cuh"
#include "kernels_fast.cuh"

namespace b200q {

constexpr int TL_BLOCK = 256, TL_WARPS = TL_BLOCK / 32, TL_ROWS = 128;

__device__ __forceinline__ uint64_t tl_policy_evict_first() {
  uint64_t pol; asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol)); return pol;
}
// predicated streaming loads: nothing is requested when `on` is 0 (the destination keeps its value)
__device__ __forceinline__ void tl_ld_b64(const long long* p, unsigned on, uint64_t pol, long long& v) {
  asm volatile("{\n\t.reg .pred q;\n\tsetp.ne.u32 q, %2, 0;\n\t@q ld.global.nc.L1::no_allocate.L2::cache_hint.b64 %0, [%1], %3;\n\t}"
               : "+l"(v) : "l"(p), "r"(on), "l"(pol));
}
__device__ __forceinline__ void tl_ld_v2b64(const long long* p, unsigned on, uint64_t pol, long long& a, long long& b) {   // p is 16-byte aligned
  asm volatile("{\n\t.reg .pred q;\n\tsetp.ne.u32 q, %3, 0;\n\t@q ld.global.nc.L1::no_allocate.L2::cache_hint.v2.b64 {%0,%1}, [%2], %4;\n\t}"
               : "+l"(a), "+l"(b) : "l"(p), "r"(on), "l"(pol));
}
__device__ __forceinline__ void tl_ld_b32(const int* p, unsigned on, uint64_t pol, int& v) {
  asm volatile("{\n\t.reg .pred q;\n\tsetp.ne.u32 q, %2, 0;\n\t@q ld.global.nc.L1::no_allocate.L2::cache_hint.b32 %0, [%1], %3;\n\t}"
               : "+r"(v) : "l"(p), "r"(on), "l"(pol));
}

// bit j set: row l + 32 j of the tile (launch-relative `rel` of j = 0) lies below n
__device__ __forceinline__ unsigned tl_rows_in(long long rel, long long n) {
  const long long left = n - rel;
  return left > 96 ? 0xFu : left > 64 ? 0x7u : left > 32 ? 0x3u : left > 0 ? 0x1u : 0u;
}

// rows r0 + 32 j (j = 0..3) of one column as sign-extended int64 + their validity bits, for the rows whose bit is set in `ld`;
// the other rows read as 0 / invalid and are not touched in memory.  `want_values` = false: only the validity (COUNT(col)).
__device__ __forceinline__ void tl_load(const DevCol& c, int phys, long long r0, unsigned ld, bool want_values, uint64_t pol, long long (&v)[4], unsigned& valid) {
  valid = ld;
  if (c.validity) {
#pragma unroll
    for (int j = 0; j < 4; j++) {
      const unsigned long long bi = (unsigned long long)(r0 + 32 * j) + c.bit_offset;
      const unsigned b = ((ld >> j) & 1u) ? __ldg(c.validity + (bi >> 3)) : 0u;
      valid &= ~((((b >> (bi & 7)) & 1u) ^ 1u) << j);
    }
  }
#pragma unroll
  for (int j = 0; j < 4; j++) v[j] = 0;
  if (!want_values) return;
  switch (phys) {
    case PH_I64: {
      const long long* p = (const long long*)c.values + r0;
#pragma unroll
      for (int j = 0; j < 4; j++) tl_ld_b64(p + 32 * j, (ld >> j) & 1u, pol, v[j]);
      break;
    }
    case PH_I32: {
      const int* p = (const int*)c.values + r0;
#pragma unroll
      for (int j = 0; j < 4; j++) { int t = 0; tl_ld_b32(p + 32 * j, (ld >> j) & 1u, pol, t); v[j] = t; }
      break;
    }
    case PH_I16: {
      const int16_t* p = (const int16_t*)c.values + r0;
#pragma unroll
      for (int j = 0; j < 4; j++) v[j] = ((ld >> j) & 1u) ? __ldg(p + 32 * j) : 0;
      break;
    }
    case PH_I8: {
      const int8_t* p = (const int8_t*)c.values + r0;
#pragma unroll
      for (int j = 0; j < 4; j++) v[j] = ((ld >> j) & 1u) ? __ldg(p + 32 * j) : 0;
      break;
    }
    default: {                                                    // PH_BOOL: bit-packed values
#pragma unroll
      for (int j = 0; j < 4; j++) {
        const unsigned long long bi = (unsigned long long)(r0 + 32 * j) + c.bit_offset;
        v[j] = ((ld >> j) & 1u) ? (__ldg((const uint8_t*)c.values + (bi >> 3)) >> (bi & 7)) & 1u : 0u;
      }
      break;
    }
  }
}

// the filter columns of the tile whose lane-0 row is `rel` (all its rows below n), and the rows that pass every interval
template <int NF>
__device__ __forceinline__ void tl_load_filters(const ColTable& cols, const FilterInterval (&fr)[2], long long row_begin, long long rel, long long n, uint64_t pol,
                                                long long (&f)[NF > 0 ? NF : 1][4], unsigned (&fv)[NF > 0 ? NF : 1]) {
  const unsigned in = tl_rows_in(rel, n);
#pragma unroll
  for (int c = 0; c < NF; c++) tl_load(cols.col[fr[c].col], fr[c].phys, row_begin + rel, in, true, pol, f[c], fv[c]);
}
template <int NF>
__device__ __forceinline__ unsigned tl_pass(const FilterInterval (&fr)[2], const long long (&f)[NF > 0 ? NF : 1][4], const unsigned (&fv)[NF > 0 ? NF : 1], unsigned in) {
  unsigned alive = in;
#pragma unroll
  for (int c = 0; c < NF; c++) {
    unsigned pass = 0;
#pragma unroll
    for (int j = 0; j < 4; j++) pass |= (unsigned)((unsigned long long)(f[c][j] - fr[c].lo) <= fr[c].span) << j;
    alive &= pass & fv[c];                                          // NULL -> row dropped (cached_exprs_evaluator.rs:518-520)
  }
  return alive;
}
// a key / argument column that is also filter column c >= 0 is taken from the filter registers instead of being read again
template <int NF>
__device__ __forceinline__ int tl_filter_of(const FilterInterval (&fr)[2], int col) {
  return NF > 0 && fr[0].col == col ? 0 : (NF > 1 && fr[NF > 1 ? 1 : 0].col == col ? 1 : -1);
}
template <int NF>
__device__ __forceinline__ void tl_column(const ColTable& cols, const FilterInterval (&fr)[2], const long long (&f)[NF > 0 ? NF : 1][4], const unsigned (&fv)[NF > 0 ? NF : 1],
                                          int col, int phys, long long r0, unsigned ld, bool want_values, uint64_t pol, long long (&v)[4], unsigned& valid) {
  const int fc = tl_filter_of<NF>(fr, col);
  tl_load(cols.col[col], phys, r0, fc < 0 ? ld : 0u, want_values, pol, v, valid);
  if (fc >= 0) {
#pragma unroll
    for (int j = 0; j < 4; j++) v[j] = fc == 0 ? f[0][j] : f[NF > 1 ? 1 : 0][j];
    valid = (fc == 0 ? fv[0] : fv[NF > 1 ? 1 : 0]) & ld;
  }
}

// resident CTAs per SM the register allocation must allow: 4 (64 registers a thread) for the instances that fit them without
// a spill, among them the q1 shape <2,1,2,1>; 3 (80 registers) for the one-key wide instances without a filter, which ptxas
// otherwise squeezes into 64 registers with spills; no bound for the others.  tile_grid sizes every grid from the result.
#define TD_MIN_CTAS(NK, NACC, NF) ((NACC == 1 ? (NK == 1 || NF < 2) : (NK == 1 && NF == 0)) ? 4 : 1)
#define TW_MIN_CTAS(NK, NF) ((NK == 1 && NF == 0) ? 3 : 1)

enum { TW_ZERO = 0, TW_ONE, TW_ADD0, TW_ADD1, TW_VALID0, TW_VALID1 };     // what an entry word accumulates

struct TileQueue {                                                  // per warp: the surviving rows of one tile
  unsigned idx[TL_ROWS];                                            // dense entry index | argument-valid bits << 28
  unsigned long long v0[TL_ROWS], v1[TL_ROWS];
};

template <int NK, int NACC, int G, int NF>
__global__ void __launch_bounds__(TL_BLOCK, TD_MIN_CTAS(NK, NACC, NF)) agg_tile_dense_kernel(const ColTable cols, const FastSpec fs, const AggLayout lay, const AggTable tab,
                                                                  long long row_begin, long long n) {
  constexpr unsigned IDX_MASK = 0x0FFFFFFFu;                        // dense_cap <= 2^26
  constexpr unsigned FULL = 0xffffffffu;
  __shared__ TileQueue queues[TL_WARPS];
  TileQueue& q = queues[threadIdx.x >> 5];
  const unsigned lane = threadIdx.x & 31, qw = lane & (G - 1);
  const long long gwarp = (long long)blockIdx.x * TL_WARPS + (threadIdx.x >> 5), nwarps = (long long)gridDim.x * TL_WARPS;
  const long long ntiles = (n + TL_ROWS - 1) / TL_ROWS;
  const bool add0 = fs.acc[0].kind == FAST_ACC_ADD, add1 = NACC == 2 && fs.acc[1].kind == FAST_ACC_ADD;
  // this lane's entry word as branch-free selectors (the G lanes of a group hold G different word kinds: a switch
  // here is a 4-way divergent branch in the innermost loop):
  //   val = c_one + (v0 & m0) + (v1 & m1) + ((pk >> vshift) & mvalid)
  unsigned long long c_one = 0, m0 = 0, m1 = 0; unsigned vshift = 28, mvalid = 0;
  {
    const int src = fs.dense_word_src[qw];
    int wkind;
    if (src == -1) wkind = TW_ONE; else if (src == -2) wkind = TW_ZERO;
    else if (src >= 2) wkind = src == 2 ? TW_VALID0 : TW_VALID1;
    else if (src == 0) wkind = add0 ? TW_ADD0 : TW_VALID0;
    else wkind = add1 ? TW_ADD1 : TW_VALID1;
    c_one = wkind == TW_ONE; m0 = wkind == TW_ADD0 ? ~0ULL : 0ULL; m1 = wkind == TW_ADD1 ? ~0ULL : 0ULL;
    mvalid = (wkind == TW_VALID0 || wkind == TW_VALID1) ? 1u : 0u; vshift = wkind == TW_VALID1 ? 29 : 28;
  }
  unsigned long long* const sink = fs.sink + ((gwarp & (FAST_SINK_WARPS - 1)) << 2) + (lane & 3);
  const uint64_t pol = tl_policy_evict_first();

  long long f[NF > 0 ? NF : 1][4]; unsigned fv[NF > 0 ? NF : 1];
  tl_load_filters<NF>(cols, fs.frange, row_begin, gwarp * TL_ROWS + lane, n, pol, f, fv);
  for (long long tile = gwarp; tile < ntiles; tile += nwarps) {
    const long long rel0 = tile * TL_ROWS + lane, row0 = row_begin + rel0;
    // ---- filter first: the key and argument columns are read only for the rows that pass
    const unsigned alive = tl_pass<NF>(fs.frange, f, fv, tl_rows_in(rel0, n));
    long long k0[4], k1[4], a0[4], a1[4]; unsigned kv0, kv1 = 0xF, av0 = 0xF, av1 = 0xF;
    tl_column<NF>(cols, fs.frange, f, fv, fs.key_col[0], fs.key_phys[0], row0, alive, true, pol, k0, kv0);
    if (NK == 2) tl_column<NF>(cols, fs.frange, f, fv, fs.key_col[1], fs.key_phys[1], row0, alive, true, pol, k1, kv1);
    else { k1[0] = k1[1] = k1[2] = k1[3] = 0; }
    if (fs.acc[0].col >= 0) tl_column<NF>(cols, fs.frange, f, fv, fs.acc[0].col, fs.acc[0].phys, row0, alive, add0, pol, a0, av0);
    else { a0[0] = a0[1] = a0[2] = a0[3] = 0; }
    if (NACC == 2 && fs.acc[1].col >= 0) tl_column<NF>(cols, fs.frange, f, fv, fs.acc[1].col, fs.acc[1].phys, row0, alive, add1, pol, a1, av1);
    else { a1[0] = a1[1] = a1[2] = a1[3] = 0; }
    // ---- the next tile's filter columns are in flight while this one is compacted and reduced
    tl_load_filters<NF>(cols, fs.frange, row_begin, rel0 + nwarps * TL_ROWS, n, pol, f, fv);
    // ---- compaction of the surviving rows with an in-range, non-NULL key
    const unsigned knull = (~kv0 | (NK == 2 ? ~kv1 : 0u)) & 0xFu;
    int total = 0; unsigned fb = 0;
#pragma unroll
    for (int j = 0; j < 4; j++) {
      unsigned long long di;
      const bool live = (alive >> j) & 1u;
      const bool in = dense_index_of<NK>(fs, k0[j], k1[j], di) && live && !((knull >> j) & 1u);
      fb |= (unsigned)(live && !in) << j;
      const unsigned m = __ballot_sync(FULL, in);
      if (in) {
        const int at = total + __popc(m & lanemask_lt());
        q.idx[at] = (unsigned)di | (((av0 >> j) & 1u) << 28) | (((av1 >> j) & 1u) << 29);
        if (add0) q.v0[at] = ((av0 >> j) & 1u) ? (unsigned long long)a0[j] : 0ULL;
        if (add1) q.v1[at] = ((av1 >> j) & 1u) ? (unsigned long long)a1[j] : 0ULL;
      }
      total += __popc(m);
    }
    __syncwarp();
    // ---- the G lanes of a group update the G words of one queued row with ONE instruction (one sector operation)
    for (int e0 = 0; e0 < total; e0 += 32 / G) {
      const int e = e0 + (int)(lane / G);
      const bool live = e < total;
      const int er = live ? e : 0;
      const unsigned pk = q.idx[er];
      unsigned long long val = c_one + ((pk >> vshift) & mvalid);
      if (add0) val += q.v0[er] & m0;                                // warp-uniform branches (kernel arguments)
      if (add1) val += q.v1[er] & m1;
      red_add_u64(live ? fs.dense_tab + (uint64_t)(pk & IDX_MASK) * G + qw : sink, live ? val : 0ULL);
    }
    __syncwarp();                                                   // the queue is rewritten by the next tile
    // ---- keys outside the dense range / NULL keys (rare): straight to the hashed slots
    if (__any_sync(FULL, fb != 0)) {
#pragma unroll
      for (int j = 0; j < 4; j++) {
        bool inserted = false;
        if ((fb >> j) & 1u) {
          const unsigned kn = ((~kv0 >> j) & 1u) | (NK == 2 ? (((~kv1 >> j) & 1u) << 1) : 0u);
          uint64_t kw[2] = {(kn & 1u) ? 0ULL : (uint64_t)k0[j], (NK == 2 && !(kn & 2u)) ? (uint64_t)k1[j] : 0ULL};
          unsigned fl = 0;
          const uint64_t si = agg_find_or_insert(lay, tab, kw, kn, agg_hash2(kw[0], kw[1], kn), &fl, &inserted);
          if (si == AGG_NO_SLOT) { const unsigned long long at = atomicAdd(tab.counters + 1, 1ULL); tab.deferred[at] = (uint32_t)(rel0 + 32 * j); }
          else {
            unsigned long long* const p = tab.accs + si * (uint64_t)lay.astride;
            unsigned long long* const ke = tab.keys + si * (uint64_t)lay.kstride;
            if ((av0 >> j) & 1u) { red_add_u64(p + fs.acc[0].word, add0 ? (unsigned long long)a0[j] : 1ULL); slot_mark(ke, fl, fs.acc[0].vbit); }
            if (NACC == 2 && ((av1 >> j) & 1u)) { red_add_u64(p + fs.acc[1].word, add1 ? (unsigned long long)a1[j] : 1ULL); slot_mark(ke, fl, fs.acc[1].vbit); }
          }
        }
        const unsigned bl = __ballot_sync(FULL, inserted);
        if (lane == 0 && bl) atomicAdd(tab.counters, (unsigned long long)__popc(bl));
      }
    }
  }
}

// persistent grid of 256-thread CTAs: one full wave of `kernel` (the CTAs per SM its registers and shared memory allow x
// the SM count), or `units` CTAs when there is less work than that
template <class K>
static int tile_grid(K kernel, int64_t units) {
  int dev = 0, sms = 132, per_sm = 1; cudaGetDevice(&dev); cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, TL_BLOCK, 0) != cudaSuccess || per_sm < 1) per_sm = 1;
  return (int)std::max<int64_t>(1, std::min<int64_t>(units, (int64_t)sms * per_sm));
}

int launch_agg_tile_dense(const ColTable& cols, const FastSpec& fs, const AggLayout& lay, const AggTable& tab, int64_t row_begin, int64_t n, cudaStream_t s) {
  if (n <= 0) return 0;
  const int64_t units = ((n + TL_ROWS - 1) / TL_ROWS + TL_WARPS - 1) / TL_WARPS;
  const int G = fs.dense_stride;
#define B200Q_TD(NK, NACC, G_, NF) do { auto k_ = agg_tile_dense_kernel<NK, NACC, G_, NF>; k_<<<tile_grid(k_, units), TL_BLOCK, 0, s>>>(cols, fs, lay, tab, row_begin, n); } while (0)
#define B200Q_TD_NF(NK, NACC, G_) do { if (fs.nfcol == 0) B200Q_TD(NK, NACC, G_, 0); else if (fs.nfcol == 1) B200Q_TD(NK, NACC, G_, 1); else B200Q_TD(NK, NACC, G_, 2); } while (0)
#define B200Q_TD_G(NK, NACC) do { if (G == 2) B200Q_TD_NF(NK, NACC, 2); else B200Q_TD_NF(NK, NACC, 4); } while (0)
  if (fs.nkeys == 1) { if (fs.nacc == 2) B200Q_TD_G(1, 2); else B200Q_TD_G(1, 1); }
  else { if (fs.nacc == 2) B200Q_TD_G(2, 2); else B200Q_TD_G(2, 1); }
#undef B200Q_TD_G
#undef B200Q_TD_NF
#undef B200Q_TD
  return 1;
}

// =====================================================================================================================
// WIDE tile aggregates: see TileAggSpec in kernels_fast.cuh
// =====================================================================================================================
template <int FLAV> __device__ __forceinline__ void tw_red(unsigned long long* p, unsigned long long v) {
  if (FLAV == TF_ADD_U64) red_add_u64(p, v);
  else if (FLAV == TF_ADD_F64) red_add_f64(p, as_f64(v));
  else red_min_s64(p, (long long)v);
}
template <int FLAV> __device__ __forceinline__ unsigned long long tw_noop() { return tile_identity(FLAV); }

// rows r0 + 32 j of one decimal128 column (bit j of `ld`): low and high words, one 128-bit load per row when the column is
// 16-byte aligned (an Arrow slice of an 8-byte aligned buffer may not be: two 64-bit loads)
__device__ __forceinline__ void tl_load_dec(const DevCol& c, long long r0, unsigned ld, uint64_t pol, long long (&lo)[4], long long (&hi)[4], unsigned& valid) {
  tl_load(c, PH_I64, r0, ld, false, pol, lo, valid);
  const long long* p = (const long long*)c.values + 2 * r0;
  const bool a16 = ((uintptr_t)c.values & 15) == 0;
#pragma unroll
  for (int j = 0; j < 4; j++) {
    lo[j] = 0; hi[j] = 0;
    if (a16) tl_ld_v2b64(p + 64 * j, (ld >> j) & 1u, pol, lo[j], hi[j]);
    else { tl_ld_b64(p + 64 * j, (ld >> j) & 1u, pol, lo[j]); tl_ld_b64(p + 64 * j + 1, (ld >> j) & 1u, pol, hi[j]); }
  }
}

__device__ __forceinline__ unsigned long long tw_convert(long long v, int cvt) {
  if (cvt == TC_I2F) return f64_bits(__ll2double_rn(v));
  if (cvt == TC_ORDER) return (unsigned long long)total_order_key((uint64_t)v);
  return (unsigned long long)v;
}

// generic update of one hashed slot (keys outside the dense range / NULL keys): the accumulator kinds of AggLayout
__device__ __forceinline__ void tw_slot_update(const AggLayout& lay, const TileAggSpec& ts, unsigned long long* ke, unsigned long long* ae, unsigned flags,
                                               unsigned long long x0, unsigned long long x1, bool valid0, bool valid1) {
  for (int a = 0; a < ts.nacc; a++) {
    const AccOp op = lay.acc[ts.acc[a].lay_acc];
    const int arg = ts.acc[a].arg;
    const bool valid = arg < 0 ? true : (arg == 0 ? valid0 : valid1);
    if (!valid) continue;
    const unsigned long long x = arg == 1 ? x1 : x0;
    unsigned long long* w = ae + op.word;
    switch (op.kind) {
      case ACC_ADD_I64: red_add_u64(w, x); break;
      case ACC_ADD_F64: red_add_f64(w, as_f64(x)); break;
      case ACC_ADD_DEC: { const unsigned long long old = atomicAdd(w, x0); red_add_u64(w + 1, x1 + ((old + x0) < old ? 1ULL : 0ULL)); break; }   // decimal: v0 = low, v1 = high word
      case ACC_COUNT: red_add_u64(w, 1ULL); break;
      case ACC_MIN_I64: case ACC_MIN_F64: red_min_s64(w, (long long)x); break;
      default: red_max_s64(w, (long long)x); break;                // ACC_MAX_I64 / ACC_MAX_F64 (f64 arrives as its totalOrder key)
    }
    slot_mark(ke, flags, op.vbit);
  }
}

template <int NK, int NF, int G, int FLAV>
__global__ void __launch_bounds__(TL_BLOCK, TW_MIN_CTAS(NK, NF)) agg_tile_wide_kernel(const ColTable cols, const TileAggSpec ts, const AggLayout lay, const AggTable tab, long long row_begin, long long n) {
  constexpr unsigned IDX_MASK = 0x0FFFFFFFu, ALWAYS = 1u << 30, FULL = 0xffffffffu;
  __shared__ TileQueue queues[TL_WARPS];
  TileQueue& q = queues[threadIdx.x >> 5];
  const unsigned lane = threadIdx.x & 31, qw = lane & (G - 1);
  const long long gwarp = (long long)blockIdx.x * TL_WARPS + (threadIdx.x >> 5), nwarps = (long long)gridDim.x * TL_WARPS;
  const long long ntiles = (n + TL_ROWS - 1) / TL_ROWS;
  const TileWord tw = ts.word[qw];                                  // this lane's entry word (branch-free selectors)
  const bool use1 = tw.srcsel == 1, use_c = tw.srcsel == 2;
  const unsigned long long noop = tw_noop<FLAV>();
  unsigned long long* const sink = ts.sink + ((gwarp & (FAST_SINK_WARPS - 1)) << 2) + (lane & 3);
  const uint64_t pol = tl_policy_evict_first();
  const bool dec = ts.arg_is_dec != 0;

  long long f[NF > 0 ? NF : 1][4]; unsigned fv[NF > 0 ? NF : 1];
  tl_load_filters<NF>(cols, ts.frange, row_begin, gwarp * TL_ROWS + lane, n, pol, f, fv);
  for (long long tile = gwarp; tile < ntiles; tile += nwarps) {
    const long long rel0 = tile * TL_ROWS + lane, row0 = row_begin + rel0;
    const unsigned alive = tl_pass<NF>(ts.frange, f, fv, tl_rows_in(rel0, n));       // filter first, as in agg_tile_dense_kernel
    long long k0[4], k1[4], a0[4], a1[4]; unsigned kv0, kv1 = 0xF, av0 = 0xF, av1 = 0xF;
    tl_column<NF>(cols, ts.frange, f, fv, ts.key_col[0], ts.key_phys[0], row0, alive, true, pol, k0, kv0);
    if (NK == 2) tl_column<NF>(cols, ts.frange, f, fv, ts.key_col[1], ts.key_phys[1], row0, alive, true, pol, k1, kv1);
    else { k1[0] = k1[1] = k1[2] = k1[3] = 0; }
    a0[0] = a0[1] = a0[2] = a0[3] = 0; a1[0] = a1[1] = a1[2] = a1[3] = 0;
    if (dec) {
      tl_load_dec(cols.col[ts.arg_col[0]], row0, alive, pol, a0, a1, av0); av1 = av0;
      if (ts.dec_mul != 1) {                                         // TryCast to a larger scale (cannot overflow: the precision grows at least as much)
#pragma unroll
        for (int j = 0; j < 4; j++) { const i128_t v = mk128((uint64_t)a0[j], (uint64_t)a1[j]) * (i128_t)ts.dec_mul; a0[j] = (long long)lo64(v); a1[j] = (long long)hi64(v); }
      }
    }
    else {
      if (ts.nargs > 0) tl_column<NF>(cols, ts.frange, f, fv, ts.arg_col[0], ts.arg_phys[0], row0, alive, ts.arg_values[0] != 0, pol, a0, av0);
      if (ts.nargs > 1) tl_column<NF>(cols, ts.frange, f, fv, ts.arg_col[1], ts.arg_phys[1], row0, alive, ts.arg_values[1] != 0, pol, a1, av1);
    }
    tl_load_filters<NF>(cols, ts.frange, row_begin, rel0 + nwarps * TL_ROWS, n, pol, f, fv);   // the next tile's, in flight from here on
    const unsigned knull = (~kv0 | (NK == 2 ? ~kv1 : 0u)) & 0xFu;
    int total = 0; unsigned fb = 0;
#pragma unroll
    for (int j = 0; j < 4; j++) {
      const unsigned long long d0 = (unsigned long long)(k0[j] - ts.dense_base), d1 = (unsigned long long)(k1[j] - ts.dense_base1);
      const unsigned long long di = NK == 1 ? d0 : d0 * ts.dense_r1 + d1;
      const bool inr = NK == 1 ? d0 < ts.dense_cap : (d0 < ts.dense_cap0 && d1 < ts.dense_r1);
      const bool live = (alive >> j) & 1u;
      const bool in = inr && live && !((knull >> j) & 1u);
      fb |= (unsigned)(live && !in) << j;
      const unsigned m = __ballot_sync(FULL, in);
      if (in) {
        const int at = total + __popc(m & lanemask_lt());
        q.idx[at] = (unsigned)di | (((av0 >> j) & 1u) << 28) | (((av1 >> j) & 1u) << 29) | ALWAYS;
        q.v0[at] = dec ? (unsigned long long)a0[j] : tw_convert(a0[j], ts.arg_cvt[0]);
        q.v1[at] = dec ? (unsigned long long)a1[j] : tw_convert(a1[j], ts.arg_cvt[1]);
      }
      total += __popc(m);
    }
    __syncwarp();
    for (int e0 = 0; e0 < total; e0 += 32 / G) {
      const int e = e0 + (int)(lane / G);
      const bool live = e < total;
      const int er = live ? e : 0;
      const unsigned pk = q.idx[er];
      const unsigned long long x = use1 ? q.v1[er] : q.v0[er];
      unsigned long long val = use_c ? tw.cst : (((x >> tw.sh) & tw.msk) ^ tw.inv);
      const bool on = live && ((pk >> tw.gate) & 1u);
      val = on ? val : noop;
      tw_red<FLAV>(live ? ts.dense_tab + (uint64_t)(pk & IDX_MASK) * G + qw : sink, val);
    }
    __syncwarp();
    if (__any_sync(FULL, fb != 0)) {                                // NULL / out-of-range keys (rare): hashed slots, generic accumulators
#pragma unroll
      for (int j = 0; j < 4; j++) {
        bool inserted = false;
        if ((fb >> j) & 1u) {
          const unsigned kn = ((~kv0 >> j) & 1u) | (NK == 2 ? (((~kv1 >> j) & 1u) << 1) : 0u);
          uint64_t kw[2] = {(kn & 1u) ? 0ULL : (uint64_t)k0[j], (NK == 2 && !(kn & 2u)) ? (uint64_t)k1[j] : 0ULL};
          unsigned fl = 0;
          const uint64_t si = agg_find_or_insert(lay, tab, kw, kn, agg_hash2(kw[0], kw[1], kn), &fl, &inserted);
          if (si == AGG_NO_SLOT) { const unsigned long long at = atomicAdd(tab.counters + 1, 1ULL); tab.deferred[at] = (uint32_t)(rel0 + 32 * j); }
          else tw_slot_update(lay, ts, tab.keys + si * (uint64_t)lay.kstride, tab.accs + si * (uint64_t)lay.astride, fl,
                              dec ? (unsigned long long)a0[j] : tw_convert(a0[j], ts.arg_cvt[0]), dec ? (unsigned long long)a1[j] : tw_convert(a1[j], ts.arg_cvt[1]),
                              (av0 >> j) & 1u, (av1 >> j) & 1u);
        }
        const unsigned bl = __ballot_sync(FULL, inserted);
        if (lane == 0 && bl) atomicAdd(tab.counters, (unsigned long long)__popc(bl));
      }
    }
  }
}

int launch_agg_tile_wide(const ColTable& cols, const TileAggSpec& ts, const AggLayout& lay, const AggTable& tab, int64_t row_begin, int64_t n, cudaStream_t s) {
  if (n <= 0 || ts.filt_never) return 0;
  const int64_t units = ((n + TL_ROWS - 1) / TL_ROWS + TL_WARPS - 1) / TL_WARPS;
#define B200Q_TW(NK, NF, G_, FL) do { auto k_ = agg_tile_wide_kernel<NK, NF, G_, FL>; k_<<<tile_grid(k_, units), TL_BLOCK, 0, s>>>(cols, ts, lay, tab, row_begin, n); } while (0)
#define B200Q_TW_FL(NK, NF, G_) do { if (ts.flavour == TF_ADD_U64) B200Q_TW(NK, NF, G_, TF_ADD_U64); else if (ts.flavour == TF_ADD_F64) B200Q_TW(NK, NF, G_, TF_ADD_F64); else B200Q_TW(NK, NF, G_, TF_MIN_S64); } while (0)
#define B200Q_TW_G(NK, NF) do { if (ts.G == 2) B200Q_TW_FL(NK, NF, 2); else if (ts.G == 4) B200Q_TW_FL(NK, NF, 4); else B200Q_TW_FL(NK, NF, 8); } while (0)
#define B200Q_TW_NF(NK) do { if (ts.nfcol == 0) B200Q_TW_G(NK, 0); else if (ts.nfcol == 1) B200Q_TW_G(NK, 1); else B200Q_TW_G(NK, 2); } while (0)
  if (ts.nkeys == 1) B200Q_TW_NF(1); else B200Q_TW_NF(2);
#undef B200Q_TW_NF
#undef B200Q_TW_G
#undef B200Q_TW_FL
#undef B200Q_TW
  return 1;
}

// ---- dense table of the wide aggregates: identities, occupancy, decimal carries, emit
__global__ void __launch_bounds__(256) tile_wide_fill_kernel(unsigned long long* tab, unsigned long long nwords, unsigned long long v) {
  for (unsigned long long i = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x; i < nwords; i += (unsigned long long)gridDim.x * blockDim.x) tab[i] = v;
}
int launch_tile_wide_init(const TileAggSpec& ts, cudaStream_t s) {
  const unsigned long long nwords = ts.dense_cap * (unsigned long long)ts.G;
  tile_wide_fill_kernel<<<tile_grid(tile_wide_fill_kernel, (int64_t)((nwords + 8191) / 8192)), 256, 0, s>>>(ts.dense_tab, nwords, tile_identity(ts.flavour));
  return 1;
}
// a presence / valid-argument word has seen a row: MIN(0) under TF_MIN_S64, a non-zero count otherwise (an f64 count
// starts at -0.0, whose bits are not 0)
__device__ __forceinline__ bool tw_marked(const TileAggSpec& ts, unsigned long long w) {
  return ts.flavour == TF_MIN_S64 ? w == 0 : ts.flavour == TF_ADD_F64 ? as_f64(w) != 0.0 : w != 0;
}
__device__ __forceinline__ bool tw_present(const TileAggSpec& ts, const unsigned long long* e) { return tw_marked(ts, e[ts.presence_word]); }
__global__ void __launch_bounds__(256) tile_wide_count_kernel(const TileAggSpec ts, unsigned long long* out) {
  unsigned long long c = 0;
  for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < ts.dense_cap; i += (uint64_t)gridDim.x * blockDim.x) c += tw_present(ts, ts.dense_tab + i * ts.G);
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) c += __shfl_xor_sync(0xffffffffu, c, d);
  if ((threadIdx.x & 31) == 0 && c) atomicAdd(out, c);
}
int launch_tile_wide_count(const TileAggSpec& ts, unsigned long long* d_out, cudaStream_t s) {
  tile_wide_count_kernel<<<tile_grid(tile_wide_count_kernel, ((int64_t)ts.dense_cap + 16383) / 16384), 256, 0, s>>>(ts, d_out);
  return 1;
}
// decimal128 SUM pieces {low 32 bits, middle 32 bits, high 64 bits} accumulated with 64-bit adds: move the carries up
__global__ void __launch_bounds__(256) tile_wide_normalise_kernel(const TileAggSpec ts) {
  for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < ts.dense_cap; i += (uint64_t)gridDim.x * blockDim.x) {
    unsigned long long* e = ts.dense_tab + i * ts.G + ts.dec_word;
    unsigned long long w0 = e[0], w1 = e[1], w2 = e[2];
    w1 += w0 >> 32; w0 &= 0xFFFFFFFFULL; w2 += w1 >> 32; w1 &= 0xFFFFFFFFULL;
    e[0] = w0; e[1] = w1; e[2] = w2;
  }
}
int launch_tile_wide_normalise(const TileAggSpec& ts, cudaStream_t s) {
  if (ts.dec_word == 0xFF) return 0;
  tile_wide_normalise_kernel<<<tile_grid(tile_wide_normalise_kernel, ((int64_t)ts.dense_cap + 16383) / 16384), 256, 0, s>>>(ts);
  return 1;
}
__global__ void __launch_bounds__(256) tile_wide_emit_kernel(const TileAggSpec ts, const AggLayout lay, const EmitTable emit, unsigned long long* out_count) {
  const unsigned lane = threadIdx.x & 31;
  const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
  const uint64_t rounds = (ts.dense_cap + stride - 1) / stride;
  for (uint64_t it = 0; it < rounds; it++) {
    const uint64_t i = it * stride + blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    const unsigned long long* e = ts.dense_tab + i * ts.G;
    const bool occ = i < ts.dense_cap && tw_present(ts, e);
    const unsigned m = __ballot_sync(0xffffffffu, occ);
    if (!m) continue;
    unsigned long long base = 0;
    if (lane == 0) base = atomicAdd(out_count, (unsigned long long)__popc(m));
    base = __shfl_sync(0xffffffffu, base, 0);
    if (!occ) continue;
    const unsigned long long at = base + __popc(m & lanemask_lt());
    // present the entry as a hashed slot: key entry [hdr][keys], accumulator entry in AggLayout word order, valid bits
    unsigned long long ke[4] = {0, 0, 0, 0}, slot[16];
    ke[lay.key_word[0]] = (unsigned long long)(ts.nkeys == 1 ? ts.dense_base + (long long)i : ts.dense_base + (long long)(i / ts.dense_r1));
    if (ts.nkeys == 2) ke[lay.key_word[1]] = (unsigned long long)(ts.dense_base1 + (long long)(i % ts.dense_r1));
#pragma unroll
    for (int w = 0; w < 16; w++) slot[w] = 0;
    unsigned flags = 0;
    for (int a = 0; a < ts.nacc; a++) {
      const AccOp op = lay.acc[ts.acc[a].lay_acc];
      const unsigned long long d = e[ts.acc[a].w0];
      switch (ts.acc[a].recon) {
        case TR_COPY: slot[op.word] = d; break;
        case TR_NOT: slot[op.word] = ~d; break;
        case TR_F2I: slot[op.word] = (unsigned long long)__double2ll_rn(as_f64(d)); break;
        default: {                                                  // TR_DEC3 (normalised: the low two pieces are < 2^32)
          const unsigned long long w0 = d, w1 = e[ts.acc[a].w0 + 1], w2 = e[ts.acc[a].w0 + 2];
          const unsigned long long c1 = w1 + (w0 >> 32);
          slot[op.word] = (w0 & 0xFFFFFFFFULL) | (c1 << 32); slot[op.word + 1] = w2 + (c1 >> 32);
          break;
        }
      }
      const uint8_t vw = ts.acc[a].valid_word;
      const bool valid = vw == 0xFF ? true : tw_marked(ts, e[vw]);
      if (op.vbit != 0xFF && valid) flags |= 1u << op.vbit;
    }
    emit_row_columns(emit, at, ke, slot, flags);
  }
}
int launch_tile_wide_emit(const TileAggSpec& ts, const AggLayout& lay, const EmitTable& emit, unsigned long long* d_out_count, cudaStream_t s) {
  tile_wide_emit_kernel<<<tile_grid(tile_wide_emit_kernel, ((int64_t)ts.dense_cap + 16383) / 16384), 256, 0, s>>>(ts, lay, emit, d_out_count);
  return 1;
}

}  // namespace b200q
