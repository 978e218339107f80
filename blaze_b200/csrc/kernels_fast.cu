// Specialised streaming HashAgg update kernels for the shapes TPC-DS q1/q3/q6 produce:
//   * 1-2 integer grouping columns read straight from the Arrow buffers (no row encoding: K4 is gone),
//   * up to 4 fused `column <cmp> literal` conjuncts (the FilterExec below the agg),
//   * 1-2 accumulators of the "64-bit add" class: SUM(int column), COUNT(column), COUNT(*).
//
// What bounds them (tools/microbench/atomics.cu measures it): the input stream runs at HBM speed but every row also
// needs a random read-modify-write into the L2-resident group table, and the chip retires a bounded number of
// scattered 32-byte RED sector operations per second.  So the design goal is ONE RED sector per row:
//   - hashed (agg_lean_hash_kernel): key entries {hdr,key..} and accumulator entries live in two arrays (a RED on a
//     sector that was just probed costs 2x: the read copies must be invalidated); the probe is a single 16-byte
//     load, collided rows are re-probed 32 at a time from a per-warp stack, and the two accumulators of a row are
//     updated by the SAME red.add.u64 instruction from two adjacent lanes (one sector operation);
//   - DENSE (integer keys whose values span a small range, e.g. TPC-DS surrogate keys; two keys are mapped onto
//     one composite index): no probe at all; an entry is 2 or 4 words updated by 2 or 4 adjacent lanes in one
//     instruction.  Keys outside the range and NULL keys take the hash table.
//       agg_lean_dense_kernel  bare M1 shape: "gangs" of G lanes own G consecutive rows and load them with one wide
//                              load each (same addresses: one LSU access); in step s the gang updates row s
//       agg_dense_row_kernel   filters / two keys / typed inputs: one row per lane, operands handed to the G lanes
//                              of a group by shuffle
//       agg_dense_smem_kernel  few groups: CTA-private table in shared memory, flushed once
//
// REDs are issued UNCONDITIONALLY: ptxas if-converts a predicated `red` into `@P ATOMG ... RZ` (an atomic
// with a return path); lanes with nothing to add send +0 to their warp's private sink sector instead.
#include <algorithm>
#include <cstdlib>
#include <cuda_runtime.h>
#include <stdint.h>

#include "agg_device.cuh"
#include "kernels_fast.cuh"

namespace b200q {

constexpr int FA_BLOCK = 256;

// streaming load: bypass L1 and mark the line evict-first in L2 so the input stream does not push the
// group table out of L2
__device__ __forceinline__ uint64_t make_evict_first_policy() {
  uint64_t pol; asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol)); return pol;
}
__device__ __forceinline__ long long ld_stream_s64(const long long* p) {
  long long v; const uint64_t pol = make_evict_first_policy();
  asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.s64 %0, [%1], %2;" : "=l"(v) : "l"(p), "l"(pol)); return v;
}
__device__ __forceinline__ bool col_valid(const DevCol& c, long long i) {
  if (!c.validity) return true;
  const unsigned long long bi = (unsigned long long)i + c.bit_offset;
  return (__ldg(c.validity + (bi >> 3)) >> (bi & 7)) & 1;
}
__device__ __forceinline__ long long col_load_int(const DevCol& c, int phys, long long i) {
  switch (phys) {
    case PH_I64: return ld_stream_s64((const long long*)c.values + i);
    case PH_I32: return (long long)__ldg((const int32_t*)c.values + i);
    case PH_I16: return (long long)__ldg((const int16_t*)c.values + i);
    case PH_I8: return (long long)__ldg((const int8_t*)c.values + i);
    default: { const unsigned long long bi = (unsigned long long)i + c.bit_offset; return (__ldg((const uint8_t*)c.values + (bi >> 3)) >> (bi & 7)) & 1; }
  }
}
__device__ __forceinline__ bool cmp_apply(int op, long long a, long long b) {
  switch (op) { case CMP_EQ: return a == b; case CMP_NE: return a != b; case CMP_LT: return a < b; case CMP_LE: return a <= b; case CMP_GT: return a > b; default: return a >= b; }
}
__device__ __forceinline__ unsigned long long* warp_sink(const FastSpec& fs, long long gwarp, unsigned m) {
  return fs.sink + ((gwarp & (FAST_SINK_WARPS - 1)) << 2) + (m & 3);
}

// 64-bit wrapping add on shared memory made of native 32-bit shared atomics: low half with the old value returned,
// high half plus the carry.  Exact mod 2^64 in any order (every carry is observed exactly once).
__device__ __forceinline__ void smem_add64(unsigned* w, unsigned long long v) {
  const unsigned lo = (unsigned)v, hi = (unsigned)(v >> 32);
  unsigned carry = 0;
  if (lo) { const unsigned old = atomicAdd(w, lo); carry = old + lo < old; }
  if (hi + carry) atomicAdd(w + 1, hi + carry);
}

template <int NK>
__device__ __forceinline__ bool dense_index(const FastSpec& fs, long long k0, long long k1, unsigned long long& idx) { return dense_index_of<NK>(fs, k0, k1, idx); }

// ---------------------------------------------------------------------------------------------------
// LEAN dense kernel: the hot loop of the M1 shape with everything resolved at compile time.
// Preconditions (checked on the host per launch): one int64 key column, accumulator/filter columns int64,
// none of them carries a validity bitmap, base pointers 32-byte aligned, row_begin % 4 == 0.
// Per 32 rows a warp issues 1 (+1) wide streaming loads and G REDG: ~2 instructions per row.
// ---------------------------------------------------------------------------------------------------
template <int G> struct i64xG { long long v[G]; };
__device__ __forceinline__ i64xG<4> ld_stream_vec(const long long* p, i64xG<4>*) {     // two 128-bit loads: the widest on sm_90
  i64xG<4> r; uint64_t pol;
  asm("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));                // not volatile: hoisted out of the loop
  asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.v2.b64 {%0,%1}, [%4], %5;\n\tld.global.nc.L1::no_allocate.L2::cache_hint.v2.b64 {%2,%3}, [%4+16], %5;"
               : "=l"(r.v[0]), "=l"(r.v[1]), "=l"(r.v[2]), "=l"(r.v[3]) : "l"(p), "l"(pol));
  return r;
}
__device__ __forceinline__ i64xG<2> ld_stream_vec(const long long* p, i64xG<2>*) {
  i64xG<2> r;
  asm volatile("ld.global.nc.L1::no_allocate.v2.b64 {%0,%1}, [%2];" : "=l"(r.v[0]), "=l"(r.v[1]) : "l"(p));
  return r;
}
__device__ __forceinline__ i64xG<1> ld_stream_vec(const long long* p, i64xG<1>*) {
  i64xG<1> r;
  asm volatile("ld.global.nc.L1::no_allocate.b64 %0, [%1];" : "=l"(r.v[0]) : "l"(p));
  return r;
}
template <int G>
__device__ __forceinline__ i64xG<G> ld_rows(const long long* col, long long rel0, long long n) {
  if (rel0 + G <= n) return ld_stream_vec(col + rel0, (i64xG<G>*)nullptr);
  i64xG<G> r;
#pragma unroll
  for (int s = 0; s < G; s++) r.v[s] = rel0 + s < n ? __ldg(col + rel0 + s) : 0;
  return r;
}

template <int NACC, int G, int NK>
__global__ void __launch_bounds__(FA_BLOCK) agg_lean_dense_kernel(const ColTable cols, const FastSpec fs, const AggLayout lay, const AggTable tab,
                                                                  long long row_begin, long long n) {
  constexpr int U = G == 2 ? 4 : 2;                             // 32-row units in flight per warp
  const unsigned lane = threadIdx.x & 31, m = lane % G, gl = lane - m;
  const long long gwarp = (long long)blockIdx.x * (FA_BLOCK / 32) + (threadIdx.x >> 5), nwarps = (long long)gridDim.x * (FA_BLOCK / 32);
  const long long nunits = (n + 31) / 32;
  const long long* kcol = (const long long*)cols.col[fs.key_col[0]].values + row_begin;
  const long long* kcol1 = NK == 2 ? (const long long*)cols.col[fs.key_col[1]].values + row_begin : nullptr;
  const int src = fs.dense_word_src[m];                         // -1: row counter (+1), -2: padding (+0), j: accumulator j, 2+j: valid arguments of j (+1: inputs are non-null here)
  const bool has_acc = src >= 0 && src < NACC;
  const bool is_add = has_acc && fs.acc[has_acc ? src : 0].kind == FAST_ACC_ADD;
  const long long* vcol = is_add ? (const long long*)cols.col[fs.acc[src].col].values + row_begin : nullptr;
  const long long cst = src == -2 ? 0 : 1;
  unsigned long long* const sink = warp_sink(fs, gwarp, m);
  unsigned long long* const dtab = fs.dense_tab + m;

  for (long long unit0 = gwarp * U; unit0 < nunits; unit0 += nwarps * U) {
    i64xG<G> k[U], k1[NK == 2 ? U : 1], v[U]; bool alive[U][G];
#pragma unroll
    for (int u = 0; u < U; u++) {
      const long long rel0 = (unit0 + u) * 32 + gl;
      k[u] = ld_rows<G>(kcol, rel0, n);
      if (NK == 2) k1[u] = ld_rows<G>(kcol1, rel0, n);
      if (is_add) v[u] = ld_rows<G>(vcol, rel0, n);
      else {
#pragma unroll
        for (int s = 0; s < G; s++) v[u].v[s] = cst;
      }
#pragma unroll
      for (int s = 0; s < G; s++) alive[u][s] = rel0 + s < n;
    }
    for (int f = 0; f < fs.nfilt; f++) {                        // fused FilterExec conjuncts
      const long long* fcol = (const long long*)cols.col[fs.filt[f].col].values + row_begin;
#pragma unroll
      for (int u = 0; u < U; u++) {
        const i64xG<G> x = ld_rows<G>(fcol, (unit0 + u) * 32 + gl, n);
#pragma unroll
        for (int s = 0; s < G; s++) alive[u][s] = alive[u][s] && cmp_apply(fs.filt[f].op, x.v[s], fs.filt[f].lit);
      }
    }
    bool oor = false;
#pragma unroll
    for (int u = 0; u < U; u++) {
#pragma unroll
      for (int s = 0; s < G; s++) {
        unsigned long long idx;
        const bool in = dense_index<NK>(fs, k[u].v[s], NK == 2 ? k1[NK == 2 ? u : 0].v[s] : 0, idx) && alive[u][s];
        oor |= alive[u][s] && !in;
        red_add_u64(in ? dtab + idx * G : sink, in ? (unsigned long long)v[u].v[s] : 0ULL);     // G lanes -> 1 sector
      }
    }
    // keys outside the dense range (rare): lane 0 of the gang routes the row through the hash table
    if (__any_sync(0xffffffffu, oor)) {
#pragma unroll
      for (int u = 0; u < U; u++) {
#pragma unroll
        for (int s = 0; s < G; s++) {
          unsigned long long idx;
          const bool in = dense_index<NK>(fs, k[u].v[s], NK == 2 ? k1[NK == 2 ? u : 0].v[s] : 0, idx);
          bool inserted = false;
          if (alive[u][s] && !in && m == 0) {
            const long long rel = (unit0 + u) * 32 + gl + s;
            uint64_t kw[2] = {(uint64_t)k[u].v[s], NK == 2 ? (uint64_t)k1[NK == 2 ? u : 0].v[s] : 0ULL};
            unsigned fl;
            const uint64_t si = agg_find_or_insert(lay, tab, kw, 0, agg_hash_words(kw, NK, 0), &fl, &inserted);
            if (si == AGG_NO_SLOT) { const unsigned long long at = atomicAdd(tab.counters + 1, 1ULL); tab.deferred[at] = (uint32_t)rel; }
            else {
              unsigned long long* const p = tab.accs + si * (uint64_t)lay.astride;
#pragma unroll
              for (int j = 0; j < NACC; j++) {
                const unsigned long long x = fs.acc[j].kind == FAST_ACC_ADD ? (unsigned long long)__ldg((const long long*)cols.col[fs.acc[j].col].values + row_begin + rel) : 1ULL;
                atomicAdd(p + fs.acc[j].word, x);
                slot_mark(tab.keys + si * (uint64_t)lay.kstride, fl, fs.acc[j].vbit);
              }
            }
          }
          const unsigned b = __ballot_sync(0xffffffffu, inserted);
          if (lane == 0 && b) atomicAdd(tab.counters, (unsigned long long)__popc(b));
        }
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------------
// Dense kernel, one row per lane: fused filters, two keys, 4-word entries, typed / nullable inputs.  The gang form
// above evaluates every row redundantly in the G lanes of its gang — free for the bare M1 shape, but with conjuncts,
// a composite index or typed loads the kernel becomes issue-bound (M2: 5.2e10 rows/s; typed M1: 2.2e10).  Here every
// lane owns one row, and the G words of an entry are still updated by ONE instruction: in step t the G lanes of a
// group receive the entry index, validity flags and operands of the group's t-th row by shuffle and lane q adds
// the value of word q.
// TYPED = false: non-null 8-byte-aligned int64 columns; TYPED = true: any integer width + validity bitmaps.
// ---------------------------------------------------------------------------------------------------
enum { DW_ZERO = 0, DW_ONE, DW_ADD0, DW_ADD1, DW_VALID0, DW_VALID1 };     // what an entry word accumulates
template <int NACC, int NK, int G, bool TYPED>
__global__ void __launch_bounds__(FA_BLOCK) agg_dense_row_kernel(const ColTable cols, const FastSpec fs, const AggLayout lay, const AggTable tab,
                                                                 long long row_begin, long long n) {
  constexpr int U = 4;
  constexpr unsigned IDX_MASK = 0x0FFFFFFFu;                    // dense_cap <= 2^26; bits 28/29: argument 0/1 is not NULL
  const unsigned lane = threadIdx.x & 31, q = lane & (G - 1);
  const long long gwarp = (long long)blockIdx.x * (FA_BLOCK / 32) + (threadIdx.x >> 5), nwarps = (long long)gridDim.x * (FA_BLOCK / 32);
  const long long nunits = (n + 31) / 32;
  const bool add0 = fs.acc[0].kind == FAST_ACC_ADD, add1 = NACC == 2 && fs.acc[1].kind == FAST_ACC_ADD;
  // this lane's entry word
  int wkind;
  {
    const int src = fs.dense_word_src[q];
    if (src == -1) wkind = DW_ONE; else if (src == -2) wkind = DW_ZERO;
    else if (src >= 2) wkind = src == 2 ? DW_VALID0 : DW_VALID1;
    else if (src == 0) wkind = add0 ? DW_ADD0 : DW_VALID0;
    else wkind = add1 ? DW_ADD1 : DW_VALID1;
  }
  unsigned long long* const sink = warp_sink(fs, gwarp, lane);

  for (long long unit0 = gwarp * U; unit0 < nunits; unit0 += nwarps * U) {
    long long k0[U], k1[U]; unsigned long long v0[U], v1[U]; bool alive[U]; unsigned meta[U];     // meta: bit0/1 key NULL, bit2/3 argument valid
#pragma unroll
    for (int u = 0; u < U; u++) {
      const long long rel = (unit0 + u) * 32 + lane, row = row_begin + rel;
      alive[u] = rel < n; meta[u] = 0xC; k0[u] = 0; k1[u] = 0; v0[u] = 0; v1[u] = 0;
      if (!alive[u]) continue;
      if (!TYPED) {
        k0[u] = ld_stream_vec((const long long*)cols.col[fs.key_col[0]].values + row, (i64xG<1>*)nullptr).v[0];
        if (NK == 2) k1[u] = ld_stream_vec((const long long*)cols.col[fs.key_col[1]].values + row, (i64xG<1>*)nullptr).v[0];
        if (add0) v0[u] = (unsigned long long)ld_stream_vec((const long long*)cols.col[fs.acc[0].col].values + row, (i64xG<1>*)nullptr).v[0];
        if (add1) v1[u] = (unsigned long long)ld_stream_vec((const long long*)cols.col[fs.acc[1].col].values + row, (i64xG<1>*)nullptr).v[0];
      } else {
        { const DevCol& c = cols.col[fs.key_col[0]]; if (col_valid(c, row)) k0[u] = col_load_int(c, fs.key_phys[0], row); else meta[u] |= 1u; }
        if (NK == 2) { const DevCol& c = cols.col[fs.key_col[1]]; if (col_valid(c, row)) k1[u] = col_load_int(c, fs.key_phys[1], row); else meta[u] |= 2u; }
        if (fs.acc[0].col >= 0) {
          const DevCol& c = cols.col[fs.acc[0].col];
          if (!col_valid(c, row)) meta[u] &= ~4u; else if (add0) v0[u] = (unsigned long long)col_load_int(c, fs.acc[0].phys, row);
        }
        if (NACC == 2 && fs.acc[1].col >= 0) {
          const DevCol& c = cols.col[fs.acc[1].col];
          if (!col_valid(c, row)) meta[u] &= ~8u; else if (add1) v1[u] = (unsigned long long)col_load_int(c, fs.acc[1].phys, row);
        }
      }
    }
    for (int f = 0; f < fs.nfilt; f++) {                        // fused FilterExec conjuncts (NULL -> row dropped)
      const DevCol& c = cols.col[fs.filt[f].col];
#pragma unroll
      for (int u = 0; u < U; u++) {
        const long long row = row_begin + (unit0 + u) * 32 + lane;
        if (!alive[u]) continue;
        if (!TYPED) alive[u] = cmp_apply(fs.filt[f].op, ld_stream_vec((const long long*)c.values + row, (i64xG<1>*)nullptr).v[0], fs.filt[f].lit);
        else alive[u] = col_valid(c, row) && cmp_apply(fs.filt[f].op, col_load_int(c, fs.filt[f].phys, row), fs.filt[f].lit);
      }
    }
#pragma unroll
    for (int u = 0; u < U; u++) {
      unsigned long long di;
      const bool in = dense_index<NK>(fs, k0[u], k1[u], di) && alive[u] && !(meta[u] & 3u);
      const unsigned pk = in ? ((unsigned)di | ((meta[u] & 0xCu) << 26)) : 0xFFFFFFFFu;
#pragma unroll
      for (int t = 0; t < G; t++) {                             // step t: the G lanes of a group update the G words of the group's t-th row
        const unsigned opk = __shfl_sync(0xffffffffu, pk, t, G);
        const unsigned long long ov0 = add0 ? __shfl_sync(0xffffffffu, v0[u], t, G) : 0ULL;
        const unsigned long long ov1 = add1 ? __shfl_sync(0xffffffffu, v1[u], t, G) : 0ULL;
        const bool live = opk != 0xFFFFFFFFu;
        unsigned long long val;
        switch (wkind) {
          case DW_ONE: val = 1; break;
          case DW_ADD0: val = ov0; break;                       // a NULL argument was loaded as 0
          case DW_ADD1: val = ov1; break;
          case DW_VALID0: val = (opk >> 28) & 1u; break;
          case DW_VALID1: val = (opk >> 29) & 1u; break;
          default: val = 0; break;
        }
        red_add_u64(live ? fs.dense_tab + (uint64_t)(opk & IDX_MASK) * G + q : sink, live ? val : 0ULL);
      }
      // keys outside the dense range / NULL keys (rare): straight to the hashed slots
      const bool fb = alive[u] && !in;
      if (__any_sync(0xffffffffu, fb)) {
        bool inserted = false;
        if (fb) {
          uint64_t kw[2] = {(uint64_t)k0[u], NK == 2 ? (uint64_t)k1[u] : 0ULL};
          const unsigned knull = meta[u] & 3u;
          unsigned fl = 0;
          const uint64_t si = agg_find_or_insert(lay, tab, kw, knull, agg_hash2(kw[0], kw[1], knull), &fl, &inserted);
          if (si == AGG_NO_SLOT) { const unsigned long long at = atomicAdd(tab.counters + 1, 1ULL); tab.deferred[at] = (uint32_t)((unit0 + u) * 32 + lane); }
          else {
            unsigned long long* const p = tab.accs + si * (uint64_t)lay.astride;
            unsigned long long* const ke = tab.keys + si * (uint64_t)lay.kstride;
            if (meta[u] & 4u) { red_add_u64(p + fs.acc[0].word, add0 ? v0[u] : 1ULL); slot_mark(ke, fl, fs.acc[0].vbit); }
            if (NACC == 2 && (meta[u] & 8u)) { red_add_u64(p + fs.acc[1].word, add1 ? v1[u] : 1ULL); slot_mark(ke, fl, fs.acc[1].vbit); }
          }
        }
        const unsigned bl = __ballot_sync(0xffffffffu, inserted);
        if (lane == 0 && bl) atomicAdd(tab.counters, (unsigned long long)__popc(bl));
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------------
// EXPERIMENTAL (b200q_conf.agg_hot_key_cache, off by default; validated on the CPU build only so far): dense kernel
// for SKEWED keys.  Every RED on a hot key serialises in the L2 (Zipf 1.1 over 2^20 keys: 1.5e10 rows/s instead of
// 1.5e11).  Each CTA keeps a direct-mapped write-combining cache of 1024 entries in shared memory: the first key that
// claims a line keeps it for the CTA's lifetime (hot keys show up early and often), its rows are accumulated with
// shared-memory atomics; every other row takes the global RED path of agg_dense_row_kernel.  Lines are added to the
// global table once, at the end.  Non-null 8-byte-aligned int64 inputs only.
// ---------------------------------------------------------------------------------------------------
constexpr int HC_LINES = 1024;
template <int NACC, int NK, int G>
__global__ void __launch_bounds__(FA_BLOCK) agg_dense_hot_kernel(const ColTable cols, const FastSpec fs, const AggLayout lay, const AggTable tab,
                                                                 long long row_begin, long long n) {
  constexpr int U = 4;
  constexpr unsigned IDX_MASK = 0x0FFFFFFFu;
  __shared__ unsigned long long c_key[HC_LINES];                // dense entry index + 1 (0: free line)
  __shared__ unsigned c_acc[HC_LINES * G * 2];                  // the entry's words as 32-bit halves (smem_add64)
  for (int i = threadIdx.x; i < HC_LINES; i += FA_BLOCK) c_key[i] = 0;
  for (int i = threadIdx.x; i < HC_LINES * G * 2; i += FA_BLOCK) c_acc[i] = 0;
  __syncthreads();
  const unsigned lane = threadIdx.x & 31, q = lane & (G - 1);
  const long long gwarp = (long long)blockIdx.x * (FA_BLOCK / 32) + (threadIdx.x >> 5), nwarps = (long long)gridDim.x * (FA_BLOCK / 32);
  const long long nunits = (n + 31) / 32;
  const bool add0 = fs.acc[0].kind == FAST_ACC_ADD, add1 = NACC == 2 && fs.acc[1].kind == FAST_ACC_ADD;
  auto word_kind = [&](int m) {                                 // what word m of an entry accumulates (non-null inputs: every argument counts)
    const int src = fs.dense_word_src[m];
    return src == -1 ? DW_ONE : src == -2 ? DW_ZERO : src >= 2 ? DW_ONE : src == 0 ? (add0 ? DW_ADD0 : DW_ONE) : (add1 ? DW_ADD1 : DW_ONE);
  };
  int wk[G];
#pragma unroll
  for (int m = 0; m < G; m++) wk[m] = word_kind(m);
  const int wkind = word_kind((int)q);
  unsigned long long* const sink = warp_sink(fs, gwarp, lane);

  for (long long unit0 = gwarp * U; unit0 < nunits; unit0 += nwarps * U) {
    long long k0[U], k1[U]; unsigned long long v0[U], v1[U]; bool alive[U];
#pragma unroll
    for (int u = 0; u < U; u++) {
      const long long rel = (unit0 + u) * 32 + lane, row = row_begin + rel;
      alive[u] = rel < n; k0[u] = 0; k1[u] = 0; v0[u] = 0; v1[u] = 0;
      if (!alive[u]) continue;
      k0[u] = ld_stream_vec((const long long*)cols.col[fs.key_col[0]].values + row, (i64xG<1>*)nullptr).v[0];
      if (NK == 2) k1[u] = ld_stream_vec((const long long*)cols.col[fs.key_col[1]].values + row, (i64xG<1>*)nullptr).v[0];
      if (add0) v0[u] = (unsigned long long)ld_stream_vec((const long long*)cols.col[fs.acc[0].col].values + row, (i64xG<1>*)nullptr).v[0];
      if (add1) v1[u] = (unsigned long long)ld_stream_vec((const long long*)cols.col[fs.acc[1].col].values + row, (i64xG<1>*)nullptr).v[0];
    }
    for (int f = 0; f < fs.nfilt; f++) {                        // fused FilterExec conjuncts
      const long long* fcol = (const long long*)cols.col[fs.filt[f].col].values + row_begin;
#pragma unroll
      for (int u = 0; u < U; u++) {
        const long long rel = (unit0 + u) * 32 + lane;
        if (alive[u]) alive[u] = cmp_apply(fs.filt[f].op, ld_stream_vec(fcol + rel, (i64xG<1>*)nullptr).v[0], fs.filt[f].lit);
      }
    }
#pragma unroll
    for (int u = 0; u < U; u++) {
      unsigned long long di;
      const bool in = dense_index<NK>(fs, k0[u], k1[u], di) && alive[u];
      bool cached = false;
      if (in) {
        const unsigned line = (unsigned)((di * 0x9E3779B97F4A7C15ULL) >> 54);                     // 1024 lines
        const unsigned long long mine = di + 1;
        unsigned long long cur = *(volatile unsigned long long*)&c_key[line];
        if (cur == 0) { cur = atomicCAS(&c_key[line], 0ULL, mine); if (cur == 0) cur = mine; }
        if (cur == mine) {
          cached = true;
          unsigned* const e = c_acc + line * (G * 2);
#pragma unroll
          for (int m = 0; m < G; m++) {
            if (wk[m] == DW_ONE) smem_add64(e + 2 * m, 1ULL);
            else if (wk[m] == DW_ADD0) smem_add64(e + 2 * m, v0[u]);
            else if (wk[m] == DW_ADD1) smem_add64(e + 2 * m, v1[u]);
          }
        }
      }
      const unsigned pk = (in && !cached) ? (unsigned)di : 0xFFFFFFFFu;
#pragma unroll
      for (int t = 0; t < G; t++) {                             // the global path: see agg_dense_row_kernel
        const unsigned opk = __shfl_sync(0xffffffffu, pk, t, G);
        const unsigned long long ov0 = add0 ? __shfl_sync(0xffffffffu, v0[u], t, G) : 0ULL;
        const unsigned long long ov1 = add1 ? __shfl_sync(0xffffffffu, v1[u], t, G) : 0ULL;
        const bool live = opk != 0xFFFFFFFFu;
        const unsigned long long val = wkind == DW_ONE ? 1ULL : wkind == DW_ADD0 ? ov0 : wkind == DW_ADD1 ? ov1 : 0ULL;
        red_add_u64(live ? fs.dense_tab + (uint64_t)(opk & IDX_MASK) * G + q : sink, live ? val : 0ULL);
      }
      const bool fb = alive[u] && !in;                          // outside the dense range (rare): hashed slots
      if (__any_sync(0xffffffffu, fb)) {
        bool inserted = false;
        if (fb) {
          uint64_t kw[2] = {(uint64_t)k0[u], NK == 2 ? (uint64_t)k1[u] : 0ULL};
          unsigned fl = 0;
          const uint64_t si = agg_find_or_insert(lay, tab, kw, 0, agg_hash2(kw[0], kw[1], 0), &fl, &inserted);
          if (si == AGG_NO_SLOT) { const unsigned long long at = atomicAdd(tab.counters + 1, 1ULL); tab.deferred[at] = (uint32_t)((unit0 + u) * 32 + lane); }
          else {
            unsigned long long* const p = tab.accs + si * (uint64_t)lay.astride;
            unsigned long long* const ke = tab.keys + si * (uint64_t)lay.kstride;
            red_add_u64(p + fs.acc[0].word, add0 ? v0[u] : 1ULL); slot_mark(ke, fl, fs.acc[0].vbit);
            if (NACC == 2) { red_add_u64(p + fs.acc[1].word, add1 ? v1[u] : 1ULL); slot_mark(ke, fl, fs.acc[1].vbit); }
          }
        }
        const unsigned bl = __ballot_sync(0xffffffffu, inserted);
        if (lane == 0 && bl) atomicAdd(tab.counters, (unsigned long long)__popc(bl));
      }
    }
  }
  __syncthreads();
  for (int line = threadIdx.x; line < HC_LINES; line += FA_BLOCK) {
    const unsigned long long key = c_key[line];
    if (!key) continue;
#pragma unroll
    for (int m = 0; m < G; m++) {
      const unsigned long long val = (unsigned long long)c_acc[(line * G + m) * 2] | ((unsigned long long)c_acc[(line * G + m) * 2 + 1] << 32);
      if (val) red_add_u64(fs.dense_tab + (key - 1) * G + m, val);
    }
  }
}

// skew probe: 65536-bucket histogram of the key hashes of a sample, then its maximum -> hist[65536]
__global__ void __launch_bounds__(256) key_skew_hist_kernel(const DevCol c0, const DevCol c1, int phys0, int phys1, int nkeys, long long n, unsigned* hist) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    if (!col_valid(c0, i) || (nkeys == 2 && !col_valid(c1, i))) continue;
    const uint64_t h = agg_hash2((uint64_t)col_load_int(c0, phys0, i), nkeys == 2 ? (uint64_t)col_load_int(c1, phys1, i) : 0ULL, 0);
    atomicAdd(hist + (h >> 48), 1u);
  }
}
__global__ void __launch_bounds__(256) key_skew_max_kernel(unsigned* hist) {
  unsigned mx = 0;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < 65536; i += gridDim.x * blockDim.x) mx = max(mx, hist[i]);
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) mx = max(mx, __shfl_xor_sync(0xffffffffu, mx, d));
  if ((threadIdx.x & 31) == 0) atomicMax(hist + 65536, mx);
}

// ---------------------------------------------------------------------------------------------------
// LEAN hashed kernel: 1-2 non-null int64 keys, non-null int64 accumulator/filter columns (same preconditions as
// the lean dense kernel), one row per lane, compacted probe rounds.  A lane-parallel probe walk waits, per warp
// step, for the LONGEST collision chain among its rows (a dependent L2 round trip per extra slot with most lanes
// idle: 2.6e10 rows/s on M1).  Here every row gets one first probe in the streaming step; rows that must look at
// another slot are pushed onto a per-warp shared-memory stack (warp-synchronous: no atomics) and re-probed 32 at a
// time, so every probe round issues a full warp of useful loads whatever the chain lengths are (5.6-6.7e10 rows/s).
// With two accumulators the two words of a row are updated by ONE instruction: neighbouring lanes exchange their
// slot / second operand with one shuffle pair and lane L updates acc0 of its own row while lane L^1 updates acc1
// of the same row (step 1: rows of even lanes, step 2: rows of odd lanes).
// ---------------------------------------------------------------------------------------------------
constexpr int LH_BLOCK = 128, LH_U = 4, LH_QCAP = 32 * (LH_U + 1);
template <int NK, bool TYPED> struct LhQueue {
  unsigned long long k0[LH_QCAP]; unsigned long long k1[NK == 2 ? LH_QCAP : 1]; unsigned long long v0[LH_QCAP], v1[LH_QCAP];
  unsigned idx[LH_QCAP], tag[LH_QCAP], row[LH_QCAP];
  uint8_t meta[TYPED ? LH_QCAP : 1];                            // TYPED: bits 0-1 key-is-NULL, bits 2-3 accumulator argument valid
};
enum { LH_HIT = 0, LH_AGAIN = 1, LH_NEW = 2, LH_IDLE = 3 };
constexpr unsigned LH_META_PLAIN = 0xC;                         // no NULL key, both accumulator arguments valid

template <int NK>
__device__ __forceinline__ int lh_eval(const AggTable& tab, int ks, unsigned cap, ulonglong2 hk, unsigned tag, unsigned knull, unsigned long long k0,
                                       unsigned long long k1, unsigned& idx, unsigned& flags) {
  const unsigned t = (unsigned)hk.x;
  if (t == tag) {
    bool hit = (unsigned)(hk.x >> 48) == knull && hk.y == k0;
    if (NK == 2 && hit) hit = ld_relaxed_u64(tab.keys + (uint64_t)idx * ks + 2) == k1;
    if (hit) { flags = (unsigned)(hk.x >> 32); return LH_HIT; }
  } else if (t == TAG_EMPTY) return LH_NEW;
  else if (t == TAG_LOCKED) return LH_AGAIN;                     // being inserted: look at the same slot again
  idx = idx + 1 == cap ? 0 : idx + 1;
  return LH_AGAIN;
}

// one warp step of rows that have a status: inserts for LH_NEW, the paired REDs for hits, push of LH_AGAIN rows
template <int NK, int NACC, bool TYPED>
__device__ __forceinline__ void lh_finish(const FastSpec& fs, const AggLayout& lay, const AggTable& tab, LhQueue<NK, TYPED>& q, int& count, unsigned lane,
                                          unsigned long long* sink, bool has_v1, int st, unsigned idx, unsigned flags, unsigned tag, unsigned meta,
                                          unsigned long long k0, unsigned long long k1, unsigned long long v0, unsigned long long v1, unsigned row) {
  constexpr unsigned NONE = 0xFFFFFFFFu;
  if (__any_sync(0xffffffffu, st == LH_NEW)) {                  // new keys: full insert protocol, one counter update per warp step
    bool inserted = false;
    if (st == LH_NEW) {
      uint64_t kw[2] = {k0, NK == 2 ? k1 : 0ULL};
      const unsigned knull = TYPED ? (meta & 3u) : 0u;
      const uint64_t si = agg_find_or_insert(lay, tab, kw, knull, agg_hash2(k0, NK == 2 ? k1 : 0ULL, knull), &flags, &inserted);
      if (si == AGG_NO_SLOT) { const unsigned long long at = atomicAdd(tab.counters + 1, 1ULL); tab.deferred[at] = row; st = LH_IDLE; }
      else { idx = (unsigned)si; st = LH_HIT; }
    }
    const unsigned b = __ballot_sync(0xffffffffu, inserted);
    if (lane == 0 && b) atomicAdd(tab.counters, (unsigned long long)__popc(b));
  }
  // accumulate (REDs unconditional: idle lanes add 0 to the warp's sink sector); accumulator entries are only ever RED.
  // A NULL argument arrives as the value 0 and only skips the "has a value" mark.
  const bool odd = lane & 1;
  const int as = lay.astride, w0 = fs.acc[0].word, w1 = NACC == 2 ? fs.acc[1].word : 0;
  const unsigned mi = st == LH_HIT ? idx : NONE;
  unsigned long long* const mine = mi != NONE ? tab.accs + (uint64_t)mi * as + w0 : sink;
  const unsigned long long mv = mi != NONE ? v0 : 0ULL;
  if (NACC == 1) red_add_u64(mine, mv);
  else {
    const unsigned pi = __shfl_xor_sync(0xffffffffu, mi, 1);                                       // neighbour's slot
    const unsigned long long pv1 = has_v1 ? __shfl_xor_sync(0xffffffffu, v1, 1) : 1ULL;
    unsigned long long* const theirs = pi != NONE ? tab.accs + (uint64_t)pi * as + w1 : sink;
    const unsigned long long tv = pi != NONE ? pv1 : 0ULL;
    red_add_u64(odd ? theirs : mine, odd ? tv : mv);            // step 1: rows of even lanes: {acc0 by the owner, acc1 by its odd neighbour}
    red_add_u64(odd ? mine : theirs, odd ? mv : tv);            // step 2: rows of odd lanes
  }
  if (mi != NONE) {
    unsigned long long* ke = tab.keys + (uint64_t)mi * lay.kstride;
    if (!TYPED || (meta & 4u)) slot_mark(ke, flags, fs.acc[0].vbit);
    if (NACC == 2 && (!TYPED || (meta & 8u))) slot_mark(ke, flags, fs.acc[1].vbit);
  }
  const unsigned m = __ballot_sync(0xffffffffu, st == LH_AGAIN);
  if (m) {
    if (st == LH_AGAIN) {
      const int at = count + __popc(m & ((1u << lane) - 1));
      q.k0[at] = k0; if (NK == 2) q.k1[at] = k1; q.v0[at] = v0; q.v1[at] = v1; q.idx[at] = idx; q.tag[at] = tag; q.row[at] = row;
      if (TYPED) q.meta[at] = (uint8_t)meta;
    }
    count += __popc(m);
  }
}

template <int NK, int NACC, bool TYPED>
__device__ __forceinline__ void lh_drain(const FastSpec& fs, const AggLayout& lay, const AggTable& tab, LhQueue<NK, TYPED>& q, int& count, unsigned lane,
                                         unsigned long long* sink, bool has_v1) {
  const int nb = count < 32 ? count : 32;
  __syncwarp();
  count -= nb;
  const bool act = (int)lane < nb; const int e = count + (act ? lane : 0);
  const unsigned long long k0 = q.k0[e], k1 = NK == 2 ? q.k1[e] : 0ULL, v0 = q.v0[e], v1 = q.v1[e];
  unsigned idx = q.idx[e], flags = 0; const unsigned tag = q.tag[e], row = q.row[e], meta = TYPED ? q.meta[e] : LH_META_PLAIN;
  __syncwarp();                                                 // entries are in registers: the stack may be overwritten
  int st = LH_IDLE;
  if (act) st = lh_eval<NK>(tab, lay.kstride, (unsigned)tab.capacity, ld_relaxed_v2u64(tab.keys + (uint64_t)idx * lay.kstride), tag, TYPED ? (meta & 3u) : 0u, k0, k1, idx, flags);
  lh_finish<NK, NACC, TYPED>(fs, lay, tab, q, count, lane, sink, has_v1, st, idx, flags, tag, meta, k0, k1, v0, v1, row);
}

// TYPED = false: non-null 8-byte-aligned int64 columns (plain streaming loads); TYPED = true: any integer width,
// validity bitmaps on keys (NULL is a group of its own: its bit goes into the hash and the header), on accumulator
// arguments (NULL adds nothing) and on filter columns (NULL -> row dropped, cached_exprs_evaluator.rs:518-520)
template <int NK, int NACC, bool TYPED>
__global__ void __launch_bounds__(LH_BLOCK, TYPED ? 4 : 6) agg_lean_hash_kernel(const ColTable cols, const FastSpec fs, const AggLayout lay, const AggTable tab,
                                                                                long long row_begin, long long n) {
  constexpr int U = LH_U;
  __shared__ LhQueue<NK, TYPED> queues[LH_BLOCK / 32];
  LhQueue<NK, TYPED>& q = queues[threadIdx.x >> 5];
  int count = 0;                                                // warp-uniform stack height
  const unsigned lane = threadIdx.x & 31;
  const long long gwarp = (long long)blockIdx.x * (LH_BLOCK / 32) + (threadIdx.x >> 5), nwarps = (long long)gridDim.x * (LH_BLOCK / 32);
  const long long nunits = (n + 31) / 32;
  const bool add0 = fs.acc[0].kind == FAST_ACC_ADD, add1 = NACC == 2 && fs.acc[1].kind == FAST_ACC_ADD;
  const long long* kcol0 = (const long long*)cols.col[fs.key_col[0]].values + row_begin;
  const long long* kcol1 = NK == 2 ? (const long long*)cols.col[fs.key_col[1]].values + row_begin : nullptr;
  const long long* vcol0 = add0 ? (const long long*)cols.col[fs.acc[0].col].values + row_begin : nullptr;
  const long long* vcol1 = add1 ? (const long long*)cols.col[fs.acc[1].col].values + row_begin : nullptr;
  unsigned long long* const sink = warp_sink(fs, gwarp, lane);
  const unsigned cap = (unsigned)tab.capacity; const int ks = lay.kstride;

  for (long long unit0 = gwarp * U; unit0 < nunits; unit0 += nwarps * U) {
    unsigned long long k0[U], k1[U], v0[U], v1[U]; bool alive[U]; unsigned meta[U];
#pragma unroll
    for (int u = 0; u < U; u++) {
      const long long rel = (unit0 + u) * 32 + lane;
      alive[u] = rel < n; meta[u] = LH_META_PLAIN;
      if (!TYPED) {
        k0[u] = alive[u] ? (unsigned long long)ld_stream_vec(kcol0 + rel, (i64xG<1>*)nullptr).v[0] : 0;
        k1[u] = (NK == 2 && alive[u]) ? (unsigned long long)ld_stream_vec(kcol1 + rel, (i64xG<1>*)nullptr).v[0] : 0;
        v0[u] = (vcol0 && alive[u]) ? (unsigned long long)ld_stream_vec(vcol0 + rel, (i64xG<1>*)nullptr).v[0] : 1ULL;
        v1[u] = (vcol1 && alive[u]) ? (unsigned long long)ld_stream_vec(vcol1 + rel, (i64xG<1>*)nullptr).v[0] : 1ULL;
      } else {
        k0[u] = 0; k1[u] = 0; v0[u] = 1; v1[u] = 1;
        if (alive[u]) {
          const long long row = row_begin + rel;
          { const DevCol& c = cols.col[fs.key_col[0]]; if (col_valid(c, row)) k0[u] = (unsigned long long)col_load_int(c, fs.key_phys[0], row); else meta[u] |= 1u; }
          if (NK == 2) { const DevCol& c = cols.col[fs.key_col[1]]; if (col_valid(c, row)) k1[u] = (unsigned long long)col_load_int(c, fs.key_phys[1], row); else meta[u] |= 2u; }
          if (fs.acc[0].col >= 0) {
            const DevCol& c = cols.col[fs.acc[0].col];
            if (!col_valid(c, row)) { meta[u] &= ~4u; v0[u] = 0; } else if (add0) v0[u] = (unsigned long long)col_load_int(c, fs.acc[0].phys, row);
          }
          if (NACC == 2 && fs.acc[1].col >= 0) {
            const DevCol& c = cols.col[fs.acc[1].col];
            if (!col_valid(c, row)) { meta[u] &= ~8u; v1[u] = 0; } else if (add1) v1[u] = (unsigned long long)col_load_int(c, fs.acc[1].phys, row);
          }
        }
      }
    }
    for (int f = 0; f < fs.nfilt; f++) {                        // fused FilterExec conjuncts
      if (!TYPED) {
        const long long* fcol = (const long long*)cols.col[fs.filt[f].col].values + row_begin;
#pragma unroll
        for (int u = 0; u < U; u++) {
          const long long rel = (unit0 + u) * 32 + lane;
          const long long x = rel < n ? ld_stream_vec(fcol + rel, (i64xG<1>*)nullptr).v[0] : 0;
          alive[u] = alive[u] && cmp_apply(fs.filt[f].op, x, fs.filt[f].lit);
        }
      } else {
        const DevCol& c = cols.col[fs.filt[f].col];
#pragma unroll
        for (int u = 0; u < U; u++) {
          const long long row = row_begin + (unit0 + u) * 32 + lane;
          if (alive[u]) alive[u] = col_valid(c, row) && cmp_apply(fs.filt[f].op, col_load_int(c, fs.filt[f].phys, row), fs.filt[f].lit);
        }
      }
    }
    unsigned idx[U], tag[U]; ulonglong2 hk[U];
#pragma unroll
    for (int u = 0; u < U; u++) {                               // first probes: U independent 16-byte loads in flight per lane
      const uint64_t h = agg_hash2(k0[u], NK == 2 ? k1[u] : 0ULL, TYPED ? (meta[u] & 3u) : 0u);
      idx[u] = __umulhi((unsigned)(h >> 32), cap); tag[u] = agg_tag(h);
      if (alive[u]) hk[u] = ld_relaxed_v2u64(tab.keys + (uint64_t)idx[u] * ks);                   // {hdr, key0}
    }
#pragma unroll
    for (int u = 0; u < U; u++) {
      unsigned flags = 0;
      const int st = alive[u] ? lh_eval<NK>(tab, ks, cap, hk[u], tag[u], TYPED ? (meta[u] & 3u) : 0u, k0[u], k1[u], idx[u], flags) : LH_IDLE;
      lh_finish<NK, NACC, TYPED>(fs, lay, tab, q, count, lane, sink, TYPED ? NACC == 2 : vcol1 != nullptr, st, idx[u], flags, tag[u], meta[u], k0[u], k1[u], v0[u], v1[u],
                                 (unsigned)((unit0 + u) * 32 + lane));
    }
    while (count >= 32) lh_drain<NK, NACC, TYPED>(fs, lay, tab, q, count, lane, sink, TYPED ? NACC == 2 : vcol1 != nullptr);
  }
  while (count > 0) lh_drain<NK, NACC, TYPED>(fs, lay, tab, q, count, lane, sink, TYPED ? NACC == 2 : vcol1 != nullptr);
}

// ---------------------------------------------------------------------------------------------------
// SMALL dense tables (<= 4096 words, i.e. a few hundred to 2048 groups): CTA-private copy in shared memory.
// With few groups every RED of a warp lands on a handful of L2 sectors and the L2 serialises them: 64 groups ran
// at 4.6e9 rows/s through the global-table kernel.  Here each CTA accumulates into its own shared-memory table with
// native 32-bit shared atomics (a 64-bit wrapping add = low-half add returning the old value + high-half add of
// the carry: exact mod 2^64 in any order) and adds its non-zero words to the global dense table once, at the end.
// TYPED = false: non-null int64 columns; TYPED = true: any integer width + validity bitmaps (NULL key -> hashed slot).
// ---------------------------------------------------------------------------------------------------
constexpr int DS_MAX_WORDS = 4096;
template <int NACC, bool TYPED, int NK>
__global__ void __launch_bounds__(FA_BLOCK) agg_dense_smem_kernel(const ColTable cols, const FastSpec fs, const AggLayout lay, const AggTable tab,
                                                                  long long row_begin, long long n) {
  constexpr int U = 4;
  __shared__ unsigned s_tab[2 * DS_MAX_WORDS];
  const int G = fs.dense_stride;
  const unsigned nwords = (unsigned)fs.dense_cap * G;
  for (unsigned i = threadIdx.x; i < 2 * nwords; i += FA_BLOCK) s_tab[i] = 0;
  __syncthreads();
  const unsigned lane = threadIdx.x & 31;
  const long long gwarp = (long long)blockIdx.x * (FA_BLOCK / 32) + (threadIdx.x >> 5), nwarps = (long long)gridDim.x * (FA_BLOCK / 32);
  const long long nunits = (n + 31) / 32;
  const bool add0 = fs.acc[0].kind == FAST_ACC_ADD, add1 = NACC == 2 && fs.acc[1].kind == FAST_ACC_ADD;

  for (long long unit0 = gwarp * U; unit0 < nunits; unit0 += nwarps * U) {
    long long k[U], k1[U]; unsigned long long v0[U], v1[U]; bool alive[U]; unsigned meta[U];       // meta: bit0/1 key NULL, bit2/3 argument valid
#pragma unroll
    for (int u = 0; u < U; u++) {
      const long long rel = (unit0 + u) * 32 + lane, row = row_begin + rel;
      alive[u] = rel < n; meta[u] = 0xC; k[u] = 0; k1[u] = 0; v0[u] = 1; v1[u] = 1;
      if (!alive[u]) continue;
      if (!TYPED) {
        k[u] = ld_stream_vec((const long long*)cols.col[fs.key_col[0]].values + row, (i64xG<1>*)nullptr).v[0];
        if (NK == 2) k1[u] = ld_stream_vec((const long long*)cols.col[fs.key_col[1]].values + row, (i64xG<1>*)nullptr).v[0];
        if (add0) v0[u] = (unsigned long long)ld_stream_vec((const long long*)cols.col[fs.acc[0].col].values + row, (i64xG<1>*)nullptr).v[0];
        if (add1) v1[u] = (unsigned long long)ld_stream_vec((const long long*)cols.col[fs.acc[1].col].values + row, (i64xG<1>*)nullptr).v[0];
      } else {
        { const DevCol& c = cols.col[fs.key_col[0]]; if (col_valid(c, row)) k[u] = col_load_int(c, fs.key_phys[0], row); else meta[u] |= 1u; }
        if (NK == 2) { const DevCol& c = cols.col[fs.key_col[1]]; if (col_valid(c, row)) k1[u] = col_load_int(c, fs.key_phys[1], row); else meta[u] |= 2u; }
        if (fs.acc[0].col >= 0) {
          const DevCol& c = cols.col[fs.acc[0].col];
          if (!col_valid(c, row)) { meta[u] &= ~4u; v0[u] = 0; } else if (add0) v0[u] = (unsigned long long)col_load_int(c, fs.acc[0].phys, row);
        }
        if (NACC == 2 && fs.acc[1].col >= 0) {
          const DevCol& c = cols.col[fs.acc[1].col];
          if (!col_valid(c, row)) { meta[u] &= ~8u; v1[u] = 0; } else if (add1) v1[u] = (unsigned long long)col_load_int(c, fs.acc[1].phys, row);
        }
      }
    }
    for (int f = 0; f < fs.nfilt; f++) {                        // fused FilterExec conjuncts (NULL -> row dropped)
      const DevCol& c = cols.col[fs.filt[f].col];
#pragma unroll
      for (int u = 0; u < U; u++) {
        const long long row = row_begin + (unit0 + u) * 32 + lane;
        if (!alive[u]) continue;
        if (!TYPED) alive[u] = cmp_apply(fs.filt[f].op, ld_stream_vec((const long long*)c.values + row, (i64xG<1>*)nullptr).v[0], fs.filt[f].lit);
        else alive[u] = col_valid(c, row) && cmp_apply(fs.filt[f].op, col_load_int(c, fs.filt[f].phys, row), fs.filt[f].lit);
      }
    }
#pragma unroll
    for (int u = 0; u < U; u++) {
      unsigned long long idx;
      const bool in = dense_index<NK>(fs, k[u], k1[u], idx) && alive[u] && !(meta[u] & 3u);
      if (in) {
        unsigned* const e = s_tab + 2 * (unsigned)idx * G;
#pragma unroll
        for (int m = 0; m < 4; m++) {
          if (m >= G) break;
          const int src = fs.dense_word_src[m];                 // -1: row counter, -2: padding, j: accumulator j, 2+j: its valid counter
          if (src == -1) smem_add64(e + 2 * m, 1ULL);
          else if (src == 0) { if (meta[u] & 4u) smem_add64(e + 2 * m, v0[u]); }
          else if (src == 1 && NACC == 2) { if (meta[u] & 8u) smem_add64(e + 2 * m, v1[u]); }
          else if (src >= 2) { if (meta[u] & (4u << (src - 2))) smem_add64(e + 2 * m, 1ULL); }     // valid arguments of accumulator src-2
        }
      }
      // keys outside the dense range / NULL keys (rare): straight to the hashed slots
      const bool fb = alive[u] && !in;
      if (__any_sync(0xffffffffu, fb)) {
        bool inserted = false;
        if (fb) {
          uint64_t kw[2] = {(uint64_t)k[u], NK == 2 ? (uint64_t)k1[u] : 0ULL};
          const unsigned knull = meta[u] & 3u;
          unsigned fl = 0;
          const uint64_t si = agg_find_or_insert(lay, tab, kw, knull, agg_hash2(kw[0], kw[1], knull), &fl, &inserted);
          if (si == AGG_NO_SLOT) { const unsigned long long at = atomicAdd(tab.counters + 1, 1ULL); tab.deferred[at] = (uint32_t)((unit0 + u) * 32 + lane); }
          else {
            unsigned long long* const p = tab.accs + si * (uint64_t)lay.astride;
            unsigned long long* const ke = tab.keys + si * (uint64_t)lay.kstride;
            if (meta[u] & 4u) { red_add_u64(p + fs.acc[0].word, v0[u]); slot_mark(ke, fl, fs.acc[0].vbit); }
            if (NACC == 2 && (meta[u] & 8u)) { red_add_u64(p + fs.acc[1].word, v1[u]); slot_mark(ke, fl, fs.acc[1].vbit); }
          }
        }
        const unsigned b = __ballot_sync(0xffffffffu, inserted);
        if (lane == 0 && b) atomicAdd(tab.counters, (unsigned long long)__popc(b));
      }
    }
  }
  __syncthreads();
  for (unsigned w = threadIdx.x; w < nwords; w += FA_BLOCK) {
    const unsigned long long val = (unsigned long long)s_tab[2 * w] | ((unsigned long long)s_tab[2 * w + 1] << 32);
    if (val) red_add_u64(fs.dense_tab + w, val);
  }
}

static int fast_grid(int64_t ntiles) {
  int dev = 0, sms = 132; cudaGetDevice(&dev); cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  const int64_t cap = (int64_t)sms * 8;          // persistent grid: a multiple of the SM count
  return (int)(ntiles < cap ? (ntiles < 1 ? 1 : ntiles) : cap);
}

int launch_agg_fast_update(const ColTable& cols, const FastSpec& fs, const AggLayout& lay, const AggTable& tab, int64_t row_begin, int64_t n, cudaStream_t s) {
  if (n <= 0) return 0;
  const int dg = fs.dense ? fs.dense_stride : 0;
  if (dg && fs.dense_cap * (unsigned long long)dg <= (unsigned long long)DS_MAX_WORDS) {
    // persistent CTAs, 3 per SM (32 KB of shared memory each); every CTA flushes its private table once
    const int g = (int)std::max<int64_t>(1, std::min<int64_t>((n + FA_BLOCK * 4 - 1) / (FA_BLOCK * 4), (int64_t)fast_grid(1 << 30) / 8 * 3));
#define B200Q_DS(NACC, TYPED, NK) agg_dense_smem_kernel<NACC, TYPED, NK><<<g, FA_BLOCK, 0, s>>>(cols, fs, lay, tab, row_begin, n)
    if (fs.nkeys == 1) {
      if (fs.lean) { if (fs.nacc == 2) B200Q_DS(2, false, 1); else B200Q_DS(1, false, 1); } else { if (fs.nacc == 2) B200Q_DS(2, true, 1); else B200Q_DS(1, true, 1); }
    } else {
      if (fs.lean) { if (fs.nacc == 2) B200Q_DS(2, false, 2); else B200Q_DS(1, false, 2); } else { if (fs.nacc == 2) B200Q_DS(2, true, 2); else B200Q_DS(1, true, 2); }
    }
#undef B200Q_DS
    return 1;
  }
  if (dg && fs.lean && fs.hot_cache) {                          // EXPERIMENTAL: skewed keys (b200q_conf.agg_hot_key_cache)
    const int g = fast_grid((n + 32 * 8 * 4 - 1) / (32 * 8 * 4));
#define B200Q_HC(NACC, NK, G) agg_dense_hot_kernel<NACC, NK, G><<<g, FA_BLOCK, 0, s>>>(cols, fs, lay, tab, row_begin, n)
    if (fs.nkeys == 1) {
      if (fs.nacc == 2) { if (dg == 2) B200Q_HC(2, 1, 2); else B200Q_HC(2, 1, 4); } else { if (dg == 2) B200Q_HC(1, 1, 2); else B200Q_HC(1, 1, 4); }
    } else {
      if (fs.nacc == 2) { if (dg == 2) B200Q_HC(2, 2, 2); else B200Q_HC(2, 2, 4); } else { if (dg == 2) B200Q_HC(1, 2, 2); else B200Q_HC(1, 2, 4); }
    }
#undef B200Q_HC
    return 1;
  }
  if (dg && fs.lean && fs.nkeys == 1 && fs.nfilt == 0) {        // the bare M1 shape: gang form, wide loads
    const int u = dg == 2 ? 4 : 2;
    const int g = fast_grid((n + 32 * 8 * u - 1) / (32 * 8 * u));
#define B200Q_LD(NACC, G) agg_lean_dense_kernel<NACC, G, 1><<<g, FA_BLOCK, 0, s>>>(cols, fs, lay, tab, row_begin, n)
    if (fs.nacc == 2) { if (dg == 2) B200Q_LD(2, 2); else B200Q_LD(2, 4); } else { if (dg == 2) B200Q_LD(1, 2); else B200Q_LD(1, 4); }
#undef B200Q_LD
    return 1;
  }
  if (dg && fs.nfcol >= 0) {                                    // filters / two keys / typed inputs: 128-row tiles, filter first (kernels_tile.cu)
    if (fs.filt_never) return 0;
    return launch_agg_tile_dense(cols, fs, lay, tab, row_begin, n, s);
  }
  if (dg) {                                                     // conjuncts that do not merge into intervals: one row per lane
    const int g = fast_grid((n + 32 * 8 * 4 - 1) / (32 * 8 * 4));
#define B200Q_DR(NACC, NK, G) do { if (fs.lean) agg_dense_row_kernel<NACC, NK, G, false><<<g, FA_BLOCK, 0, s>>>(cols, fs, lay, tab, row_begin, n); \
                                   else agg_dense_row_kernel<NACC, NK, G, true><<<g, FA_BLOCK, 0, s>>>(cols, fs, lay, tab, row_begin, n); } while (0)
    if (fs.nkeys == 1) {
      if (fs.nacc == 2) { if (dg == 2) B200Q_DR(2, 1, 2); else B200Q_DR(2, 1, 4); } else { if (dg == 2) B200Q_DR(1, 1, 2); else B200Q_DR(1, 1, 4); }
    } else {
      if (fs.nacc == 2) { if (dg == 2) B200Q_DR(2, 2, 2); else B200Q_DR(2, 2, 4); } else { if (dg == 2) B200Q_DR(1, 2, 2); else B200Q_DR(1, 2, 4); }
    }
#undef B200Q_DR
    return 1;
  }
  if (!dg) {
    const int64_t tiles = (n + 32 * (LH_BLOCK / 32) * LH_U - 1) / (32 * (LH_BLOCK / 32) * LH_U);
    const int g = (int)std::max<int64_t>(1, std::min<int64_t>(tiles, (int64_t)fast_grid(1 << 30) / 8 * (fs.lean ? 6 : 4)));
#define B200Q_LH(NK, NACC, TYPED) agg_lean_hash_kernel<NK, NACC, TYPED><<<g, LH_BLOCK, 0, s>>>(cols, fs, lay, tab, row_begin, n)
    if (fs.lean) { if (fs.nkeys == 1) { if (fs.nacc == 2) B200Q_LH(1, 2, false); else B200Q_LH(1, 1, false); } else { if (fs.nacc == 2) B200Q_LH(2, 2, false); else B200Q_LH(2, 1, false); } }
    else { if (fs.nkeys == 1) { if (fs.nacc == 2) B200Q_LH(1, 2, true); else B200Q_LH(1, 1, true); } else { if (fs.nacc == 2) B200Q_LH(2, 2, true); else B200Q_LH(2, 1, true); } }
#undef B200Q_LH
    return 1;
  }
  return 0;
}

// ---------------------------------------------------------------------------------------------------
// key range of the first batch (decides DENSE mode)
// ---------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) key_range_kernel(const DevCol col, int phys, long long n, long long* out /*[0]=min,[1]=max,[2]=non-null count*/) {
  long long mn = INT64_MAX, mx = INT64_MIN; unsigned long long cnt = 0;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    if (!col_valid(col, i)) continue;
    const long long v = col_load_int(col, phys, i);
    mn = v < mn ? v : mn; mx = v > mx ? v : mx; cnt++;
  }
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) {
    const long long a = __shfl_xor_sync(0xffffffffu, mn, d), b = __shfl_xor_sync(0xffffffffu, mx, d);
    mn = a < mn ? a : mn; mx = b > mx ? b : mx; cnt += __shfl_xor_sync(0xffffffffu, cnt, d);
  }
  // one update of the three result words per CTA, not per warp: same-address atomics serialise in L2
  __shared__ long long s_mn[8], s_mx[8]; __shared__ unsigned long long s_cnt[8];
  const int w = threadIdx.x >> 5;
  if ((threadIdx.x & 31) == 0) { s_mn[w] = mn; s_mx[w] = mx; s_cnt[w] = cnt; }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int j = 1; j < (int)(blockDim.x >> 5); j++) { mn = s_mn[j] < mn ? s_mn[j] : mn; mx = s_mx[j] > mx ? s_mx[j] : mx; cnt += s_cnt[j]; }
    atomicMin(out, mn); atomicMax(out + 1, mx); atomicAdd((unsigned long long*)out + 2, cnt);
  }
}
int launch_key_skew_probe(const DevCol* key_cols, const uint8_t* phys, int nkeys, int64_t n, unsigned* d_hist, cudaStream_t s) {
  key_skew_hist_kernel<<<fast_grid((n + 2047) / 2048), 256, 0, s>>>(key_cols[0], key_cols[nkeys == 2 ? 1 : 0], phys[0], phys[nkeys == 2 ? 1 : 0], nkeys, n, d_hist);
  key_skew_max_kernel<<<32, 256, 0, s>>>(d_hist);
  return 2;
}
int launch_key_range(const DevCol& col, int phys, int64_t n, long long* d_out, cudaStream_t s) {
  key_range_kernel<<<fast_grid((n + 2047) / 2048), 256, 0, s>>>(col, phys, n, d_out);
  return 1;
}

// ---------------------------------------------------------------------------------------------------
// emit of the dense table (same output columns as agg_emit_kernel)
// ---------------------------------------------------------------------------------------------------
__device__ __forceinline__ void dense_store(const EmitCol& c, unsigned long long at, uint64_t lo, bool valid) {
  if (c.valid_bytes) c.valid_bytes[at] = valid ? 1 : 0;
  switch (c.phys) {
    case PH_BOOL: ((uint8_t*)c.values)[at] = lo != 0; break;
    case PH_I8: ((int8_t*)c.values)[at] = (int8_t)lo; break;
    case PH_I16: ((int16_t*)c.values)[at] = (int16_t)lo; break;
    case PH_I32: ((int32_t*)c.values)[at] = (int32_t)lo; break;
    default: ((uint64_t*)c.values)[at] = lo; break;
  }
}
__global__ void __launch_bounds__(256) agg_emit_dense_kernel(const FastSpec fs, const EmitTable emit, const DenseEmitMap map, unsigned long long* out_count) {
  const unsigned lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
  __shared__ unsigned s_warp[8];
  __shared__ unsigned long long s_base;
  const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
  const uint64_t rounds = (fs.dense_cap + stride - 1) / stride;
  const uint32_t r1 = (uint32_t)fs.dense_r1;                   // dense_cap <= 2^26 entries: key order indices fit 32 bits
  for (uint64_t it = 0; it < rounds; it++) {
    const uint32_t i = (uint32_t)(it * stride + blockIdx.x * (uint64_t)blockDim.x + threadIdx.x);   // key order: (key0 - dense_base) * dense_r1 + (key1 - dense_base1)
    const uint32_t q = fs.nkeys == 2 ? i / r1 : i, r = fs.nkeys == 2 ? i - q * r1 : 0;
    const uint64_t pe = fs.nkeys == 2 && fs.dense_key0_minor ? dense_entry2(fs, q, r) : i;
    const unsigned long long* e = fs.dense_tab + pe * fs.dense_stride;
    const bool occ = i < fs.dense_cap && e[fs.dense_presence_word] != 0;
    const unsigned m = __ballot_sync(0xffffffffu, occ);
    // one output reservation per CTA and round (a per-warp atomicAdd on the one counter serialises in L2); the warps of a CTA
    // take consecutive runs, so the rows stay in key order within the CTA's round as they were within a warp
    if (lane == 0) s_warp[warp] = __popc(m);
    __syncthreads();
    if (threadIdx.x == 0) {
      unsigned tot = 0;
      for (unsigned j = 0; j < nwarps; j++) { const unsigned c = s_warp[j]; s_warp[j] = tot; tot += c; }
      s_base = tot ? atomicAdd(out_count, (unsigned long long)tot) : 0;
    }
    __syncthreads();
    const unsigned long long base = s_base + s_warp[warp];
    __syncthreads();                                            // s_warp / s_base are rewritten in the next round
    if (!occ) continue;
    const unsigned long long at = base + __popc(m & lanemask_lt());
    for (int c = 0; c < emit.ncols; c++) {
      const EmitCol ec = emit.col[c];
      if (ec.kind == EMIT_KEY) {
        const long long kv = fs.nkeys == 1 ? fs.dense_base + (long long)i
                           : ec.key == 0 ? fs.dense_base + (long long)q : fs.dense_base1 + (long long)r;
        dense_store(ec, at, (uint64_t)kv, true);
      }
      else {
        const int w = map.word[c], vw = map.valid_word[c];
        const bool valid = vw == 0xFF ? true : e[vw] != 0;
        dense_store(ec, at, valid ? e[w] : 0, valid);
      }
    }
  }
}
int launch_agg_emit_dense(const FastSpec& fs, const EmitTable& emit, const DenseEmitMap& map, unsigned long long* d_out_count, cudaStream_t s) {
  agg_emit_dense_kernel<<<fast_grid(((int64_t)fs.dense_cap + 255) / 256), 256, 0, s>>>(fs, emit, map, d_out_count);
  return 1;
}

// number of occupied dense entries
__global__ void __launch_bounds__(256) dense_count_kernel(const FastSpec fs, unsigned long long* out) {
  unsigned long long c = 0;
  for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < fs.dense_cap; i += (uint64_t)gridDim.x * blockDim.x)
    c += fs.dense_tab[i * fs.dense_stride + fs.dense_presence_word] != 0;
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) c += __shfl_xor_sync(0xffffffffu, c, d);
  if ((threadIdx.x & 31) == 0 && c) atomicAdd(out, c);
}
int launch_dense_count(const FastSpec& fs, unsigned long long* d_out, cudaStream_t s) {
  dense_count_kernel<<<fast_grid(((int64_t)fs.dense_cap + 255) / 256), 256, 0, s>>>(fs, d_out);
  return 1;
}

}  // namespace b200q
