// Hand-written sm_90a kernels of the Filter / Project / HashAgg hot path (generic, VM-driven forms;
// the specialised streaming kernels live in kernels_fast.cu).
//
//   filter_project_kernel  K1+K2+K3 of SURVEY.md §2.4 fused: predicate mask, ordered stream compaction
//                          (single pass, decoupled look-back) and projection — filtered rows never
//                          round-trip through HBM.  Replaces CachedExprsEvaluator::filter_project
//                          (cached_exprs_evaluator.rs:82-166).
//   agg_update_kernel      K4+K5+K6(+K7): key evaluation, open-addressing upsert and accumulator update
//                          in one pass.  Replaces HashingData::update_batch (agg_table.rs:519-538):
//                          create_grouping_rows + AggHashMap::upsert_records + partial_update/partial_merge.
//   agg_emit_kernel        K8+K9: table scan -> dense Arrow columns (build_agg_columns, agg_ctx.rs:303-326).
//   frozen_* kernels       the reference's frozen accumulator-row byte format (acc.rs:335-365,
//                          count.rs:193-211, io/mod.rs:60-83) for the Binary `#9223372036854775807` column.
#include <cstdio>
#include <cstdlib>
#include <cuda_runtime.h>
#include <stdint.h>

#include "agg_device.cuh"
#include "kernels.cuh"
#include "vm.cuh"
#include "emit_device.cuh"

namespace b200q {

// ---------------------------------------------------------------------------------------------------
// small device helpers (atomics, hash, find-or-insert: agg_device.cuh)
// ---------------------------------------------------------------------------------------------------
__device__ __forceinline__ void load_program(const VmProgram* __restrict__ g, VmInstr* s_code, uint64_t* s_pool) {
  const uint32_t nc = g->n_code, np = g->n_pool;
  for (uint32_t i = threadIdx.x; i < nc; i += blockDim.x) s_code[i] = g->code[i];
  for (uint32_t i = threadIdx.x; i < np; i += blockDim.x) s_pool[i] = g->pool[i];
  __syncthreads();
}

// ---------------------------------------------------------------------------------------------------
// FilterExec / ProjectExec
// ---------------------------------------------------------------------------------------------------
constexpr int FP_BLOCK = 256;
constexpr int FP_R = 2;
constexpr int FP_TILE = FP_BLOCK * FP_R;
constexpr int FP_NW = FP_BLOCK / 32;
constexpr unsigned long long ST_AGG = 1ULL << 62, ST_PREFIX = 2ULL << 62, ST_VALUE = (1ULL << 62) - 1;

int64_t filter_project_num_tiles(int64_t n) { return (n + FP_TILE - 1) / FP_TILE; }

struct FpSink {
  const OutTable& outs;
  long long wbase[FP_R];     // output position of the first surviving row of this warp-row
  unsigned amask[FP_R];      // ballot of surviving lanes
  bool* alive;
  unsigned lt;

  __device__ __forceinline__ void put_bits(uint32_t* bitmap, int r, bool bit) const {
    // compact this warp-row's bits by the survivor mask and OR them into the pre-zeroed bitmap
    const unsigned m = amask[r];
    const unsigned rank = __popc(m & lt);
    const unsigned w = __reduce_or_sync(0xffffffffu, (alive[r] && bit) ? (1u << rank) : 0u);
    if ((threadIdx.x & 31) == 0 && m) {
      const unsigned cnt = __popc(m);
      const unsigned long long p = (unsigned long long)wbase[r];
      const unsigned sh = (unsigned)(p & 31);
      if (w << sh) atomicOr(bitmap + (p >> 5), w << sh);
      if (sh + cnt > 32 && (w >> (32 - sh))) atomicOr(bitmap + (p >> 5) + 1, w >> (32 - sh));
    }
  }

  __device__ __forceinline__ void out(int r, int idx, int phys, uint64_t lo, uint64_t hi, bool valid) const {
    if (outs.validity[idx]) put_bits(outs.validity[idx], r, valid);
    if (phys == PH_BOOL) { put_bits((uint32_t*)outs.values[idx], r, lo != 0); return; }
    if (!alive[r]) return;
    const long long p = wbase[r] + __popc(amask[r] & lt);
    void* v = outs.values[idx];
    switch (phys) {
      case PH_I8: ((int8_t*)v)[p] = (int8_t)lo; break;
      case PH_I16: ((int16_t*)v)[p] = (int16_t)lo; break;
      case PH_I32: ((int32_t*)v)[p] = (int32_t)lo; break;
      case PH_I64: case PH_F64: ((uint64_t*)v)[p] = lo; break;
      case PH_F32: ((float*)v)[p] = (float)as_f64(lo); break;
      case PH_SEL: ((uint32_t*)v)[p] = (uint32_t)lo; break;
      default: ((uint64_t*)v)[2 * p] = lo; ((uint64_t*)v)[2 * p + 1] = hi; break;
    }
  }
};

__global__ void __launch_bounds__(FP_BLOCK) filter_project_kernel(const VmProgram* __restrict__ prog, const ColTable cols, const OutTable outs,
                                                                  long long n, long long ntiles, int has_filters,
                                                                  unsigned long long* tile_status, unsigned long long* scratch) {
  __shared__ VmInstr s_code[VM_MAX_CODE];
  __shared__ uint64_t s_pool[VM_MAX_POOL];
  __shared__ long long s_tile, s_excl;
  __shared__ unsigned s_cnt[FP_R * FP_NW], s_off[FP_R * FP_NW];
  load_program(prog, s_code, s_pool);
  const unsigned lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int* err = (int*)(scratch + 2);

  while (true) {
    if (threadIdx.x == 0) s_tile = (long long)atomicAdd(scratch + 0, 1ULL);   // ticket: lower tiles are always already running
    __syncthreads();
    const long long tile = s_tile;
    if (tile >= ntiles) break;
    long long row[FP_R]; bool inb[FP_R], alive[FP_R];
#pragma unroll
    for (int r = 0; r < FP_R; r++) { row[r] = tile * FP_TILE + r * FP_BLOCK + threadIdx.x; inb[r] = row[r] < n; alive[r] = inb[r]; }

    FpSink sink{outs, {}, {}, alive, lanemask_lt()};
    int pc = 0;
    if (has_filters) {
      NullSink ns;
      pc = vm_run<FP_R>(s_code, s_pool, 0, cols, row, inb, alive, err, ns);     // stops after VM_COMPACT
#pragma unroll
      for (int r = 0; r < FP_R; r++) { sink.amask[r] = __ballot_sync(0xffffffffu, alive[r]); if (lane == 0) s_cnt[r * FP_NW + warp] = __popc(sink.amask[r]); }
      __syncthreads();
      if (warp == 0) {
        unsigned v = lane < FP_R * FP_NW ? s_cnt[lane] : 0, incl = v;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) { unsigned t = __shfl_up_sync(0xffffffffu, incl, d); if (lane >= d) incl += t; }
        if (lane < FP_R * FP_NW) s_off[lane] = incl - v;
        const unsigned long long total = __shfl_sync(0xffffffffu, incl, 31);
        // decoupled look-back over the tile status words
        unsigned long long excl = 0;
        if (tile > 0) {
          if (lane == 0) st_relaxed_u64(tile_status + tile, ST_AGG | total);
          long long j = tile - 1;
          while (true) {
            const long long idx = j - lane;
            unsigned long long s = idx >= 0 ? ld_relaxed_u64(tile_status + idx) : ST_PREFIX;
            if (__any_sync(0xffffffffu, (s >> 62) == 0)) continue;                 // a predecessor has not published yet
            const unsigned pm = __ballot_sync(0xffffffffu, (s >> 62) == 2);
            unsigned long long val = s & ST_VALUE;
            if (pm) {
              const int first = __ffs(pm) - 1;                                     // nearest tile with an inclusive prefix
              if ((int)lane > first) val = 0;
            }
#pragma unroll
            for (int d = 16; d > 0; d >>= 1) val += __shfl_xor_sync(0xffffffffu, val, d);
            excl += val;
            if (pm) break;
            j -= 32;
          }
        }
        if (lane == 0) {
          st_relaxed_u64(tile_status + tile, ST_PREFIX | (excl + total));
          s_excl = (long long)excl;
          if (tile == ntiles - 1) scratch[1] = excl + total;
        }
      }
      __syncthreads();
#pragma unroll
      for (int r = 0; r < FP_R; r++) sink.wbase[r] = s_excl + s_off[r * FP_NW + warp];
    } else {
#pragma unroll
      for (int r = 0; r < FP_R; r++) { sink.amask[r] = __ballot_sync(0xffffffffu, alive[r]); sink.wbase[r] = tile * FP_TILE + r * FP_BLOCK + warp * 32; }
      if (tile == ntiles - 1 && threadIdx.x == 0) scratch[1] = (unsigned long long)n;
    }
    vm_run<FP_R>(s_code, s_pool, pc, cols, row, inb, alive, err, sink);
    __syncthreads();
  }
}

int launch_filter_project(const VmProgram* d_prog, const ColTable& cols, const OutTable& outs, int nouts, int64_t n, bool has_filters,
                          unsigned long long* d_tile_status, unsigned long long* d_scratch, cudaStream_t s) {
  (void)nouts;
  const int64_t ntiles = filter_project_num_tiles(n);
  if (ntiles == 0) return 0;
  int dev = 0, sms = 132; cudaGetDevice(&dev); cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  const int64_t grid = ntiles < (int64_t)sms * 8 ? ntiles : (int64_t)sms * 8;     // persistent: a multiple of the SM count
  filter_project_kernel<<<(unsigned)grid, FP_BLOCK, 0, s>>>(d_prog, cols, outs, n, ntiles, has_filters ? 1 : 0, d_tile_status, d_scratch);
  return 1;
}

static int grid_for(int64_t ntiles, int per_sm);

// ---------------------------------------------------------------------------------------------------
// lean FilterExec / ProjectExec for the M0 shape: 1-4 non-null int64 input columns, `col cmp literal` conjuncts,
// projections that are a column or `column op column|literal`; expressions evaluated directly (no bytecode).
//
// In the single-pass look-back form a tile spends most of its life WAITING for its exclusive prefix with its rows
// parked in registers and no loads in flight; wider windows, larger tiles, back-off and earlier tickets do not
// change that.  Large batches therefore take an order-free two-pass form:
//   pass 1  count : every warp streams the FILTER columns of its 256-row chunks and writes one survivor count
//   (scan)        : exclusive scan of the chunk counts (3 tiny launches)
//   pass 2  apply : every warp streams all referenced columns of its chunks, re-evaluates the conjuncts and
//                   writes the projected survivors at the chunk's offset (warps are fully independent: no
//                   barriers, no spinning, 2 x NC x 8 independent loads per lane in flight)
// The filter columns are read twice (M0: 32 B/row of traffic for 24 algorithmic bytes) but both passes stream
// at HBM speed.  Small batches (latency-bound anyway) keep the single-pass kernel: one launch.
// ---------------------------------------------------------------------------------------------------
constexpr int FL_R = 8;                          // rows per lane per chunk
constexpr int FL_CHUNK = 32 * FL_R;              // 256 rows: the unit of the order-free form
constexpr int FL_BLOCK = 256;                    // single-pass form: 8 chunks per tile
constexpr int FL_NW = FL_BLOCK / 32;
constexpr int FL_TILE = FL_BLOCK * FL_R;
constexpr int64_t FL_TWO_PASS_MIN_ROWS = 1 << 20;
struct LeanFpDev {
  int32_t nfilt, nout, nfcols;
  const long long* col[4];
  uint8_t fcol[4];                                                       // distinct columns the conjuncts read
  struct { uint8_t slot, mask; long long lit; } filt[4];                 // mask: bit0 '<', bit1 '==', bit2 '>'
  struct { uint8_t kind, a, b; long long lit; long long* dst; } out[8];  // b == 0xFF: literal operand
};
static int64_t fl_num_chunks(int64_t n) { return (n + FL_CHUNK - 1) / FL_CHUNK; }
int64_t filter_project_lean_scratch_bytes(int64_t n) {
  const int64_t nc = fl_num_chunks(n);
  if (n >= FL_TWO_PASS_MIN_ROWS) return (nc + (nc + 1) + scan_num_blocks(nc) + 8) * 4;     // counts, offsets, block sums
  return ((n + FL_TILE - 1) / FL_TILE) * 8;                                               // tile status words
}

__device__ __forceinline__ long long ld_stream_i64(const long long* p) {
  long long v; asm volatile("ld.global.nc.L1::no_allocate.b64 %0, [%1];" : "=l"(v) : "l"(p)); return v;
}
__device__ __forceinline__ bool fl_cmp(unsigned mask, long long x, long long lit) { return mask & (x < lit ? 1u : (x == lit ? 2u : 4u)); }

// one chunk: 8 x 8-byte streaming loads per lane and column (row = row0 + r*32: 256 contiguous bytes per warp instruction)
template <int NCOLS>
__device__ __forceinline__ void fl_load(const LeanFpDev& sp, const uint8_t* slots, long long row0, long long n, long long (&x)[NCOLS][FL_R]) {
  if (row0 - (threadIdx.x & 31) + FL_CHUNK <= n) {
#pragma unroll
    for (int c = 0; c < NCOLS; c++)
#pragma unroll
      for (int r = 0; r < FL_R; r++) x[c][r] = ld_stream_i64(sp.col[slots ? slots[c] : c] + row0 + r * 32);
  } else {
#pragma unroll
    for (int c = 0; c < NCOLS; c++)
#pragma unroll
      for (int r = 0; r < FL_R; r++) x[c][r] = row0 + r * 32 < n ? ld_stream_i64(sp.col[slots ? slots[c] : c] + row0 + r * 32) : 0;
  }
}
// survivors of a chunk as one ballot per warp-row; `slots` maps register column -> input slot (null: identity)
template <int NCOLS>
__device__ __forceinline__ unsigned fl_filter(const LeanFpDev& sp, const uint8_t* slots, long long row0, long long n, const long long (&x)[NCOLS][FL_R], unsigned (&am)[FL_R]) {
  bool alive[FL_R];
#pragma unroll
  for (int r = 0; r < FL_R; r++) alive[r] = row0 + r * 32 < n;
  for (int f = 0; f < sp.nfilt; f++) {
    const unsigned mask = sp.filt[f].mask; const long long lit = sp.filt[f].lit; const int slot = sp.filt[f].slot;
#pragma unroll
    for (int c = 0; c < NCOLS; c++) {
      if (slot != (slots ? slots[c] : c)) continue;
#pragma unroll
      for (int r = 0; r < FL_R; r++) alive[r] = alive[r] && fl_cmp(mask, x[c][r], lit);
    }
  }
  unsigned total = 0;
#pragma unroll
  for (int r = 0; r < FL_R; r++) { am[r] = __ballot_sync(0xffffffffu, alive[r]); total += __popc(am[r]); }
  return total;
}
// projected survivors of a chunk -> consecutive positions from `wbase`
template <int NC>
__device__ __forceinline__ void fl_store(const LeanFpDev& sp, const long long (&x)[NC][FL_R], const unsigned (&am)[FL_R], long long wbase) {
  const unsigned lane = threadIdx.x & 31, lt = lanemask_lt();
  for (int o = 0; o < sp.nout; o++) {
    const int kind = sp.out[o].kind, sa = sp.out[o].a, sb = sp.out[o].b;
    long long* const dst = sp.out[o].dst + wbase;
    unsigned rank = 0;
#pragma unroll
    for (int r = 0; r < FL_R; r++) {
      long long va = x[0][r], vb = sp.out[o].lit;
#pragma unroll
      for (int c = 1; c < NC; c++) va = sa == c ? x[c][r] : va;
#pragma unroll
      for (int c = 0; c < NC; c++) vb = sb == c ? x[c][r] : vb;
      const unsigned long long a = (unsigned long long)va, b = (unsigned long long)vb;
      const unsigned long long v = kind == 0 ? a : kind == 1 ? a + b : kind == 2 ? a - b : a * b;     // wrapping, like the reference
      if ((am[r] >> lane) & 1) dst[rank + __popc(am[r] & lt)] = (long long)v;
      rank += __popc(am[r]);
    }
  }
}

// ---- order-free two-pass form ----
template <int NFC>
__global__ void __launch_bounds__(256) filter_count_lean_kernel(const LeanFpDev sp, long long n, long long nchunks, int32_t* __restrict__ counts) {
  const long long gwarp = (long long)blockIdx.x * 8 + (threadIdx.x >> 5), nwarps = (long long)gridDim.x * 8;
  const unsigned lane = threadIdx.x & 31;
  for (long long ch = gwarp; ch < nchunks; ch += nwarps) {
    const long long row0 = ch * FL_CHUNK + lane;
    long long x[NFC][FL_R]; unsigned am[FL_R];
    fl_load<NFC>(sp, sp.fcol, row0, n, x);
    const unsigned total = fl_filter<NFC>(sp, sp.fcol, row0, n, x, am);
    if (lane == 0) counts[ch] = (int32_t)total;
  }
}
template <int NC>
__global__ void __launch_bounds__(256) filter_apply_lean_kernel(const LeanFpDev sp, long long n, long long nchunks, const int32_t* __restrict__ offsets,
                                                                 unsigned long long* scratch) {
  const long long gwarp = (long long)blockIdx.x * 8 + (threadIdx.x >> 5), nwarps = (long long)gridDim.x * 8;
  const unsigned lane = threadIdx.x & 31;
  for (long long ch = gwarp; ch < nchunks; ch += nwarps) {
    const long long row0 = ch * FL_CHUNK + lane;
    const long long wbase = offsets[ch];
    long long x[NC][FL_R]; unsigned am[FL_R];
    fl_load<NC>(sp, nullptr, row0, n, x);
    const unsigned total = fl_filter<NC>(sp, nullptr, row0, n, x, am);
    fl_store<NC>(sp, x, am, wbase);
    if (ch == nchunks - 1 && lane == 0) scratch[1] = (unsigned long long)(wbase + total);
  }
}

// ---- single-pass form (decoupled look-back over 2048-row tiles, ticketed) ----
template <int NC, int OCC>
__global__ void __launch_bounds__(FL_BLOCK, OCC) filter_project_lean_kernel(const LeanFpDev sp, long long n, long long ntiles,
                                                                            unsigned long long* tile_status, unsigned long long* scratch) {
  __shared__ long long s_tile, s_base[FL_NW];
  __shared__ unsigned s_cnt[FL_NW];
  const unsigned lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  while (true) {
    // ticket: lower tiles are always already running (deadlock-free whatever the residency of the grid is).  Taken as
    // late as possible: a ticket held by a CTA that has not published its aggregate yet stalls every later tile
    if (threadIdx.x == 0) s_tile = (long long)atomicAdd(scratch + 0, 1ULL);
    __syncthreads();
    const long long tile = s_tile;
    if (tile >= ntiles) break;
    const long long row0 = tile * FL_TILE + warp * FL_CHUNK + lane;
    long long x[NC][FL_R]; unsigned am[FL_R];
    fl_load<NC>(sp, nullptr, row0, n, x);
    const unsigned wt = fl_filter<NC>(sp, nullptr, row0, n, x, am);
    if (lane == 0) s_cnt[warp] = wt;
    __syncthreads();
    if (warp == 0) {
      const unsigned v = lane < FL_NW ? s_cnt[lane] : 0;
      unsigned incl = v;
#pragma unroll
      for (int d = 1; d < FL_NW; d <<= 1) { unsigned t = __shfl_up_sync(0xffffffffu, incl, d); if (lane >= d) incl += t; }
      const unsigned long long total = __shfl_sync(0xffffffffu, incl, FL_NW - 1);
      unsigned long long excl = 0;
      if (sp.nfilt == 0) excl = (unsigned long long)tile * FL_TILE;        // nothing filtered: positions are the row numbers
      else if (tile > 0) {
        if (lane == 0) st_relaxed_u64(tile_status + tile, ST_AGG | total);
        long long j = tile - 1;
        while (true) {                                                     // decoupled look-back, 32 predecessors per round
          const long long idx = j - lane;
          unsigned long long st = idx >= 0 ? ld_relaxed_u64(tile_status + idx) : ST_PREFIX;
          if (__any_sync(0xffffffffu, (st >> 62) == 0)) { __nanosleep(64); continue; }   // a predecessor has not published yet
          const unsigned pm = __ballot_sync(0xffffffffu, (st >> 62) == 2);
          unsigned long long val = st & ST_VALUE;
          if (pm) { const int first = __ffs(pm) - 1; if ((int)lane > first) val = 0; }   // nearest tile with an inclusive prefix
#pragma unroll
          for (int d = 16; d > 0; d >>= 1) val += __shfl_xor_sync(0xffffffffu, val, d);
          excl += val;
          if (pm) break;
          j -= 32;
        }
      }
      if (lane == 0) {
        if (sp.nfilt) st_relaxed_u64(tile_status + tile, ST_PREFIX | (excl + total));
        if (tile == ntiles - 1) scratch[1] = excl + total;
      }
      if (lane < FL_NW) s_base[lane] = (long long)(excl + (incl - v));
    }
    __syncthreads();
    fl_store<NC>(sp, x, am, s_base[warp]);
  }
}

int launch_filter_project_lean(const ColTable& cols, int ncols, const LeanFpSpec& sp, long long* const* out_values, int64_t n,
                               void* d_work /* filter_project_lean_scratch_bytes(n), zeroed */, unsigned long long* d_scratch, cudaStream_t s) {
  if (n <= 0) return 0;
  static const uint8_t cmp_mask[6] = {2, 5, 1, 3, 4, 6};                   // CMP_EQ, NE, LT, LE, GT, GE
  LeanFpDev d{}; d.nfilt = sp.nfilt; d.nout = sp.nout;
  for (int c = 0; c < ncols; c++) d.col[c] = (const long long*)cols.col[c].values;
  for (int f = 0; f < sp.nfilt; f++) {
    d.filt[f].slot = (uint8_t)sp.filt[f].col; d.filt[f].mask = cmp_mask[sp.filt[f].op]; d.filt[f].lit = sp.filt[f].lit;
    bool seen = false;
    for (int i = 0; i < d.nfcols; i++) seen |= d.fcol[i] == d.filt[f].slot;
    if (!seen) d.fcol[d.nfcols++] = d.filt[f].slot;
  }
  for (int o = 0; o < sp.nout; o++) {
    d.out[o].kind = sp.out[o].kind; d.out[o].a = (uint8_t)sp.out[o].a; d.out[o].b = sp.out[o].b < 0 ? 0xFF : (uint8_t)sp.out[o].b;
    d.out[o].lit = sp.out[o].lit; d.out[o].dst = out_values[o];
  }
  if (sp.nfilt && n >= FL_TWO_PASS_MIN_ROWS) {
    const int64_t nch = fl_num_chunks(n);
    int32_t* counts = (int32_t*)d_work; int32_t* offsets = counts + nch; int32_t* sums = offsets + nch + 1;
    const unsigned grid = grid_for((nch + 7) / 8, 8);
    switch (d.nfcols) {
      case 1: filter_count_lean_kernel<1><<<grid, 256, 0, s>>>(d, n, nch, counts); break;
      case 2: filter_count_lean_kernel<2><<<grid, 256, 0, s>>>(d, n, nch, counts); break;
      case 3: filter_count_lean_kernel<3><<<grid, 256, 0, s>>>(d, n, nch, counts); break;
      default: filter_count_lean_kernel<4><<<grid, 256, 0, s>>>(d, n, nch, counts); break;
    }
    const int scan_launches = launch_exclusive_scan_i32(counts, offsets, nch, sums, s);
    const unsigned grid2 = grid_for((nch + 7) / 8, ncols <= 2 ? 6 : 3);
    switch (ncols) {
      case 1: filter_apply_lean_kernel<1><<<grid2, 256, 0, s>>>(d, n, nch, offsets, d_scratch); break;
      case 2: filter_apply_lean_kernel<2><<<grid2, 256, 0, s>>>(d, n, nch, offsets, d_scratch); break;
      case 3: filter_apply_lean_kernel<3><<<grid2, 256, 0, s>>>(d, n, nch, offsets, d_scratch); break;
      default: filter_apply_lean_kernel<4><<<grid2, 256, 0, s>>>(d, n, nch, offsets, d_scratch); break;
    }
    return 2 + scan_launches;
  }
  const int64_t ntiles = (n + FL_TILE - 1) / FL_TILE;
  unsigned long long* status = (unsigned long long*)d_work;
  switch (ncols) {
    case 1: filter_project_lean_kernel<1, 4><<<grid_for(ntiles, 4), FL_BLOCK, 0, s>>>(d, n, ntiles, status, d_scratch); break;
    case 2: filter_project_lean_kernel<2, 4><<<grid_for(ntiles, 4), FL_BLOCK, 0, s>>>(d, n, ntiles, status, d_scratch); break;
    case 3: filter_project_lean_kernel<3, 2><<<grid_for(ntiles, 2), FL_BLOCK, 0, s>>>(d, n, ntiles, status, d_scratch); break;
    default: filter_project_lean_kernel<4, 2><<<grid_for(ntiles, 2), FL_BLOCK, 0, s>>>(d, n, ntiles, status, d_scratch); break;
  }
  return 1;
}

// ---------------------------------------------------------------------------------------------------
// HashAgg: update
// ---------------------------------------------------------------------------------------------------
constexpr int AG_BLOCK = 256;
constexpr int AG_R = 2;
constexpr int AG_TILE = AG_BLOCK * AG_R;

struct AggSink {
  uint64_t (*buf)[AGG_MAX_ROW_WORDS];
  uint32_t* vb;
  const uint8_t* out_word;
  __device__ __forceinline__ void out(int r, int idx, int phys, uint64_t lo, uint64_t hi, bool valid) const {
    const int w = out_word[idx];
    buf[r][w] = lo;
    if (phys == PH_DEC128) buf[r][w + 1] = hi;
    if (valid) vb[r] |= 1u << idx;
  }
};

__device__ __forceinline__ uint64_t hash_keys(const AggLayout& lay, const uint64_t* buf, uint32_t vb, uint32_t& knull, uint64_t* kw) {
  knull = 0;
  int w = 0;
  for (int k = 0; k < lay.nkeys; k++) {
    const int o = lay.key_out[k];
    const bool valid = (vb >> o) & 1;
    if (!valid) knull |= 1u << k;
    for (int i = 0; i < lay.key_nwords[k]; i++) kw[w++] = valid ? buf[lay.out_word[o] + i] : 0;   // NULL keys are canonicalised to 0 + null bit
  }
  return agg_hash_words(kw, w, knull);
}

__device__ __forceinline__ void dec_minmax(unsigned long long* key_entry, unsigned long long* acc_word, i128_t v, bool is_min) {
  unsigned* flags = (unsigned*)key_entry + 1;
  while (atomicOr(flags, FLAG_SLOT_LOCK) & FLAG_SLOT_LOCK) {}
  __threadfence();
  volatile unsigned long long* p = acc_word;
  const i128_t cur = mk128(p[0], p[1]);
  if (is_min ? v < cur : v > cur) { p[0] = lo64(v); p[1] = hi64(v); }
  __threadfence();
  atomicAnd(flags, ~FLAG_SLOT_LOCK);
}

__device__ __forceinline__ void acc_apply(uint8_t kind, unsigned long long* ke, unsigned long long* w, const uint64_t* arg) {
  switch (kind) {
    case ACC_ADD_I64: red_add_u64(w, arg[0]); break;
    case ACC_ADD_F64: red_add_f64(w, as_f64(arg[0])); break;
    case ACC_ADD_DEC: {
      const unsigned long long old = atomicAdd(w, (unsigned long long)arg[0]);
      const unsigned long long carry = (old + arg[0]) < old ? 1ULL : 0ULL;     // exact: every carry is counted once, adds commute
      red_add_u64(w + 1, arg[1] + carry);
      break;
    }
    case ACC_COUNT: red_add_u64(w, 1ULL); break;
    case ACC_MIN_I64: red_min_s64(w, (long long)arg[0]); break;
    case ACC_MAX_I64: red_max_s64(w, (long long)arg[0]); break;
    case ACC_MIN_F64: red_min_s64(w, total_order_key(arg[0])); break;
    case ACC_MAX_F64: red_max_s64(w, total_order_key(arg[0])); break;
    case ACC_MIN_DEC: dec_minmax(ke, w, mk128(arg[0], arg[1]), true); break;
    default: dec_minmax(ke, w, mk128(arg[0], arg[1]), false); break;
  }
}

// FIRST / FIRST_IGNORES_NULL: the row's value replaces the slot's when the row's arrival ordinal is smaller.  The ordinal of
// a slot only ever decreases, so a relaxed load that already shows a smaller one ends the work with no atomic (every row
// that is not its group's earliest so far); otherwise the slot lock of the 128-bit MIN / MAX makes the re-check and the
// writes of ordinal, value words and validity bit one step.  The FIRST accumulators of one aggregate share the ordinal
// word: the earliest row writes each of them in its own lock hold, and `<=` lets it pass the ordinal it wrote itself.
// Returns false when a smaller ordinal was seen (the caller skips the other accumulators on that ordinal word).
__device__ __forceinline__ bool first_apply(unsigned long long* ke, unsigned long long* ae, const AccOp& a, const uint64_t* arg, bool arg_valid, uint64_t ord) {
  if (ld_relaxed_u64(ae + a.oword) < ord) return false;
  unsigned* flags = (unsigned*)ke + 1;
  while (atomicOr(flags, FLAG_SLOT_LOCK) & FLAG_SLOT_LOCK) {}
  __threadfence();
  volatile unsigned long long* p = ae;
  const bool win = ord <= p[a.oword];
  if (win) {
    p[a.oword] = ord;
    p[a.word] = arg[0];
    if (a.nwords == 2) p[a.word + 1] = arg[1];
    if (a.vbit != 0xFF) { if (arg_valid) atomicOr(flags, 1u << a.vbit); else atomicAnd(flags, ~(1u << a.vbit)); }
  }
  __threadfence();
  atomicAnd(flags, ~FLAG_SLOT_LOCK);
  return win;
}

// eligibility of a row for a FIRST accumulator (`o0`: value output, `o1`: flag output or AGG_NO_ARG; validity bits in `vb`)
__device__ __forceinline__ bool first_eligible(const AccOp& a, const AggLayout& lay, const uint64_t* buf, uint32_t vb, int o0, int o1) {
  if (a.kind == ACC_FIRST_VALID) return o0 != AGG_NO_ARG && ((vb >> o0) & 1);                // first_ignores_null.rs: a valid value
  if (o1 == AGG_NO_ARG) return true;                                                        // first.rs update: any row
  return ((vb >> o1) & 1) && buf[lay.out_word[o1]] != 0;                                    // first.rs merge: the state's flag is set
}

// find-or-insert the key, then apply every accumulator update; returns false when the row had to be deferred
__device__ __forceinline__ bool agg_upsert(const AggLayout& lay, const AggTable& tab, const uint64_t* buf, uint32_t vb, uint64_t ord) {
  uint64_t kw[AGG_MAX_KEYS * 2];
  uint32_t knull;
  const uint64_t h = hash_keys(lay, buf, vb, knull, kw);
  unsigned flags;
  bool inserted = false;
  const uint64_t slot = agg_find_or_insert(lay, tab, kw, knull, h, &flags, &inserted);
  if (slot == AGG_NO_SLOT) return false;
  if (inserted) atomicAdd(tab.counters, 1ULL);
  unsigned long long* const ke = tab.keys + slot * (uint64_t)lay.kstride;
  unsigned long long* const ae = tab.accs + slot * (uint64_t)lay.astride;
  // accumulate (K6 / K7)
  int lost = -1;                           // ordinal word on which this row already lost to an earlier row
  for (int j = 0; j < lay.nacc; j++) {
    const AccOp a = lay.acc[j];
    const int o = a.arg_out[0];
    const uint64_t* arg = buf + lay.out_word[o];
    if (acc_is_first(a.kind)) {
      if (a.oword != lost && first_eligible(a, lay, buf, vb, o, a.nargs > 1 ? a.arg_out[1] : AGG_NO_ARG) &&
          !first_apply(ke, ae, a, arg, (vb >> o) & 1, ord)) lost = a.oword;
      continue;
    }
    bool valid = true;
    for (int i = 0; i < a.nargs; i++) valid = valid && ((vb >> a.arg_out[i]) & 1);
    if (!valid) continue;
    acc_apply(a.kind, ke, ae + a.word, arg);
    slot_mark(ke, flags, a.vbit);
  }
  return true;
}

// agg_upsert for one grouping set: constant keys come from the set's descriptor, arguments from the set's VM outputs
__device__ __forceinline__ bool agg_upsert_set(const AggLayout& lay, const AggTable& tab, const uint64_t* buf, uint32_t vb, const AggSetDesc* __restrict__ sd, uint64_t ord) {
  uint64_t kw[AGG_MAX_KEYS * 2];
  uint32_t knull = 0;
  int w = 0;
  for (int k = 0; k < lay.nkeys; k++) {
    const int o = sd->key_out[k];
    if (o == AGG_KEY_CONST) {
      const bool null = (sd->key_null >> k) & 1;
      if (null) knull |= 1u << k;
      for (int i = 0; i < lay.key_nwords[k]; i++, w++) kw[w] = null ? 0 : sd->key_const[w];
    } else {
      const bool valid = (vb >> o) & 1;
      if (!valid) knull |= 1u << k;
      for (int i = 0; i < lay.key_nwords[k]; i++) kw[w++] = valid ? buf[lay.out_word[o] + i] : 0;
    }
  }
  const uint64_t h = agg_hash_words(kw, w, knull);
  unsigned flags;
  bool inserted = false;
  const uint64_t slot = agg_find_or_insert(lay, tab, kw, knull, h, &flags, &inserted);
  if (slot == AGG_NO_SLOT) return false;
  if (inserted) atomicAdd(tab.counters, 1ULL);
  unsigned long long* const ke = tab.keys + slot * (uint64_t)lay.kstride;
  unsigned long long* const ae = tab.accs + slot * (uint64_t)lay.astride;
  const uint32_t skip = sd->acc_skip;
  int lost = -1;
  for (int j = 0; j < lay.nacc; j++) {
    if ((skip >> j) & 1) continue;
    const AccOp a = lay.acc[j];
    if (acc_is_first(a.kind)) {            // a value that is a NULL literal in this set is AGG_NO_ARG: a NULL value
      const int o = sd->acc_arg[j][0];
      const bool ov = o != AGG_NO_ARG && ((vb >> o) & 1);
      if (a.oword != lost && first_eligible(a, lay, buf, vb, o, sd->acc_arg[j][1]) &&
          !first_apply(ke, ae, a, buf + lay.out_word[o == AGG_NO_ARG ? 0 : o], ov, ord)) lost = a.oword;
      continue;
    }
    bool valid = true;
    for (int i = 0; i < 4; i++) { const int o = sd->acc_arg[j][i]; if (o != AGG_NO_ARG) valid = valid && ((vb >> o) & 1); }
    if (!valid) continue;
    const int o = sd->acc_arg[j][0];
    acc_apply(a.kind, ke, ae + a.word, buf + lay.out_word[o == AGG_NO_ARG ? 0 : o]);
    slot_mark(ke, flags, a.vbit);
  }
  return true;
}

__global__ void __launch_bounds__(AG_BLOCK) agg_update_kernel(const VmProgram* __restrict__ prog, const ColTable cols, const AggLayout lay, const AggTable tab,
                                                              long long row_begin, long long n, const uint32_t* __restrict__ row_list,
                                                              unsigned long long ord_base) {
  __shared__ VmInstr s_code[VM_MAX_CODE];
  __shared__ uint64_t s_pool[VM_MAX_POOL];
  load_program(prog, s_code, s_pool);
  int* err = (int*)(tab.counters + 2);
  const long long ntiles = (n + AG_TILE - 1) / AG_TILE;
  for (long long tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    long long row[AG_R]; bool inb[AG_R], alive[AG_R];
    uint32_t rel[AG_R];
#pragma unroll
    for (int r = 0; r < AG_R; r++) {
      const long long i = tile * AG_TILE + r * AG_BLOCK + threadIdx.x;
      inb[r] = i < n; alive[r] = inb[r];
      rel[r] = inb[r] ? (row_list ? row_list[i] : (uint32_t)i) : 0;
      row[r] = row_begin + rel[r];
    }
    uint64_t buf[AG_R][AGG_MAX_ROW_WORDS];
    uint32_t vb[AG_R];
#pragma unroll
    for (int r = 0; r < AG_R; r++) vb[r] = 0;
    AggSink sink{buf, vb, lay.out_word};
    vm_run<AG_R>(s_code, s_pool, 0, cols, row, inb, alive, err, sink);
#pragma unroll
    for (int r = 0; r < AG_R; r++) {
      if (alive[r] && !agg_upsert(lay, tab, buf[r], vb[r], ord_base + (unsigned long long)row[r])) {
        const unsigned long long at = atomicAdd(tab.counters + 1, 1ULL);
        tab.deferred[at] = rel[r];
      }
    }
  }
}

// Expand fused into the aggregate: one VM evaluation per row, then one upsert per grouping set.  A replay list entry is
// row * nsets + set and replays that set only, so sets of the row that already landed are not counted twice.
__global__ void __launch_bounds__(AG_BLOCK) agg_update_sets_kernel(const VmProgram* __restrict__ prog, const ColTable cols, const AggLayout lay, const AggTable tab,
                                                                   long long row_begin, long long n, const uint32_t* __restrict__ row_list,
                                                                   const AggSetDesc* __restrict__ sets, int nsets, unsigned long long ord_base) {
  __shared__ VmInstr s_code[VM_MAX_CODE];
  __shared__ uint64_t s_pool[VM_MAX_POOL];
  load_program(prog, s_code, s_pool);
  int* err = (int*)(tab.counters + 2);
  const long long ntiles = (n + AG_TILE - 1) / AG_TILE;
  for (long long tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    long long row[AG_R]; bool inb[AG_R], alive[AG_R];
    uint32_t rel[AG_R]; int only[AG_R];
#pragma unroll
    for (int r = 0; r < AG_R; r++) {
      const long long i = tile * AG_TILE + r * AG_BLOCK + threadIdx.x;
      inb[r] = i < n; alive[r] = inb[r];
      const uint32_t e = inb[r] ? (row_list ? row_list[i] : (uint32_t)i) : 0;
      rel[r] = row_list ? e / (uint32_t)nsets : e;
      only[r] = row_list ? (int)(e % (uint32_t)nsets) : -1;
      row[r] = row_begin + rel[r];
    }
    uint64_t buf[AG_R][AGG_MAX_ROW_WORDS];
    uint32_t vb[AG_R];
#pragma unroll
    for (int r = 0; r < AG_R; r++) vb[r] = 0;
    AggSink sink{buf, vb, lay.out_word};
    vm_run<AG_R>(s_code, s_pool, 0, cols, row, inb, alive, err, sink);
#pragma unroll
    for (int r = 0; r < AG_R; r++) {
      if (!alive[r]) continue;
      const int s0 = only[r] < 0 ? 0 : only[r], s1 = only[r] < 0 ? nsets : only[r] + 1;
      for (int s = s0; s < s1; s++) {
        if (!agg_upsert_set(lay, tab, buf[r], vb[r], sets + s, (ord_base + (unsigned long long)row[r]) * (unsigned)nsets + (unsigned)s)) {
          const unsigned long long at = atomicAdd(tab.counters + 1, 1ULL);
          tab.deferred[at] = rel[r] * (uint32_t)nsets + (uint32_t)s;
        }
      }
    }
  }
}

static int grid_for(int64_t ntiles, int per_sm) {
  int dev = 0, sms = 132; cudaGetDevice(&dev); cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  const int64_t cap = (int64_t)sms * per_sm;       // grid = multiple of the SM count (persistent, grid-stride)
  return (int)(ntiles < cap ? (ntiles < 1 ? 1 : ntiles) : cap);
}

int launch_agg_update(const VmProgram* d_prog, const ColTable& cols, const AggLayout& lay, const AggTable& tab, int64_t row_begin, int64_t n,
                      const uint32_t* d_row_list, uint64_t ord_base, cudaStream_t s) {
  if (n <= 0) return 0;
  const int64_t ntiles = (n + AG_TILE - 1) / AG_TILE;
  agg_update_kernel<<<grid_for(ntiles, 8), AG_BLOCK, 0, s>>>(d_prog, cols, lay, tab, row_begin, n, d_row_list, ord_base);
  return 1;
}

int launch_agg_update_sets(const VmProgram* d_prog, const ColTable& cols, const AggLayout& lay, const AggTable& tab, int64_t row_begin, int64_t n,
                           const uint32_t* d_row_list, const AggSetDesc* d_sets, int nsets, uint64_t ord_base, cudaStream_t s) {
  if (n <= 0) return 0;
  const int64_t ntiles = (n + AG_TILE - 1) / AG_TILE;
  agg_update_sets_kernel<<<grid_for(ntiles, 8), AG_BLOCK, 0, s>>>(d_prog, cols, lay, tab, row_begin, n, d_row_list, d_sets, nsets, ord_base);
  return 1;
}

// ---------------------------------------------------------------------------------------------------
// HashAgg: grow (rehash into a larger table)
// ---------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) agg_rehash_kernel(const AggLayout lay, const AggTable old_tab, const AggTable new_tab) {
  const uint64_t cap = old_tab.capacity;
  for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < cap; i += (uint64_t)gridDim.x * blockDim.x) {
    const unsigned long long* src = old_tab.keys + i * (uint64_t)lay.kstride;
    const unsigned long long hdr = src[0];
    if ((unsigned)hdr < 2) continue;
    const unsigned knull = (unsigned)(hdr >> 48);
    const uint64_t h = agg_hash_words((const uint64_t*)src + 1, lay.nkw, knull);
    uint64_t s = agg_first_slot(h, new_tab.capacity);
    while (true) {
      unsigned long long* dst = new_tab.keys + s * (uint64_t)lay.kstride;
      if (atomicCAS((unsigned*)dst, TAG_EMPTY, TAG_LOCKED) == TAG_EMPTY) {
        for (int w = 1; w < lay.kstride; w++) dst[w] = src[w];
        for (int w = 0; w < lay.astride; w++) new_tab.accs[s * (uint64_t)lay.astride + w] = old_tab.accs[i * (uint64_t)lay.astride + w];
        ((unsigned*)dst)[1] = (unsigned)(hdr >> 32) & ~FLAG_SLOT_LOCK;
        __threadfence();
        st_release_u32((unsigned*)dst, (unsigned)hdr);
        atomicAdd(new_tab.counters, 1ULL);
        break;
      }
      s = agg_next_slot(s, new_tab.capacity);
    }
  }
}

int launch_agg_rehash(const AggLayout& lay, const AggTable& old_tab, const AggTable& new_tab, cudaStream_t s) {
  const int64_t cap = (int64_t)old_tab.capacity;
  agg_rehash_kernel<<<grid_for((cap + 255) / 256, 8), 256, 0, s>>>(lay, old_tab, new_tab);
  return 1;
}

// ---------------------------------------------------------------------------------------------------
// HashAgg: emit
// ---------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) agg_emit_kernel(const AggLayout lay, const AggTable tab, const EmitTable emit, unsigned long long* out_count) {
  const uint64_t cap = tab.capacity;
  const unsigned lane = threadIdx.x & 31;
  const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
  const uint64_t rounds = (cap + stride - 1) / stride;
  for (uint64_t it = 0; it < rounds; it++) {
    const uint64_t i = it * stride + blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    const unsigned long long* ke = tab.keys + i * (uint64_t)lay.kstride;
    const unsigned long long* slot = tab.accs + i * (uint64_t)lay.astride;      // accumulator entry
    unsigned long long hdr = 0;
    if (i < cap) hdr = ke[0];
    const bool occ = (unsigned)hdr >= 2;
    const unsigned m = __ballot_sync(0xffffffffu, occ);
    if (!m) continue;
    unsigned long long base = 0;
    if (lane == 0) base = atomicAdd(out_count, (unsigned long long)__popc(m));       // warp-aggregated claim of output rows
    base = __shfl_sync(0xffffffffu, base, 0);
    if (!occ) continue;
    const unsigned long long at = base + __popc(m & lanemask_lt());
    const unsigned flags = (unsigned)(hdr >> 32);
    emit_row_columns(emit, at, ke, slot, flags);
  }
}

int launch_agg_emit(const AggLayout& lay, const AggTable& tab, const EmitTable& emit, unsigned long long* d_out_count, cudaStream_t s) {
  const int64_t cap = (int64_t)tab.capacity;
  agg_emit_kernel<<<grid_for((cap + 255) / 256, 8), 256, 0, s>>>(lay, tab, emit, d_out_count);
  return 1;
}

__global__ void copy_words_to_host_kernel(const unsigned long long* __restrict__ src, unsigned long long* __restrict__ dst, int n) {
  if ((int)threadIdx.x < n) dst[threadIdx.x] = src[threadIdx.x];
}
int launch_copy_words_to_host(const unsigned long long* src, unsigned long long* pinned_dst, int n, cudaStream_t s) {
  copy_words_to_host_kernel<<<1, 32, 0, s>>>(src, pinned_dst, n);
  return 1;
}

__global__ void __launch_bounds__(256) pack_valid_kernel(const uint8_t* __restrict__ bytes, uint32_t* __restrict__ bits, long long n) {
  const long long nwords = (n + 31) / 32;
  const unsigned lane = threadIdx.x & 31;
  // one warp packs 32 words (1024 rows) per step: lane l reads byte (w*32 + l), ballot gives the word
  const long long warp_id = (blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5, nwarps = ((long long)gridDim.x * blockDim.x) >> 5;
  for (long long w = warp_id; w < nwords; w += nwarps) {
    const long long i = w * 32 + lane;
    const unsigned m = __ballot_sync(0xffffffffu, i < n && bytes[i] != 0);
    if (lane == 0) bits[w] = m;
  }
}

int launch_pack_valid(const uint8_t* bytes, uint32_t* bits, int64_t n, cudaStream_t s) {
  if (n <= 0) return 0;
  pack_valid_kernel<<<grid_for((n + 8191) / 8192, 8), 256, 0, s>>>(bytes, bits, n);
  return 1;
}

// ---------------------------------------------------------------------------------------------------
// frozen accumulator rows (the Binary `#9223372036854775807` column)
// ---------------------------------------------------------------------------------------------------
__device__ __forceinline__ int varint_len(unsigned long long v) { int n = 1; while (v >= 128) { v >>= 7; n++; } return n; }

__device__ __forceinline__ unsigned long long state_value_bits(const FrozenField& f, long long i, unsigned long long& hi) {
  hi = 0;
  switch (f.phys) {
    case PH_I8: return (unsigned long long)(long long)((const int8_t*)f.values)[i];
    case PH_I16: return (unsigned long long)(long long)((const int16_t*)f.values)[i];
    case PH_I32: return (unsigned long long)(long long)((const int32_t*)f.values)[i];
    case PH_F32: return (unsigned long long)((const uint32_t*)f.values)[i];
    case PH_DEC128: hi = ((const unsigned long long*)f.values)[2 * i + 1]; return ((const unsigned long long*)f.values)[2 * i];
    default: return ((const unsigned long long*)f.values)[i];
  }
}

__global__ void __launch_bounds__(256) frozen_lengths_kernel(const FrozenTable ft, long long n, int32_t* __restrict__ lengths) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    int len = 0;
    for (int k = 0; k < ft.nfields; k++) {
      const FrozenField& f = ft.f[k];
      if (f.kind == FZ_COUNT) len += varint_len(((const unsigned long long*)f.values)[i]);
      else if (f.kind == FZ_BOOL) len += 1;
      else len += 1 + ((f.valid ? f.valid[i] != 0 : true) ? f.width : 0);
    }
    lengths[i] = len;
  }
}

__global__ void __launch_bounds__(256) frozen_write_kernel(const FrozenTable ft, long long n, const int32_t* __restrict__ offsets, uint8_t* __restrict__ data) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    uint8_t* p = data + offsets[i];
    for (int k = 0; k < ft.nfields; k++) {
      const FrozenField& f = ft.f[k];
      if (f.kind == FZ_COUNT) {
        unsigned long long v = ((const unsigned long long*)f.values)[i];           // write_len (io/mod.rs:60-68)
        while (v >= 128) { *p++ = (uint8_t)(128 + (v & 127)); v >>= 7; }
        *p++ = (uint8_t)v;
      } else if (f.kind == FZ_BOOL) {                                              // acc.rs:180-190
        const uint8_t v = ((const uint8_t*)f.values)[i] != 0;
        *p++ = f.valid ? (f.valid[i] ? 1 + v : 0) : (v ? 2 : 0);
      } else {
        const bool valid = f.valid ? f.valid[i] != 0 : true;
        *p++ = valid ? 1 : 0;                                                      // acc.rs:335-346
        if (valid) {
          unsigned long long hi, lo = state_value_bits(f, i, hi);
          for (int b = 0; b < f.width && b < 8; b++) *p++ = (uint8_t)(lo >> (8 * b));
          for (int b = 8; b < f.width; b++) *p++ = (uint8_t)(hi >> (8 * (b - 8)));
        }
      }
    }
  }
}

__global__ void __launch_bounds__(256) frozen_read_kernel(const FrozenTable ft, long long n, const int32_t* __restrict__ offsets, long long obase,
                                                          const uint8_t* __restrict__ data, int* err) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const uint8_t* p = data + offsets[obase + i];
    const uint8_t* end = data + offsets[obase + i + 1];
    for (int k = 0; k < ft.nfields; k++) {
      const FrozenField& f = ft.f[k];
      if (f.kind == FZ_COUNT) {                                                    // read_len (io/mod.rs:70-83)
        unsigned long long v = 0; int shift = 0;
        while (true) {
          if (p >= end) { atomicOr(err, 4); break; }
          const uint8_t b = *p++;
          if (b < 128) { v += (unsigned long long)b << shift; break; }
          v += (unsigned long long)(b - 128) << shift; shift += 7;
        }
        ((unsigned long long*)f.values)[i] = v;
      } else if (f.kind == FZ_BOOL) {                                              // acc.rs:193-207
        if (p >= end) { atomicOr(err, 4); break; }
        const uint8_t b = *p++;
        if (f.valid) { ((uint8_t*)f.valid)[i] = b != 0; ((uint8_t*)f.values)[i] = b > 1; }
        else ((uint8_t*)f.values)[i] = b != 0;                                     // FIRST's flag: any non-zero byte is set
      } else {                                                                     // acc.rs:349-365
        if (p >= end) { atomicOr(err, 4); break; }
        const bool valid = *p++ == 1;
        unsigned long long lo = 0, hi = 0;
        if (valid) {
          if (p + f.width > end) { atomicOr(err, 4); break; }
          for (int b = 0; b < f.width && b < 8; b++) lo |= (unsigned long long)(*p++) << (8 * b);
          for (int b = 8; b < f.width; b++) hi |= (unsigned long long)(*p++) << (8 * (b - 8));
        }
        ((uint8_t*)f.valid)[i] = valid ? 1 : 0;
        switch (f.phys) {
          case PH_I8: ((int8_t*)f.values)[i] = (int8_t)lo; break;
          case PH_I16: ((int16_t*)f.values)[i] = (int16_t)lo; break;
          case PH_I32: case PH_F32: ((uint32_t*)f.values)[i] = (uint32_t)lo; break;
          case PH_DEC128: ((unsigned long long*)f.values)[2 * i] = lo; ((unsigned long long*)f.values)[2 * i + 1] = hi; break;
          default: ((unsigned long long*)f.values)[i] = lo; break;
        }
      }
    }
  }
}

int launch_frozen_lengths(const FrozenTable& ft, int64_t n, int32_t* lengths, cudaStream_t s) {
  if (n <= 0) return 0;
  frozen_lengths_kernel<<<grid_for((n + 255) / 256, 8), 256, 0, s>>>(ft, n, lengths); return 1;
}
int launch_frozen_write(const FrozenTable& ft, int64_t n, const int32_t* offsets, uint8_t* data, cudaStream_t s) {
  if (n <= 0) return 0;
  frozen_write_kernel<<<grid_for((n + 255) / 256, 8), 256, 0, s>>>(ft, n, offsets, data); return 1;
}
int launch_frozen_read(const FrozenTable& ft, int64_t n, const int32_t* offsets, int64_t offsets_base, const uint8_t* data, int* d_err, cudaStream_t s) {
  if (n <= 0) return 0;
  frozen_read_kernel<<<grid_for((n + 255) / 256, 8), 256, 0, s>>>(ft, n, offsets, offsets_base, data, d_err); return 1;
}

// exclusive scan of int32 (n -> n+1 offsets): block sums, scan of the sums by one block, final pass
constexpr int SCAN_BLOCK = 256, SCAN_ITEMS = 8, SCAN_TILE = SCAN_BLOCK * SCAN_ITEMS;
int64_t scan_num_blocks(int64_t n) { return (n + SCAN_TILE - 1) / SCAN_TILE; }

__device__ __forceinline__ int block_exclusive_scan(int v, int* total, int* smem /*>=9 ints*/) {
  const unsigned lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int incl = v;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) { int t = __shfl_up_sync(0xffffffffu, incl, d); if (lane >= d) incl += t; }
  if (lane == 31) smem[warp] = incl;
  __syncthreads();
  if (warp == 0) {
    int w = lane < SCAN_BLOCK / 32 ? smem[lane] : 0, wi = w;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) { int t = __shfl_up_sync(0xffffffffu, wi, d); if (lane >= d) wi += t; }
    if (lane < SCAN_BLOCK / 32) smem[lane] = wi - w;
    if (lane == SCAN_BLOCK / 32 - 1) smem[8] = wi;
  }
  __syncthreads();
  const int res = incl - v + smem[warp];
  *total = smem[8];
  __syncthreads();
  return res;
}

__global__ void __launch_bounds__(SCAN_BLOCK) scan_block_sums_kernel(const int32_t* __restrict__ in, long long n, int32_t* __restrict__ block_sums) {
  __shared__ int smem[9];
  const long long base = blockIdx.x * (long long)SCAN_TILE;
  int s = 0;
  for (int k = 0; k < SCAN_ITEMS; k++) { const long long i = base + k * SCAN_BLOCK + threadIdx.x; if (i < n) s += in[i]; }
  int total; block_exclusive_scan(s, &total, smem);
  if (threadIdx.x == 0) block_sums[blockIdx.x] = total;
}
__global__ void __launch_bounds__(SCAN_BLOCK) scan_sums_kernel(int32_t* block_sums, long long nb) {
  __shared__ int smem[9];
  int carry = 0;
  for (long long base = 0; base < nb; base += SCAN_BLOCK) {
    const long long i = base + threadIdx.x;
    const int v = i < nb ? block_sums[i] : 0;
    int total; const int ex = block_exclusive_scan(v, &total, smem);
    if (i < nb) block_sums[i] = carry + ex;
    carry += total;
  }
}
__global__ void __launch_bounds__(SCAN_BLOCK) scan_final_kernel(const int32_t* __restrict__ in, int32_t* __restrict__ out, long long n, const int32_t* __restrict__ block_sums) {
  __shared__ int smem[9];
  const long long base = blockIdx.x * (long long)SCAN_TILE + (long long)threadIdx.x * SCAN_ITEMS;
  int v[SCAN_ITEMS], s = 0;
#pragma unroll
  for (int k = 0; k < SCAN_ITEMS; k++) { v[k] = base + k < n ? in[base + k] : 0; s += v[k]; }
  int total; int ex = block_exclusive_scan(s, &total, smem) + block_sums[blockIdx.x];
#pragma unroll
  for (int k = 0; k < SCAN_ITEMS; k++) { if (base + k < n) out[base + k] = ex; ex += v[k]; }
  // the last element out[n] = grand total: written by the thread that owns index n-1
  if (n > 0 && base <= n - 1 && n - 1 < base + SCAN_ITEMS) out[n] = ex;   // ex now = exclusive prefix after this thread's items
}

int launch_exclusive_scan_i32(const int32_t* in, int32_t* out, int64_t n, int32_t* d_block_sums, cudaStream_t s) {
  if (n <= 0) { cudaMemsetAsync(out, 0, sizeof(int32_t), s); return 0; }
  const int64_t nb = scan_num_blocks(n);
  scan_block_sums_kernel<<<(unsigned)nb, SCAN_BLOCK, 0, s>>>(in, n, d_block_sums);
  scan_sums_kernel<<<1, SCAN_BLOCK, 0, s>>>(d_block_sums, nb);
  scan_final_kernel<<<(unsigned)nb, SCAN_BLOCK, 0, s>>>(in, out, n, d_block_sums);
  return 3;
}

// ---------------------------------------------------------------------------------------------------
// variable-width gather (FilterExec / ProjectExec carrying Utf8 / Binary columns)
// ---------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) varlen_lengths_kernel(const DevCol src, const uint32_t* __restrict__ sel, long long m, int32_t* __restrict__ lengths,
                                                             uint32_t* __restrict__ out_valid, unsigned long long* __restrict__ total) {
  const unsigned lane = threadIdx.x & 31;
  unsigned long long sum = 0;
  // 32 consecutive output rows per warp step: one validity word per step
  for (long long base = (blockIdx.x * (long long)blockDim.x + threadIdx.x) & ~31LL; base < m; base += (long long)gridDim.x * blockDim.x) {
    const long long i = base + lane;
    bool valid = false;
    if (i < m) {
      const long long j = sel ? (long long)sel[i] : i;
      const int32_t len = src.offsets[j + 1] - src.offsets[j];
      lengths[i] = len; sum += (unsigned long long)len;
      valid = true;
      if (src.validity) { const unsigned long long bi = (unsigned long long)j + src.bit_offset; valid = (src.validity[bi >> 3] >> (bi & 7)) & 1; }
    }
    const unsigned w = __ballot_sync(0xffffffffu, valid);
    if (out_valid && lane == 0) out_valid[base >> 5] = w;
  }
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, d);
  if (lane == 0 && sum) atomicAdd(total, sum);
}

struct alignas(16) V16 { unsigned long long lo, hi; };     // one 128-bit load / store

// 16 output bytes from a source that is `m` (1..15) bytes past a 16-byte boundary: two aligned 16-byte loads, then each output word is
// a funnel shift of two neighbouring source words
__device__ __forceinline__ V16 shifted16(const V16* __restrict__ src, int v, unsigned m) {
  const V16 a = src[v], b = src[v + 1];
  const uint32_t w[8] = {(uint32_t)a.lo, (uint32_t)(a.lo >> 32), (uint32_t)a.hi, (uint32_t)(a.hi >> 32),
                         (uint32_t)b.lo, (uint32_t)(b.lo >> 32), (uint32_t)b.hi, (uint32_t)(b.hi >> 32)};
  const unsigned q = m >> 2, sh = (m & 3) * 8;
  uint32_t x[5];
#pragma unroll
  for (int i = 0; i < 5; i++) x[i] = q == 0 ? w[i] : q == 1 ? w[i + 1] : q == 2 ? w[i + 2] : w[i + 3];
  uint32_t o[4];
#pragma unroll
  for (int i = 0; i < 4; i++) o[i] = (uint32_t)(((((uint64_t)x[i + 1]) << 32) | x[i]) >> sh);
  V16 r; r.lo = o[0] | ((unsigned long long)o[1] << 32); r.hi = o[2] | ((unsigned long long)o[3] << 32);
  return r;
}

// n bytes sp -> dp by the whole warp.  Runs of 64 bytes or more are stored as aligned 16-byte vectors: the loads are aligned
// 16-byte vectors too, shifted into place when source and destination disagree modulo 16 (both loads of a lane hold at least one
// byte of the run, so they stay inside its buffer).  Heads and tails are coalesced byte copies.
__device__ __forceinline__ void warp_copy_bytes(const uint8_t* sp, uint8_t* dp, int n, unsigned lane) {
  int done = 0;
  if (n >= 64) {
    const int head = (int)((16 - ((uintptr_t)dp & 15)) & 15);
    if ((int)lane < head) dp[lane] = sp[lane];
    const int nv = (n - head) >> 4;
    const uint8_t* s = sp + head; V16* vd = (V16*)(dp + head);
    const unsigned mis = (unsigned)((uintptr_t)s & 15);
    if (mis == 0) { const V16* vs = (const V16*)s; for (int v = (int)lane; v < nv; v += 32) vd[v] = vs[v]; }
    else { const V16* vs = (const V16*)(s - mis); for (int v = (int)lane; v < nv; v += 32) vd[v] = shifted16(vs, v, mis); }
    done = head + (nv << 4);
  }
  for (int b = done + (int)lane; b < n; b += 32) dp[b] = sp[b];
}

// One warp per group of 32 output rows; the rows are copied one after the other by the whole warp, so a long string spreads over
// 32 lanes (and every warp of the grid keeps its own rows).
__global__ void __launch_bounds__(256) varlen_copy_kernel(const DevCol src, const uint32_t* __restrict__ sel, long long m,
                                                          const int32_t* __restrict__ out_offsets, uint8_t* __restrict__ out) {
  const unsigned lane = threadIdx.x & 31;
  const long long warps = ((long long)gridDim.x * blockDim.x) >> 5;
  const uint8_t* data = (const uint8_t*)src.values;
  for (long long base = ((blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5) * 32; base < m; base += warps * 32) {
    const long long i = base + lane;
    long long s0 = 0, d0 = 0; int len = 0;
    if (i < m) { const long long j = sel ? (long long)sel[i] : i; s0 = src.offsets[j]; len = src.offsets[j + 1] - (int32_t)s0; d0 = out_offsets[i]; }
    const int cnt = (int)(m - base < 32 ? m - base : 32);
    for (int k = 0; k < cnt; k++)
      warp_copy_bytes(data + __shfl_sync(0xffffffffu, s0, k), out + __shfl_sync(0xffffffffu, d0, k), __shfl_sync(0xffffffffu, len, k), lane);
  }
}

int launch_varlen_lengths(const DevCol& src, const uint32_t* sel, int64_t m, int32_t* lengths, uint32_t* out_valid, unsigned long long* d_total, cudaStream_t s) {
  if (m <= 0) return 0;
  varlen_lengths_kernel<<<grid_for((m + 255) / 256, 8), 256, 0, s>>>(src, sel, m, lengths, out_valid, d_total);
  return 1;
}
int launch_varlen_copy(const DevCol& src, const uint32_t* sel, int64_t m, const int32_t* out_offsets, uint8_t* out_data, cudaStream_t s) {
  if (m <= 0) return 0;
  varlen_copy_kernel<<<grid_for((m + 255) / 256, 8), 256, 0, s>>>(src, sel, m, out_offsets, out_data);
  return 1;
}

// ---------------------------------------------------------------------------------------------------
// IpcReaderExec: batch_serde records -> coalesced columns (the inverse of the shuffle encode kernels).  Every extent a kernel
// reads was checked by the host walk of the records (ipc_records.cc) before the launch.
// ---------------------------------------------------------------------------------------------------
// `W` byte planes of `rows` bytes -> `rows` little-endian values of W bytes.  A warp reads 32 consecutive bytes of each plane
// (one sector per plane) and stores 32 whole values: one naturally aligned store per value (16 bytes for decimal128).
template <int W>
__device__ __forceinline__ void ipc_untranspose(const uint8_t* __restrict__ src, uint8_t* __restrict__ dst, long long rows, long long r0, long long r1) {
  for (long long r = r0 + threadIdx.x; r < r1; r += blockDim.x) {
    unsigned long long lo = 0, hi = 0;
#pragma unroll
    for (int k = 0; k < W; k++) {
      const unsigned long long b = __ldg(src + (long long)k * rows + r);
      if (k < 8) lo |= b << (8 * k); else hi |= b << (8 * (k - 8));
    }
    if constexpr (W == 16) { V16 v; v.lo = lo; v.hi = hi; ((V16*)dst)[r] = v; }
    else if constexpr (W == 8) ((unsigned long long*)dst)[r] = lo;
    else if constexpr (W == 4) ((uint32_t*)dst)[r] = (uint32_t)lo;
    else if constexpr (W == 2) ((uint16_t*)dst)[r] = (uint16_t)lo;
    else dst[r] = (uint8_t)lo;
  }
}

// one block per (record, column) tile of IPC_TILE rows; one launch covers every fixed-width column of a flush
__global__ void __launch_bounds__(256) ipc_decode_fixed_kernel(const IpcFixedJob* __restrict__ jobs, const IpcTile* __restrict__ tiles, long long ntiles) {
  for (long long t = blockIdx.x; t < ntiles; t += gridDim.x) {
    const IpcTile tl = tiles[t];
    const IpcFixedJob j = jobs[tl.job];
    const long long r0 = (long long)tl.row0, r1 = r0 + IPC_TILE < j.rows ? r0 + IPC_TILE : j.rows;
    switch (j.width) {
      case 1: ipc_untranspose<1>(j.src, j.dst, j.rows, r0, r1); break;
      case 2: ipc_untranspose<2>(j.src, j.dst, j.rows, r0, r1); break;
      case 4: ipc_untranspose<4>(j.src, j.dst, j.rows, r0, r1); break;
      case 8: ipc_untranspose<8>(j.src, j.dst, j.rows, r0, r1); break;
      default: ipc_untranspose<16>(j.src, j.dst, j.rows, r0, r1); break;
    }
  }
}

// Validity bitmaps and Boolean values: records start at any output row, so their bits are re-packed at a bit offset.  One thread
// per output word (no atomics): it finds the record holding the word's first row and takes up to 32 bits from each record the
// word overlaps, as a funnel shift of the (at most 5) source bytes that hold them.  A record without a bitmap (src null) gives
// all-valid bits.
__global__ void __launch_bounds__(256) ipc_decode_bits_kernel(const IpcBitCol* __restrict__ cols, int ncols, const long long* __restrict__ rec_row, long long nrec, long long rows) {
  const long long nwords = (rows + 31) >> 5;
  for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < nwords * ncols; t += (long long)gridDim.x * blockDim.x) {
    const IpcBitCol c = cols[t / nwords];
    const long long w = t % nwords;
    const long long b0 = w << 5, b1 = b0 + 32 < rows ? b0 + 32 : rows;
    long long lo = 0, hi = nrec - 1;                                   // the last record that starts at or before b0
    while (lo < hi) { const long long mid = (lo + hi + 1) >> 1; if (rec_row[mid] <= b0) lo = mid; else hi = mid - 1; }
    uint32_t word = 0;
    for (long long r = lo, b = b0; b < b1; r++) {
      const long long rs = rec_row[r], rn = rec_row[r + 1], re = rn < b1 ? rn : b1;
      if (re <= b) continue;                                           // a record of 0 rows
      const int len = (int)(re - b);
      const uint32_t mask = len == 32 ? 0xFFFFFFFFu : (1u << len) - 1;
      const uint8_t* src = c.src[r];
      uint32_t bits = mask;
      if (src) {
        const long long sb = b - rs, byte = sb >> 3, nbytes = (rn - rs + 7) >> 3;
        unsigned long long v = 0;
#pragma unroll
        for (int k = 0; k < 5; k++) if (byte + k < nbytes) v |= (unsigned long long)__ldg(src + byte + k) << (8 * k);
        bits = (uint32_t)(v >> (sb & 7)) & mask;
      }
      word |= bits << (int)(b - b0);
      b = re;
    }
    c.dst[w] = word;
  }
}

// Binary / Utf8 row bytes: each record's bytes are contiguous in the stream and in the output, so a flush is a list of range
// copies (cut by the host into pieces of at most IPC_COPY_PIECE bytes).  Each warp loads 32 pieces (one per lane) and copies them one
// after the other, as varlen_copy_kernel does with rows.
__global__ void __launch_bounds__(256) ipc_decode_bytes_kernel(const IpcCopy* __restrict__ copies, long long n) {
  const unsigned lane = threadIdx.x & 31;
  const long long warps = ((long long)gridDim.x * blockDim.x) >> 5;
  for (long long base = ((blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5) * 32; base < n; base += warps * 32) {
    const long long i = base + lane;
    unsigned long long sp = 0, dp = 0; int len = 0;
    if (i < n) { sp = (unsigned long long)copies[i].src; dp = (unsigned long long)copies[i].dst; len = (int)copies[i].len; }
    const int cnt = (int)(n - base < 32 ? n - base : 32);
    for (int k = 0; k < cnt; k++)
      warp_copy_bytes((const uint8_t*)__shfl_sync(0xffffffffu, sp, k), (uint8_t*)__shfl_sync(0xffffffffu, dp, k), __shfl_sync(0xffffffffu, len, k), lane);
  }
}

int launch_ipc_decode_fixed(const IpcFixedJob* jobs, const IpcTile* tiles, int64_t ntiles, cudaStream_t s) {
  if (ntiles <= 0) return 0;
  ipc_decode_fixed_kernel<<<grid_for(ntiles, 8), 256, 0, s>>>(jobs, tiles, ntiles);
  return 1;
}
int launch_ipc_decode_bits(const IpcBitCol* cols, int ncols, const int64_t* rec_row, int64_t nrec, int64_t rows, cudaStream_t s) {
  if (ncols <= 0 || rows <= 0) return 0;
  ipc_decode_bits_kernel<<<grid_for(((rows + 31) / 32 * ncols + 255) / 256, 8), 256, 0, s>>>(cols, ncols, (const long long*)rec_row, nrec, rows);
  return 1;
}
int launch_ipc_decode_bytes(const IpcCopy* copies, int64_t n, cudaStream_t s) {
  if (n <= 0) return 0;
  ipc_decode_bytes_kernel<<<grid_for((n + 7) / 8, 8), 256, 0, s>>>(copies, n);
  return 1;
}

// ---------------------------------------------------------------------------------------------------
// Spark murmur3 (seed 42) + pmod — hash/mur.rs:19-87, spark_hash.rs:62-200, shuffle/mod.rs:163-188
// ---------------------------------------------------------------------------------------------------
// (the murmur3 rounds are in hash.cuh)

struct PhysList { uint8_t phys[VM_MAX_COLS]; };

__global__ void __launch_bounds__(256) murmur3_partition_kernel(const ColTable cols, const PhysList pl, int ncols, long long n, int num_partitions, uint32_t* __restrict__ out) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    uint32_t h = 42;
    for (int c = 0; c < ncols; c++) {
      const DevCol col = cols.col[c];
      if (col.validity) { const unsigned long long bi = (unsigned long long)i + col.bit_offset; if (!((col.validity[bi >> 3] >> (bi & 7)) & 1)) continue; }   // NULL leaves the hash unchanged
      uint32_t w[4]; int nw;
      switch (pl.phys[c]) {
        case PH_BOOL: { const unsigned long long bi = (unsigned long long)i + col.bit_offset; w[0] = (((const uint8_t*)col.values)[bi >> 3] >> (bi & 7)) & 1; nw = 1; break; }
        case PH_I8: w[0] = (uint32_t)(int32_t)((const int8_t*)col.values)[i]; nw = 1; break;
        case PH_I16: w[0] = (uint32_t)(int32_t)((const int16_t*)col.values)[i]; nw = 1; break;
        case PH_I32: case PH_F32: w[0] = ((const uint32_t*)col.values)[i]; nw = 1; break;
        case PH_I64: case PH_F64: { const unsigned long long v = ((const unsigned long long*)col.values)[i]; w[0] = (uint32_t)v; w[1] = (uint32_t)(v >> 32); nw = 2; break; }
        default: { const unsigned long long a = ((const unsigned long long*)col.values)[2 * i], b = ((const unsigned long long*)col.values)[2 * i + 1];
                   w[0] = (uint32_t)a; w[1] = (uint32_t)(a >> 32); w[2] = (uint32_t)b; w[3] = (uint32_t)(b >> 32); nw = 4; break; }
      }
      uint32_t h1 = h;
      for (int k = 0; k < nw; k++) h1 = mm3_mix_h1(h1, mm3_mix_k1(w[k]));
      h = mm3_fmix(h1, (uint32_t)(4 * nw));
    }
    int32_t m = (int32_t)h % num_partitions;                                       // rem_euclid
    if (m < 0) m += num_partitions;
    out[i] = (uint32_t)m;
  }
}

int launch_murmur3_partition(const ColTable& cols, const uint8_t* phys, int ncols, int64_t n, int32_t num_partitions, uint32_t* out, cudaStream_t s) {
  if (n <= 0) return 0;
  PhysList pl; for (int i = 0; i < ncols && i < VM_MAX_COLS; i++) pl.phys[i] = phys[i];
  murmur3_partition_kernel<<<grid_for((n + 255) / 256, 8), 256, 0, s>>>(cols, pl, ncols, n, num_partitions, out);
  return 1;
}

}  // namespace b200q
