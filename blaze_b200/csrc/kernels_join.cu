// Hash join on the GPU (SURVEY.md §8(f) rank 2): build + probe + gather kernels of JoinBuildStage / JoinProbeStage.
//
// Reference (paths relative to the reference's native-engine/datafusion-ext-plans/src/):
//   Table::create_from_key_columns, lookup_many      joins/join_hash_map.rs:105-275
//   FullJoiner::join / finish                        joins/bhj/full_join.rs:209-362
//   SemiJoiner::join / finish                        joins/bhj/semi_join.rs:146-312
// The reference sorts (hash, row) pairs on the host to group duplicates into `mapped_indices` ranges, then probes 8-lane
// groups with software prefetch; every probe batch builds index vectors on one core and `take`s the columns.  Here the
// table has one slot per distinct key (the keys themselves are stored, so there is no separate compare pass), the rows of
// a key hang off the slot as a chain through `next[]` with their count in the slot, and a probe is: one lookup per row
// that yields (chain head, match count) -> exclusive scan of the counts -> one pass that walks the chains and writes
// (probe row, build row) pairs at their final positions -> one coalesced-write gather per output column.  The build side
// (date_dim-sized) stays L2-resident; the probe side streams.  Row order is not a contract (assert_batches_sorted_eq!).
#include <cuda_runtime.h>
#include <stdint.h>

#include <algorithm>

#include "kernels_join.cuh"

namespace b200q {

namespace {

constexpr int JB = 256;
#ifndef JOIN_MIN_CTAS
#define JOIN_MIN_CTAS 4       // the probe kernels are latency-bound (ncu: 34 % warps active at 70-80 registers): cap the registers for 4 CTAs per SM
#endif

int jgrid(int64_t n, int per_block = JB * 4) {
  int dev = 0, sms = 132; cudaGetDevice(&dev); cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  return (int)std::max<int64_t>(1, std::min<int64_t>((n + per_block - 1) / per_block, (int64_t)sms * 8));
}

__device__ __forceinline__ bool load_key(const JoinKeys& k, long long i, unsigned long long (&w)[2]) {
  w[0] = w[1] = 0;
#pragma unroll
  for (int c = 0; c < 2; c++) {
    if (c >= k.nkeys) break;
    const DevCol col = k.col[c];
    if (col.validity) { const unsigned long long bi = (unsigned long long)i + col.bit_offset; if (!((col.validity[bi >> 3] >> (bi & 7)) & 1)) return false; }
    long long v;
    switch (k.phys[c]) {
      case PH_I8: v = ((const int8_t*)col.values)[i]; break;
      case PH_I16: v = ((const int16_t*)col.values)[i]; break;
      case PH_I32: v = ((const int32_t*)col.values)[i]; break;
      default: v = ((const long long*)col.values)[i]; break;
    }
    w[c] = (unsigned long long)v;
  }
  return true;
}

__device__ __forceinline__ uint32_t key_hash(const unsigned long long (&w)[2]) {
  unsigned long long h = (w[0] ^ (w[1] * 0xC2B2AE3D27D4EB4Full)) * 0x9E3779B97F4A7C15ull;      // multiplicative (Fibonacci) hash: the high bits mix every input bit
  return (uint32_t)(h >> 32) ^ (uint32_t)(h >> 13);
}

// slot publication: keys are written, fenced, then the state becomes 2; readers fence after they have seen 2
__device__ __forceinline__ uint32_t ld_state(const uint32_t* p) { const uint32_t v = *(const volatile uint32_t*)p; __threadfence(); return v; }
__device__ __forceinline__ void st_state(uint32_t* p, uint32_t v) { __threadfence(); atomicExch(p, v); }

__global__ void __launch_bounds__(JB) join_build_kernel(const JoinKeys k, long long n, const JoinTable t) {
  for (long long i = blockIdx.x * (long long)JB + threadIdx.x; i < n; i += (long long)gridDim.x * JB) {
    unsigned long long w[2];
    t.next[i] = JOIN_NIL;
    if (!load_key(k, i, w)) continue;                                 // rows with a NULL key are not in the map (join_hash_map.rs:119-128)
    uint32_t slot = key_hash(w) & t.mask;
    while (true) {
      uint32_t st = ld_state(t.state + slot);
      if (st == 0) {
        st = atomicCAS(t.state + slot, 0u, 1u);
        if (st == 0) {
          t.keys[(size_t)slot * t.nkw] = w[0];
          if (t.nkw > 1) t.keys[(size_t)slot * t.nkw + 1] = w[1];
          st_state(t.state + slot, 2u);
          st = 2;
        }
      }
      while (st == 1) st = ld_state(t.state + slot);                    // another lane is publishing this slot's key
      const bool same = t.keys[(size_t)slot * t.nkw] == w[0] && (t.nkw == 1 || t.keys[(size_t)slot * t.nkw + 1] == w[1]);
      if (same) {
        t.next[i] = atomicExch(t.head + slot, (uint32_t)i);
        const uint32_t c = atomicAdd(t.count + slot, 1u) + 1;
        if (c > 1) atomicMax(t.stats, c);                              // stats[0] = rows of the most duplicated key (0 / 1: keys are unique)
        break;
      }
      slot = (slot + 1) & t.mask;
    }
  }
}

// probe view: ONE 16-byte load per probed slot for single-key tables ({key, count << 32 | head}; head = NIL marks an empty slot)
__device__ __forceinline__ bool probe(const JoinTable& t, const unsigned long long (&w)[2], uint32_t& head, uint32_t& count) {
  uint32_t slot = key_hash(w) & t.mask;
  while (true) {
    unsigned long long hc;
    bool same;
    if (t.nkw == 1) { const ulonglong2 e = *(const ulonglong2*)(t.packed + (size_t)slot * 2); hc = e.y; same = e.x == w[0]; }
    else { const ulonglong2 e = *(const ulonglong2*)(t.packed + (size_t)slot * 4); hc = t.packed[(size_t)slot * 4 + 2]; same = e.x == w[0] && e.y == w[1]; }
    if ((uint32_t)hc == JOIN_NIL) return false;
    if (same) { head = (uint32_t)hc; count = (uint32_t)(hc >> 32); return true; }
    slot = (slot + 1) & t.mask;
  }
}
__global__ void __launch_bounds__(JB) join_pack_kernel(const JoinTable t) {
  const unsigned long long cap = (unsigned long long)t.mask + 1;
  const int stride = t.nkw == 1 ? 2 : 4;
  for (unsigned long long s = blockIdx.x * (unsigned long long)JB + threadIdx.x; s < cap; s += (unsigned long long)gridDim.x * JB) {
    const bool used = t.state[s] == 2;
    for (int i = 0; i < t.nkw; i++) t.packed[s * stride + i] = used ? t.keys[s * t.nkw + i] : 0;
    t.packed[s * stride + t.nkw] = used ? ((unsigned long long)t.count[s] << 32) | t.head[s] : (unsigned long long)JOIN_NIL;
  }
}

__global__ void __launch_bounds__(JB, JOIN_MIN_CTAS) join_probe_count_kernel(const JoinKeys k, long long n, const JoinTable t, int probe_outer, uint32_t* __restrict__ head, int32_t* __restrict__ count,
                                                              unsigned long long* total) {
  // 8 rows per thread and step: the eight key loads, then the eight table probes, are independent of each other — with one row per
  // thread the kernel is latency-bound (16 KB of key loads in flight per SM, measured 4.4e10 rows/s)
  constexpr int R = 8;
  unsigned long long mine = 0;
  const long long ntiles = (n + JB * R - 1) / (JB * R);
  for (long long tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const long long t0 = tile * (JB * R);
    unsigned long long w[R][2]; bool ok[R];
#pragma unroll
    for (int r = 0; r < R; r++) { const long long i = t0 + r * JB + threadIdx.x; ok[r] = i < n && load_key(k, i, w[r]); }      // a NULL in any key column never matches (full_join.rs:262-267)
#pragma unroll
    for (int r = 0; r < R; r++) {
      const long long i = t0 + r * JB + threadIdx.x;
      uint32_t h = JOIN_NIL, c = 0;
      if (ok[r]) probe(t, w[r], h, c);
      if (i < n) {
        if (probe_outer && c == 0) c = 1;
        head[i] = h;
        if (count) count[i] = (int32_t)c;
        mine += c;
      }
    }
  }
  if (total) {
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) mine += __shfl_xor_sync(0xFFFFFFFFu, mine, d);
    if ((threadIdx.x & 31) == 0 && mine) atomicAdd(total, mine);
  }
}

__global__ void __launch_bounds__(JB) join_probe_emit_kernel(long long n, const JoinTable t, const uint32_t* __restrict__ head, const int32_t* __restrict__ offs,
                                                             uint32_t* __restrict__ pidx, uint32_t* __restrict__ bidx, uint8_t* mark) {
  for (long long i = blockIdx.x * (long long)JB + threadIdx.x; i < n; i += (long long)gridDim.x * JB) {
    long long o = offs[i];
    const long long end = offs[i + 1];
    uint32_t b = head[i];
    if (b == JOIN_NIL) { if (o < end) { pidx[o] = (uint32_t)i; bidx[o] = JOIN_NIL; } continue; }      // unmatched outer row
    for (; b != JOIN_NIL && o < end; b = t.next[b], o++) {
      pidx[o] = (uint32_t)i; bidx[o] = b;
      if (mark) mark[b] = 1;
    }
  }
}

__global__ void __launch_bounds__(JB) join_mark_build_kernel(long long n, const JoinTable t, const uint32_t* __restrict__ head, uint8_t* mark) {
  for (long long i = blockIdx.x * (long long)JB + threadIdx.x; i < n; i += (long long)gridDim.x * JB) {
    uint32_t b = head[i];
    if (b == JOIN_NIL || mark[b]) continue;                            // all rows of this key were marked together (semi_join.rs:214-226)
    for (; b != JOIN_NIL; b = t.next[b]) mark[b] = 1;
  }
}

// Fused probe of the pair-producing joins (Inner / Left / Right / Full): lookup, then the CTA reserves the output rows of its
// 2048 consecutive probe rows with ONE atomic on `cursor` (block scan of the match counts) and every thread writes its
// (probe row, build row) pairs — no per-row intermediates, no global scan.  The output rows of a tile are contiguous and
// come from a contiguous input range, so the gathers that follow stay inside a 16 KB window per column; the order is not a contract.
// pidx == null: only count (cursor += matches), for build sides with duplicated keys whose output size is not bounded by n.
// The sums are 64-bit: one key may have up to 2^30 rows, so a thread's 8 rows can reach 2^33 and a tile 2^41.  In 32 bits a
// tile of 2048 rows of a 2^21-row key wraps to 0 and the caller sees no output instead of refusing the batch.
constexpr int JP_ROWS = 8;
__global__ void __launch_bounds__(JB) join_probe_pairs_kernel(const JoinKeys k, long long n, const JoinTable t, int probe_outer, unsigned long long* cursor,
                                                              uint32_t* __restrict__ pidx, uint32_t* __restrict__ bidx, uint8_t* mark) {
  __shared__ unsigned long long s_warp[JB / 32];
  __shared__ unsigned long long s_base;
  const unsigned lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const long long ntiles = (n + JB * JP_ROWS - 1) / (JB * JP_ROWS);
  for (long long tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const long long t0 = tile * (JB * JP_ROWS);
    uint32_t h[JP_ROWS]; unsigned c[JP_ROWS]; unsigned long long mine = 0;
#pragma unroll
    for (int r = 0; r < JP_ROWS; r++) {
      const long long i = t0 + r * JB + threadIdx.x;
      unsigned long long w[2];
      h[r] = JOIN_NIL; c[r] = 0;
      if (i < n) {
        if (load_key(k, i, w)) probe(t, w, h[r], c[r]);
        if (probe_outer && c[r] == 0) c[r] = 1;
      }
      mine += c[r];
    }
    unsigned long long inc = mine;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) { const unsigned long long o = __shfl_up_sync(0xFFFFFFFFu, inc, d); if (lane >= d) inc += o; }
    if (lane == 31) s_warp[warp] = inc;
    __syncthreads();
    unsigned long long before = 0, total = 0;
    for (int w = 0; w < JB / 32; w++) { const unsigned long long v = s_warp[w]; if (w < (int)warp) before += v; total += v; }
    if (threadIdx.x == 0 && total) s_base = atomicAdd(cursor, (unsigned long long)total);
    __syncthreads();
    if (pidx && mine) {
      unsigned long long o = s_base + before + inc - mine;
#pragma unroll
      for (int r = 0; r < JP_ROWS; r++) {
        if (c[r] == 0) continue;
        const uint32_t i = (uint32_t)(t0 + r * JB + threadIdx.x);
        if (h[r] == JOIN_NIL) { pidx[o] = i; bidx[o] = JOIN_NIL; o++; continue; }                     // unmatched outer row
        for (uint32_t b = h[r]; b != JOIN_NIL; b = t.next[b], o++) { pidx[o] = i; bidx[o] = b; if (mark) mark[b] = 1; }
      }
    }
    __syncthreads();
  }
}

// LeftSemi / LeftAnti with the probed side as the join side: idx[...] = the probe rows that have (invert: have no) partner
__global__ void __launch_bounds__(JB) join_probe_select_kernel(const JoinKeys k, long long n, const JoinTable t, int invert, unsigned long long* cursor, uint32_t* __restrict__ idx) {
  const unsigned lane = threadIdx.x & 31;
  const long long nround = (n + 31) & ~31LL;
  for (long long i = blockIdx.x * (long long)JB + threadIdx.x; i < nround; i += (long long)gridDim.x * JB) {
    unsigned long long w[2];
    bool keep = false;
    if (i < n) { uint32_t h_, c_; const bool found = load_key(k, i, w) && probe(t, w, h_, c_); keep = found != (invert != 0); }
    const unsigned m = __ballot_sync(0xFFFFFFFFu, keep);
    if (m == 0) continue;
    unsigned long long base = 0;
    if (lane == 0) base = atomicAdd(cursor, (unsigned long long)__popc(m));
    base = __shfl_sync(0xFFFFFFFFu, base, 0);
    if (keep) idx[base + __popc(m & ((1u << lane) - 1))] = (uint32_t)i;
  }
}

// semi-style probes where the BUILD side is the join side: lookup + mark the key's rows
__global__ void __launch_bounds__(JB) join_probe_mark_kernel(const JoinKeys k, long long n, const JoinTable t, uint8_t* mark) {
  for (long long i = blockIdx.x * (long long)JB + threadIdx.x; i < n; i += (long long)gridDim.x * JB) {
    unsigned long long w[2];
    if (!load_key(k, i, w)) continue;
    uint32_t b, c_;
    if (!probe(t, w, b, c_)) continue;
    if (mark[b]) continue;                                             // all rows of this key were marked together (semi_join.rs:214-226)
    for (; b != JOIN_NIL; b = t.next[b]) mark[b] = 1;
  }
}

template <typename T>
__global__ void __launch_bounds__(JB) join_gather_kernel(const T* __restrict__ src, const uint8_t* __restrict__ vbits, uint32_t bit_offset, const uint8_t* __restrict__ vbytes,
                                                         const uint32_t* __restrict__ idx, long long n, T* __restrict__ out, uint8_t* __restrict__ out_valid) {
  for (long long i = blockIdx.x * (long long)JB + threadIdx.x; i < n; i += (long long)gridDim.x * JB) {
    const uint32_t j = idx[i];
    T v{}; uint8_t ok = 0;
    if (j != JOIN_NIL) {
      ok = 1;
      if (vbytes) ok = vbytes[j];
      else if (vbits) { const unsigned long long bi = (unsigned long long)j + bit_offset; ok = (vbits[bi >> 3] >> (bi & 7)) & 1; }
      if (ok) v = src[j];
    }
    out[i] = v;
    if (out_valid) out_valid[i] = ok;
  }
}

struct u128 { unsigned long long a, b; };

// all output columns of one side in ONE pass over the index vector: column c of row i = src_c[idx[i]] (NULL when idx is NIL or
// the source value is NULL); validity leaves as one byte per row
__global__ void __launch_bounds__(JB) join_gather_multi_kernel(const GatherSpec g, const uint32_t* __restrict__ idx, long long n) {
  for (long long i = blockIdx.x * (long long)JB + threadIdx.x; i < n; i += (long long)gridDim.x * JB) {
    const uint32_t j = idx[i];
    for (int c = 0; c < g.ncols; c++) {
      const GatherCol col = g.col[c];
      uint8_t ok = 0;
      if (j != JOIN_NIL) {
        ok = 1;
        if (col.vbytes) ok = col.vbytes[j];
        else if (col.vbits) { const unsigned long long bi = (unsigned long long)j + col.bit_offset; ok = (col.vbits[bi >> 3] >> (bi & 7)) & 1; }
      }
      switch (col.width) {
        case 1: ((uint8_t*)col.out)[i] = ok ? ((const uint8_t*)col.src)[j] : 0; break;
        case 2: ((uint16_t*)col.out)[i] = ok ? ((const uint16_t*)col.src)[j] : 0; break;
        case 4: ((uint32_t*)col.out)[i] = ok ? ((const uint32_t*)col.src)[j] : 0; break;
        case 8: ((unsigned long long*)col.out)[i] = ok ? ((const unsigned long long*)col.src)[j] : 0; break;
        default: { u128 v{0, 0}; if (ok) v = ((const u128*)col.src)[j]; ((u128*)col.out)[i] = v; break; }
      }
      if (col.out_valid) col.out_valid[i] = ok;
    }
  }
}

// Fused probe + gather of the pair-producing joins when the map side's keys are UNIQUE (the PK side of a PK-FK join: every probe
// row has at most one partner).  One pass over the probe batch: lookup, ballots give every survivor its rank inside the tile in
// ROW order, one atomic per 2048-row tile reserves the tile's output rows, and the probe-side columns are copied (coalesced in,
// coalesced out) and the map-side columns gathered (L2-resident dimension table) straight into the output columns — no index
// vectors at all.  `total` rows were counted by a first pass (join_probe_pairs_kernel without outputs), so the outputs are exact.
__global__ void __launch_bounds__(JB, JOIN_MIN_CTAS) join_probe_fused_kernel(const uint32_t* __restrict__ head, long long n, int probe_outer, unsigned long long* cursor,
                                                              const GatherSpec pc, const GatherSpec bc, uint8_t* mark) {
  __shared__ unsigned s_cnt[JP_ROWS * (JB / 32) + 1];
  __shared__ unsigned long long s_base;
  const unsigned lane = threadIdx.x & 31, warp = threadIdx.x >> 5, lt = (1u << lane) - 1;
  const long long ntiles = (n + JB * JP_ROWS - 1) / (JB * JP_ROWS);
  for (long long tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const long long t0 = tile * (JB * JP_ROWS);
    uint32_t h[JP_ROWS]; unsigned bal[JP_ROWS];
#pragma unroll
    for (int r = 0; r < JP_ROWS; r++) {
      const long long i = t0 + r * JB + threadIdx.x;
      h[r] = JOIN_NIL; bool out = false;
      if (i < n) { h[r] = head[i]; out = h[r] != JOIN_NIL || probe_outer; }
      bal[r] = __ballot_sync(0xFFFFFFFFu, out);
      if (lane == 0) s_cnt[r * (JB / 32) + warp] = __popc(bal[r]);
      if (!out) h[r] = 0xFFFFFFFEu;                                        // no output row for this probe row
    }
    __syncthreads();
    if (warp == 0) {                                                       // exclusive prefix of the 64 (round, warp) counts in row order
      unsigned a = s_cnt[2 * lane], b = s_cnt[2 * lane + 1], inc = a + b;
#pragma unroll
      for (int d = 1; d < 32; d <<= 1) { const unsigned o = __shfl_up_sync(0xFFFFFFFFu, inc, d); if (lane >= d) inc += o; }
      const unsigned total = __shfl_sync(0xFFFFFFFFu, inc, 31);
      s_cnt[2 * lane] = inc - a - b; s_cnt[2 * lane + 1] = inc - b;
      if (lane == 0 && total) s_base = atomicAdd(cursor, (unsigned long long)total);
    }
    __syncthreads();
    // output positions of this thread's rows (row order inside the tile)
    unsigned long long o[JP_ROWS];
#pragma unroll
    for (int r = 0; r < JP_ROWS; r++) o[r] = s_base + s_cnt[r * (JB / 32) + warp] + __popc(bal[r] & lt);
    // column by column: the eight loads of a column are issued back to back, then its eight stores
    for (int c = 0; c < pc.ncols; c++) {
      const GatherCol col = pc.col[c];
      if (col.width == 8) {
        unsigned long long v[JP_ROWS];
#pragma unroll
        for (int r = 0; r < JP_ROWS; r++) if (h[r] != 0xFFFFFFFEu) v[r] = ((const unsigned long long*)col.src)[t0 + r * JB + threadIdx.x];
#pragma unroll
        for (int r = 0; r < JP_ROWS; r++) if (h[r] != 0xFFFFFFFEu) ((unsigned long long*)col.out)[o[r]] = v[r];
      } else {
#pragma unroll
        for (int r = 0; r < JP_ROWS; r++) {
          if (h[r] == 0xFFFFFFFEu) continue;
          const long long i = t0 + r * JB + threadIdx.x;
          switch (col.width) {
            case 1: ((uint8_t*)col.out)[o[r]] = ((const uint8_t*)col.src)[i]; break;
            case 2: ((uint16_t*)col.out)[o[r]] = ((const uint16_t*)col.src)[i]; break;
            case 4: ((uint32_t*)col.out)[o[r]] = ((const uint32_t*)col.src)[i]; break;
            default: ((u128*)col.out)[o[r]] = ((const u128*)col.src)[i]; break;
          }
        }
      }
      if (col.out_valid) {
#pragma unroll
        for (int r = 0; r < JP_ROWS; r++) {
          if (h[r] == 0xFFFFFFFEu) continue;
          uint8_t ok = 1;
          if (col.vbits) { const unsigned long long bi = (unsigned long long)(t0 + r * JB + threadIdx.x) + col.bit_offset; ok = (col.vbits[bi >> 3] >> (bi & 7)) & 1; }
          col.out_valid[o[r]] = ok;
        }
      }
    }
    if (mark) {
#pragma unroll
      for (int r = 0; r < JP_ROWS; r++) if (h[r] < 0xFFFFFFFEu) mark[h[r]] = 1;
    }
    for (int c = 0; c < bc.ncols; c++) {
      const GatherCol col = bc.col[c];
      if (col.width == 8 && !col.vbytes) {
        unsigned long long v[JP_ROWS];
#pragma unroll
        for (int r = 0; r < JP_ROWS; r++) v[r] = h[r] < 0xFFFFFFFEu ? ((const unsigned long long*)col.src)[h[r]] : 0;
#pragma unroll
        for (int r = 0; r < JP_ROWS; r++) if (h[r] != 0xFFFFFFFEu) { ((unsigned long long*)col.out)[o[r]] = v[r]; if (col.out_valid) col.out_valid[o[r]] = h[r] != JOIN_NIL; }
      } else {
#pragma unroll
        for (int r = 0; r < JP_ROWS; r++) {
          if (h[r] == 0xFFFFFFFEu) continue;
          const uint32_t b = h[r];
          uint8_t ok = b != JOIN_NIL;
          if (ok && col.vbytes) ok = col.vbytes[b];
          switch (col.width) {
            case 1: ((uint8_t*)col.out)[o[r]] = ok ? ((const uint8_t*)col.src)[b] : 0; break;
            case 2: ((uint16_t*)col.out)[o[r]] = ok ? ((const uint16_t*)col.src)[b] : 0; break;
            case 4: ((uint32_t*)col.out)[o[r]] = ok ? ((const uint32_t*)col.src)[b] : 0; break;
            case 8: ((unsigned long long*)col.out)[o[r]] = ok ? ((const unsigned long long*)col.src)[b] : 0; break;
            default: { u128 v{0, 0}; if (ok) v = ((const u128*)col.src)[b]; ((u128*)col.out)[o[r]] = v; break; }
          }
          if (col.out_valid) col.out_valid[o[r]] = ok;
        }
      }
    }
    __syncthreads();
  }
}

__global__ void __launch_bounds__(JB) unpack_bits_kernel(const uint8_t* __restrict__ bits, uint32_t bit_offset, long long n, uint8_t* __restrict__ bytes) {
  for (long long i = blockIdx.x * (long long)JB + threadIdx.x; i < n; i += (long long)gridDim.x * JB) {
    const unsigned long long bi = (unsigned long long)i + bit_offset;
    bytes[i] = bits ? ((bits[bi >> 3] >> (bi & 7)) & 1) : 1;
  }
}

__global__ void __launch_bounds__(JB) join_flags_kernel(const uint32_t* __restrict__ head, long long n, int invert, int32_t* __restrict__ flags) {
  for (long long i = blockIdx.x * (long long)JB + threadIdx.x; i < n; i += (long long)gridDim.x * JB) flags[i] = ((head[i] != JOIN_NIL) ? 1 : 0) ^ invert;
}
__global__ void __launch_bounds__(JB) join_match_bytes_kernel(const uint32_t* __restrict__ head, long long n, uint8_t* __restrict__ bytes) {
  for (long long i = blockIdx.x * (long long)JB + threadIdx.x; i < n; i += (long long)gridDim.x * JB) bytes[i] = head[i] != JOIN_NIL;
}
__global__ void __launch_bounds__(JB) bytes_to_flags_kernel(const uint8_t* __restrict__ bytes, long long n, int invert, int32_t* __restrict__ flags) {
  for (long long i = blockIdx.x * (long long)JB + threadIdx.x; i < n; i += (long long)gridDim.x * JB) flags[i] = (bytes[i] ? 1 : 0) ^ invert;
}
__global__ void __launch_bounds__(JB) compact_indices_kernel(const int32_t* __restrict__ flags, const int32_t* __restrict__ offs, long long n, uint32_t* __restrict__ idx) {
  for (long long i = blockIdx.x * (long long)JB + threadIdx.x; i < n; i += (long long)gridDim.x * JB) if (flags[i]) idx[offs[i]] = (uint32_t)i;
}

}  // namespace

int launch_join_build(const JoinKeys& k, int64_t n, const JoinTable& t, cudaStream_t s) {
  if (n > 0) join_build_kernel<<<jgrid(n), JB, 0, s>>>(k, n, t);
  join_pack_kernel<<<jgrid((int64_t)t.mask + 1), JB, 0, s>>>(t);
  return n > 0 ? 2 : 1;
}
int launch_join_probe_count(const JoinKeys& k, int64_t n, const JoinTable& t, int probe_outer, uint32_t* d_head, int32_t* d_count, cudaStream_t s, unsigned long long* d_total) {
  if (n <= 0) return 0;
  join_probe_count_kernel<<<jgrid(n, JB * 8), JB, 0, s>>>(k, n, t, probe_outer, d_head, d_count, d_total);
  return 1;
}
int launch_join_probe_emit(int64_t n, const JoinTable& t, const uint32_t* d_head, const int32_t* d_offs, uint32_t* d_pidx, uint32_t* d_bidx, uint8_t* mark, cudaStream_t s) {
  if (n <= 0) return 0;
  join_probe_emit_kernel<<<jgrid(n), JB, 0, s>>>(n, t, d_head, d_offs, d_pidx, d_bidx, mark);
  return 1;
}
int launch_join_mark_build(int64_t n, const JoinTable& t, const uint32_t* d_head, uint8_t* mark, cudaStream_t s) {
  if (n <= 0) return 0;
  join_mark_build_kernel<<<jgrid(n), JB, 0, s>>>(n, t, d_head, mark);
  return 1;
}
int launch_join_probe_pairs(const JoinKeys& k, int64_t n, const JoinTable& t, int probe_outer, unsigned long long* d_cursor, uint32_t* d_pidx, uint32_t* d_bidx, uint8_t* mark, cudaStream_t s) {
  if (n <= 0) return 0;
  join_probe_pairs_kernel<<<jgrid(n, JB * JP_ROWS), JB, 0, s>>>(k, n, t, probe_outer, d_cursor, d_pidx, d_bidx, mark);
  return 1;
}
int launch_join_probe_select(const JoinKeys& k, int64_t n, const JoinTable& t, int invert, unsigned long long* d_cursor, uint32_t* d_idx, cudaStream_t s) {
  if (n <= 0) return 0;
  join_probe_select_kernel<<<jgrid(n), JB, 0, s>>>(k, n, t, invert, d_cursor, d_idx);
  return 1;
}
int launch_join_probe_mark(const JoinKeys& k, int64_t n, const JoinTable& t, uint8_t* mark, cudaStream_t s) {
  if (n <= 0) return 0;
  join_probe_mark_kernel<<<jgrid(n), JB, 0, s>>>(k, n, t, mark);
  return 1;
}
int launch_join_gather(const void* src, const uint8_t* vbits, uint32_t bit_offset, const uint8_t* vbytes, int width, const uint32_t* idx, int64_t n, void* out, uint8_t* out_valid, cudaStream_t s) {
  if (n <= 0) return 0;
  const int g = jgrid(n);
  switch (width) {
    case 1: join_gather_kernel<uint8_t><<<g, JB, 0, s>>>((const uint8_t*)src, vbits, bit_offset, vbytes, idx, n, (uint8_t*)out, out_valid); break;
    case 2: join_gather_kernel<uint16_t><<<g, JB, 0, s>>>((const uint16_t*)src, vbits, bit_offset, vbytes, idx, n, (uint16_t*)out, out_valid); break;
    case 4: join_gather_kernel<uint32_t><<<g, JB, 0, s>>>((const uint32_t*)src, vbits, bit_offset, vbytes, idx, n, (uint32_t*)out, out_valid); break;
    case 8: join_gather_kernel<unsigned long long><<<g, JB, 0, s>>>((const unsigned long long*)src, vbits, bit_offset, vbytes, idx, n, (unsigned long long*)out, out_valid); break;
    default: join_gather_kernel<u128><<<g, JB, 0, s>>>((const u128*)src, vbits, bit_offset, vbytes, idx, n, (u128*)out, out_valid); break;
  }
  return 1;
}
int launch_join_gather_multi(const GatherSpec& g, const uint32_t* idx, int64_t n, cudaStream_t s) {
  if (n <= 0 || g.ncols == 0) return 0;
  join_gather_multi_kernel<<<jgrid(n), JB, 0, s>>>(g, idx, n);
  return 1;
}
int launch_join_probe_fused(const uint32_t* d_head, int64_t n, int probe_outer, unsigned long long* d_cursor, const GatherSpec& probe_cols, const GatherSpec& build_cols,
                            uint8_t* mark, cudaStream_t s) {
  if (n <= 0) return 0;
  join_probe_fused_kernel<<<jgrid(n, JB * JP_ROWS), JB, 0, s>>>(d_head, n, probe_outer, d_cursor, probe_cols, build_cols, mark);
  return 1;
}
int launch_unpack_bits(const uint8_t* bits, uint32_t bit_offset, int64_t n, uint8_t* bytes, cudaStream_t s) {
  if (n <= 0) return 0;
  unpack_bits_kernel<<<jgrid(n), JB, 0, s>>>(bits, bit_offset, n, bytes);
  return 1;
}
int launch_join_flags(const uint32_t* d_head, int64_t n, int invert, int32_t* d_flags, cudaStream_t s) {
  if (n <= 0) return 0;
  join_flags_kernel<<<jgrid(n), JB, 0, s>>>(d_head, n, invert, d_flags);
  return 1;
}
int launch_join_match_bytes(const uint32_t* d_head, int64_t n, uint8_t* d_bytes, cudaStream_t s) {
  if (n <= 0) return 0;
  join_match_bytes_kernel<<<jgrid(n), JB, 0, s>>>(d_head, n, d_bytes);
  return 1;
}
int launch_bytes_to_flags(const uint8_t* bytes, int64_t n, int invert, int32_t* d_flags, cudaStream_t s) {
  if (n <= 0) return 0;
  bytes_to_flags_kernel<<<jgrid(n), JB, 0, s>>>(bytes, n, invert, d_flags);
  return 1;
}
int launch_join_compact_indices(const int32_t* d_flags, const int32_t* d_offs, int64_t n, uint32_t* d_idx, cudaStream_t s) {
  if (n <= 0) return 0;
  compact_indices_kernel<<<jgrid(n), JB, 0, s>>>(d_flags, d_offs, n, d_idx);
  return 1;
}

}  // namespace b200q
