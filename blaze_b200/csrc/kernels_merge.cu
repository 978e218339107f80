// SortMergeJoinExec on the GPU (smj_stage.cu drives these): both sides arrive sorted by the join keys, so the equal range of
// every left key in the right side comes from a MERGE of the two sorted key sequences instead of a hash table.
//
// Reference (datafusion-ext-plans/src/sort_merge_join_exec.rs, joins/smj/*.rs): two cursors walk the sides in key order,
// `compare_cursor!` (:357-365) skips keys with a NULL, equal runs are joined as a cartesian block, and a side that is not
// sorted gives wrong rows.  Here:
//   1. smj_normalise_kernel: per row, the order words of the keys (sort_normalise_word, the SortExec transform under the node's
//      sort_options) and one flag byte; the same pass compares every row with its predecessor, so unsorted input is refused.
//   2. smj_merge_kernel: merge path (Odeh et al., "Merge Path - Parallel Merging Made Simple", 2012).  The merged sequence of
//      the left batch and the relevant right rows is cut into tiles of M_TILE items; one diagonal search per tile boundary
//      finds how many items of each side come before it, the tile's keys are staged in shared memory once (coalesced), and
//      every item finds its rank in the other side's part of the tile there.  Run with ties going to the left row, a left
//      row's rank is its lower bound in the right side (and a right row's rank the left rows <= it); with ties going to the
//      right row, its upper bound.  One launch: the first half of the grid runs the first rule, the second half the other.
//   3. counts per left row, a 64-bit exclusive scan, and one emit pass writing (left row, right row | NIL) pairs in output order.
#include <cuda_runtime.h>
#include <stdint.h>

#include <algorithm>

#include "kernels_join.cuh"
#include "kernels_merge.cuh"

namespace b200q {

namespace {

constexpr int MB = 256, M_TILE = 2048, SC_ITEMS = 8, SC_TILE = MB * SC_ITEMS;

int mgrid(int64_t n, int per_block = MB * 4) {
  int dev = 0, sms = 132; cudaGetDevice(&dev); cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  return (int)std::max<int64_t>(1, std::min<int64_t>((n + per_block - 1) / per_block, (int64_t)sms * 8));
}

struct Key { unsigned long long w0, w1; uint32_t f; };

__device__ __forceinline__ Key load_key(const MergeKeys& k, long long i) {
  Key r; r.w0 = k.w0[i]; r.w1 = k.w1 ? k.w1[i] : 0; r.f = k.flags[i]; return r;
}
// the tuple (null rank 0, w0, null rank 1, w1): -1 / 0 / 1
__device__ __forceinline__ int key_cmp(const Key& a, const Key& b) {
  const unsigned an0 = a.f & 1, bn0 = b.f & 1;
  if (an0 != bn0) return an0 < bn0 ? -1 : 1;
  if (a.w0 != b.w0) return a.w0 < b.w0 ? -1 : 1;
  const unsigned an1 = (a.f >> 1) & 1, bn1 = (b.f >> 1) & 1;
  if (an1 != bn1) return an1 < bn1 ? -1 : 1;
  if (a.w1 != b.w1) return a.w1 < b.w1 ? -1 : 1;
  return 0;
}

struct NormArgs { SortKeyCol k[2]; int nkeys; };

__device__ __forceinline__ uint32_t null_rank(bool valid, uint8_t nulls_first) { return valid ? (nulls_first ? 1u : 0u) : (nulls_first ? 0u : 1u); }

__device__ __forceinline__ Key norm_row(const NormArgs& a, long long r) {
  Key o; bool v0 = true, v1 = true;
  o.w0 = sort_normalise_word(a.k[0], r, &v0);
  o.w1 = 0;
  uint32_t f = null_rank(v0, a.k[0].nulls_first);
  if (a.nkeys > 1) { o.w1 = sort_normalise_word(a.k[1], r, &v1); f |= null_rank(v1, a.k[1].nulls_first) << 1; }
  if (!v0 || !v1) f |= SMJ_ANY_NULL;
  o.f = f;
  return o;
}

__global__ void __launch_bounds__(MB) smj_normalise_kernel(const NormArgs a, long long n, unsigned long long* __restrict__ w0, unsigned long long* __restrict__ w1,
                                                           uint8_t* __restrict__ flags, const SmjCarry* __restrict__ carry, SmjStatus* st) {
  for (long long i = blockIdx.x * (long long)MB + threadIdx.x; i < n; i += (long long)gridDim.x * MB) {
    const Key k = norm_row(a, i);
    w0[i] = k.w0; if (w1) w1[i] = k.w1; flags[i] = (uint8_t)k.f;
    bool has_prev = i > 0; Key p;
    if (has_prev) p = norm_row(a, i - 1);                      // the neighbour's words are recomputed from its (cached) values
    else if (carry && carry->has) { p.w0 = carry->w0; p.w1 = carry->w1; p.f = carry->flags; has_prev = true; }
    if (has_prev && key_cmp(p, k) > 0) st->unsorted = 1;
  }
}

__global__ void smj_carry_kernel(const unsigned long long* w0, const unsigned long long* w1, const uint8_t* flags, long long n, SmjCarry* carry) {
  if (threadIdx.x == 0 && blockIdx.x == 0 && n > 0) { carry->w0 = w0[n - 1]; carry->w1 = w1 ? w1[n - 1] : 0; carry->flags = flags[n - 1]; carry->has = 1; }
}

// first right row in [0, m) whose key is >= k (upper: > k)
__device__ long long right_bound(const MergeKeys& right, long long m, const Key& k, bool upper) {
  long long a = 0, b = m;
  while (a < b) {
    const long long mid = (a + b) >> 1;
    const int c = key_cmp(load_key(right, mid), k);
    if (upper ? c <= 0 : c < 0) a = mid + 1; else b = mid;
  }
  return a;
}

__global__ void smj_bounds_kernel(const MergeKeys left, long long n, const MergeKeys right, long long m, SmjStatus* st) {
  if (threadIdx.x == 0) st->rb0 = (unsigned long long)right_bound(right, m, load_key(left, 0), false);
  if (threadIdx.x == 1) st->rb1 = (unsigned long long)right_bound(right, m, load_key(left, n - 1), true);
}

// blocks [0, ntiles): ties put the left row first -> lo (lower bounds) and pr; blocks [ntiles, 2 ntiles): ties put the right row
// first -> hi (upper bounds).  `right` starts at right row rb0 and holds m rows
__global__ void __launch_bounds__(MB) smj_merge_kernel(const MergeKeys left, long long n, const MergeKeys right, long long m, long long rb0, long long ntiles,
                                                       uint32_t* __restrict__ lo, uint32_t* __restrict__ hi, uint32_t* __restrict__ pr) {
  __shared__ unsigned long long s_w0[M_TILE], s_w1[M_TILE];
  __shared__ uint8_t s_f[M_TILE];
  __shared__ long long s_split[2];
  const bool upper = (long long)blockIdx.x >= ntiles;
  const long long d0 = ((long long)blockIdx.x - (upper ? ntiles : 0)) * M_TILE, d1 = min(d0 + (long long)M_TILE, n + m);
  if (threadIdx.x < 2) {                                       // diagonal search: left items among the first d merged items
    const long long d = threadIdx.x ? d1 : d0;
    long long a = max(0LL, d - m), b = min(d, n);
    while (a < b) {
      const long long mid = (a + b) >> 1;
      const int c = key_cmp(load_key(left, mid), load_key(right, d - 1 - mid));
      if (upper ? c < 0 : c <= 0) a = mid + 1; else b = mid;
    }
    s_split[threadIdx.x] = a;
  }
  __syncthreads();
  const long long a0 = s_split[0], a1 = s_split[1], b0 = d0 - a0;
  const int na = (int)(a1 - a0), nt = (int)(d1 - d0), nb = nt - na;
  for (int j = threadIdx.x; j < nt; j += MB) {                // left part of the tile, then its right part
    const Key k = j < na ? load_key(left, a0 + j) : load_key(right, b0 + (j - na));
    s_w0[j] = k.w0; s_w1[j] = k.w1; s_f[j] = (uint8_t)k.f;
  }
  __syncthreads();
  for (int j = threadIdx.x; j < nt; j += MB) {
    Key k; k.w0 = s_w0[j]; k.w1 = s_w1[j]; k.f = s_f[j];
    if (j < na) {                                              // right items of the tile before this left row
      int x = 0, y = nb;
      while (x < y) {
        const int mid = (x + y) >> 1;
        Key o; o.w0 = s_w0[na + mid]; o.w1 = s_w1[na + mid]; o.f = s_f[na + mid];
        const int c = key_cmp(o, k);
        if (upper ? c <= 0 : c < 0) x = mid + 1; else y = mid;
      }
      const uint32_t r = (uint32_t)(rb0 + b0 + x);
      if (upper) hi[a0 + j] = r; else lo[a0 + j] = r;
    } else if (!upper) {                                       // left items of the tile whose key is <= this right row's
      int x = 0, y = na;
      while (x < y) {
        const int mid = (x + y) >> 1;
        Key o; o.w0 = s_w0[mid]; o.w1 = s_w1[mid]; o.f = s_f[mid];
        if (key_cmp(o, k) <= 0) x = mid + 1; else y = mid;
      }
      pr[b0 + (j - na)] = (uint32_t)(a0 + x);
    }
  }
}

enum { JT_INNER = 0, JT_LEFT, JT_RIGHT, JT_FULL, JT_SEMI, JT_ANTI, JT_EXISTENCE };

__global__ void __launch_bounds__(MB) smj_counts_kernel(const uint8_t* __restrict__ lflags, long long n, const uint32_t* __restrict__ lo, const uint32_t* __restrict__ hi,
                                                        int jt, unsigned long long* __restrict__ counts) {
  for (long long i = blockIdx.x * (long long)MB + threadIdx.x; i < n; i += (long long)gridDim.x * MB) {
    const unsigned long long k = (lflags[i] & SMJ_ANY_NULL) ? 0 : (unsigned long long)(hi[i] - lo[i]);
    unsigned long long c;
    switch (jt) {
      case JT_LEFT: case JT_FULL: c = k ? k : 1; break;
      case JT_SEMI: c = k ? 1 : 0; break;
      case JT_ANTI: c = k ? 0 : 1; break;
      case JT_EXISTENCE: c = 1; break;
      default: c = k;
    }
    counts[i] = c;
  }
}

__global__ void __launch_bounds__(MB) smj_mark_kernel(const MergeKeys left, const MergeKeys right, long long rb0, long long rb1, const uint32_t* __restrict__ pr, uint8_t* __restrict__ matched) {
  for (long long r = rb0 + blockIdx.x * (long long)MB + threadIdx.x; r < rb1; r += (long long)gridDim.x * MB) {
    if (right.flags[r] & SMJ_ANY_NULL) continue;
    const uint32_t p = pr[r - rb0];                            // left rows with a key <= this row's: the last of them may be equal
    if (p > 0 && key_cmp(load_key(left, (long long)p - 1), load_key(right, r)) == 0) matched[r] = 1;
  }
}

__global__ void __launch_bounds__(MB) smj_unmatched_kernel(const uint8_t* __restrict__ matched, long long s0, long long nw, unsigned long long* __restrict__ flags) {
  for (long long w = blockIdx.x * (long long)MB + threadIdx.x; w < nw; w += (long long)gridDim.x * MB) flags[w] = matched[s0 + w] ? 0 : 1;
}

// exclusive scan of one value per thread over the block (every thread of the block calls it); *total = the block's sum
__device__ unsigned long long block_exclusive_scan(unsigned long long v, unsigned long long* total) {
  __shared__ unsigned long long s_warp[32], s_total;
  const unsigned lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = (blockDim.x + 31) >> 5;
  unsigned long long inc = v;
  for (unsigned o = 1; o < 32; o <<= 1) { const unsigned long long y = __shfl_up_sync(0xFFFFFFFFu, inc, o); if (lane >= o) inc += y; }
  if (lane == 31) s_warp[warp] = inc;
  __syncthreads();
  if (warp == 0) {
    const unsigned long long x = lane < nwarps ? s_warp[lane] : 0;
    unsigned long long xi = x;
    for (unsigned o = 1; o < 32; o <<= 1) { const unsigned long long y = __shfl_up_sync(0xFFFFFFFFu, xi, o); if (lane >= o) xi += y; }
    __syncwarp();
    s_warp[lane] = xi - x;                                     // exclusive prefix of the warp sums
    if (lane == 31) s_total = xi;
  }
  __syncthreads();
  const unsigned long long res = s_warp[warp] + inc - v;
  *total = s_total;
  __syncthreads();
  return res;
}

__global__ void __launch_bounds__(MB) smj_scan_reduce_kernel(const unsigned long long* __restrict__ in, long long n, unsigned long long* __restrict__ sums) {
  const long long t0 = (long long)blockIdx.x * SC_TILE;
  unsigned long long v = 0;
  for (int j = threadIdx.x; j < SC_TILE; j += MB) if (t0 + j < n) v += in[t0 + j];
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xFFFFFFFFu, v, o);
  __shared__ unsigned long long s[MB / 32];
  if ((threadIdx.x & 31) == 0) s[threadIdx.x >> 5] = v;
  __syncthreads();
  if (threadIdx.x == 0) { unsigned long long t = 0; for (int w = 0; w < MB / 32; w++) t += s[w]; sums[blockIdx.x] = t; }
}

// one block of MB threads: sums[0..nb) -> their exclusive scan in place, sums[nb] = total
__global__ void __launch_bounds__(MB) smj_scan_blocks_kernel(unsigned long long* sums, long long nb) {
  __shared__ unsigned long long s_carry;
  if (threadIdx.x == 0) s_carry = 0;
  __syncthreads();
  for (long long c0 = 0; c0 < nb; c0 += MB) {
    const long long i = c0 + threadIdx.x;
    const unsigned long long v = i < nb ? sums[i] : 0;
    unsigned long long total;
    const unsigned long long ex = block_exclusive_scan(v, &total);
    const unsigned long long carry = s_carry;
    if (i < nb) sums[i] = carry + ex;
    __syncthreads();
    if (threadIdx.x == 0) s_carry = carry + total;
    __syncthreads();
  }
  if (threadIdx.x == 0) sums[nb] = s_carry;
}

__global__ void __launch_bounds__(MB) smj_scan_apply_kernel(const unsigned long long* __restrict__ in, long long n, const unsigned long long* __restrict__ sums, long long nb,
                                                            unsigned long long* __restrict__ out) {
  const long long t0 = (long long)blockIdx.x * SC_TILE + (long long)threadIdx.x * SC_ITEMS;
  unsigned long long v[SC_ITEMS], s = 0;
#pragma unroll
  for (int j = 0; j < SC_ITEMS; j++) { v[j] = t0 + j < n ? in[t0 + j] : 0; s += v[j]; }
  unsigned long long total;
  unsigned long long run = sums[blockIdx.x] + block_exclusive_scan(s, &total);
#pragma unroll
  for (int j = 0; j < SC_ITEMS; j++) { if (t0 + j < n) out[t0 + j] = run; run += v[j]; }
  if (blockIdx.x == 0 && threadIdx.x == 0) out[n] = sums[nb];
}

__global__ void __launch_bounds__(MB) smj_emit_kernel(const SmjEmit e) {
  const long long total = e.n + e.nw;
  for (long long i = blockIdx.x * (long long)MB + threadIdx.x; i < total; i += (long long)gridDim.x * MB) {
    if (i < e.n) {
      const unsigned long long lo = e.lo[i];
      const long long start = (long long)(e.L[i] + (e.U ? e.U[(long long)lo - e.s0] : 0));
      const long long cnt = (long long)(e.L[i + 1] - e.L[i]);
      const long long k = (e.lflags[i] & SMJ_ANY_NULL) ? 0 : (long long)(e.hi[i] - lo);
      const long long jb = max(0LL, e.o0 - start), je = min(cnt, e.o1 - start);
      for (long long j = jb; j < je; j++) {
        const long long o = start + j - e.o0;
        e.pidx[o] = (uint32_t)i;
        if (e.bidx) e.bidx[o] = k ? (uint32_t)(lo + j) : JOIN_NIL;
        if (e.exists) e.exists[o] = k > 0;
      }
    } else {
      const long long w = i - e.n, r = e.s0 + w;
      if (e.matched[r]) continue;
      const long long p = r < e.rb0 ? 0 : (long long)e.pr[r - e.rb0];
      const long long o = (long long)(e.L[p] + e.U[w]);
      if (o >= e.o0 && o < e.o1) { e.pidx[o - e.o0] = JOIN_NIL; e.bidx[o - e.o0] = (uint32_t)r; }
    }
  }
}

}  // namespace

int launch_smj_normalise(const SortKeyCol* keys, int nkeys, int64_t n, unsigned long long* w0, unsigned long long* w1, uint8_t* flags,
                         SmjCarry* d_carry, SmjStatus* d_status, cudaStream_t s) {
  if (n <= 0) return 0;
  NormArgs a{}; a.nkeys = nkeys;
  for (int i = 0; i < nkeys; i++) a.k[i] = keys[i];
  smj_normalise_kernel<<<mgrid(n), MB, 0, s>>>(a, n, w0, nkeys > 1 ? w1 : nullptr, flags, d_carry, d_status);
  if (!d_carry) return 1;
  smj_carry_kernel<<<1, 32, 0, s>>>(w0, nkeys > 1 ? w1 : nullptr, flags, n, d_carry);
  return 2;
}
int launch_smj_bounds(const MergeKeys& left, int64_t n, const MergeKeys& right, int64_t m, SmjStatus* d_status, cudaStream_t s) {
  if (n <= 0) return 0;
  smj_bounds_kernel<<<1, 32, 0, s>>>(left, n, right, m, d_status);
  return 1;
}
int launch_smj_merge(const MergeKeys& left, int64_t n, const MergeKeys& right, int64_t rb0, int64_t rb1, uint32_t* lo, uint32_t* hi, uint32_t* pr, cudaStream_t s) {
  if (n <= 0) return 0;
  MergeKeys r = right;                                         // the merged right part starts at rb0
  r.w0 += rb0; if (r.w1) r.w1 += rb0; r.flags += rb0;
  const int64_t m = rb1 - rb0, ntiles = (n + m + M_TILE - 1) / M_TILE;
  smj_merge_kernel<<<(unsigned)(2 * ntiles), MB, 0, s>>>(left, n, r, m, rb0, ntiles, lo, hi, pr);
  return 1;
}
int launch_smj_counts(const MergeKeys& left, int64_t n, const uint32_t* lo, const uint32_t* hi, int join_type, unsigned long long* counts, cudaStream_t s) {
  if (n <= 0) return 0;
  smj_counts_kernel<<<mgrid(n), MB, 0, s>>>(left.flags, n, lo, hi, join_type, counts);
  return 1;
}
int launch_smj_mark(const MergeKeys& left, const MergeKeys& right, int64_t rb0, int64_t rb1, const uint32_t* pr, uint8_t* matched, cudaStream_t s) {
  if (rb1 <= rb0) return 0;
  smj_mark_kernel<<<mgrid(rb1 - rb0), MB, 0, s>>>(left, right, rb0, rb1, pr, matched);
  return 1;
}
int launch_smj_unmatched(const uint8_t* matched, int64_t s0, int64_t nw, unsigned long long* flags, cudaStream_t s) {
  if (nw <= 0) return 0;
  smj_unmatched_kernel<<<mgrid(nw), MB, 0, s>>>(matched, s0, nw, flags);
  return 1;
}
int64_t smj_scan_tmp_words(int64_t n) { return (n + SC_TILE - 1) / SC_TILE + 1; }
int launch_smj_scan(const unsigned long long* in, unsigned long long* out, int64_t n, unsigned long long* d_tmp, cudaStream_t s) {
  if (n <= 0) { cudaMemsetAsync(out, 0, 8, s); return 0; }
  const int64_t nb = (n + SC_TILE - 1) / SC_TILE;
  smj_scan_reduce_kernel<<<(unsigned)nb, MB, 0, s>>>(in, n, d_tmp);
  smj_scan_blocks_kernel<<<1, MB, 0, s>>>(d_tmp, nb);
  smj_scan_apply_kernel<<<(unsigned)nb, MB, 0, s>>>(in, n, d_tmp, nb, out);
  return 3;
}
int launch_smj_emit(const SmjEmit& e, cudaStream_t s) {
  if (e.n + e.nw <= 0 || e.o1 <= e.o0) return 0;
  smj_emit_kernel<<<mgrid(e.n + e.nw), MB, 0, s>>>(e);
  return 1;
}

}  // namespace b200q
