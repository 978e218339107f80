// Microbenchmark: the streaming front end of the tile HashAgg kernels (kernels_tile.cu) on 4 int64 columns of 2^28 rows
// (32 B/row, the M2 row shape).  Decides the row-to-lane mapping, the prefetch depth and whether reading the key / value
// columns only for the rows that pass the filter pays, and whether bucketing the survivors beats their REDs (DESIGN §3.1).
// Build: nvcc -O3 -std=c++17 -gencode arch=compute_90a,code=sm_90a -o tile_stream tile_stream.cu -L/usr/local/cuda/lib64/stubs -lnvidia-ml
// Run:   tile_stream [rows] [part]      (part: only section 5)
//   shapes   a: lane owns 4 consecutive rows, two 128-bit loads per column (32-byte lane stride)
//            b: lane-contiguous 128-bit loads (rows 2l, 2l+1 and 64+2l, 64+2l+1 of a 128-row tile)
//            c: 8-byte loads, lane l holds rows l + 32 j
//            d: cp.async 16-byte copies of the tile into shared memory, read back as c
//   policies plain, L2::evict_first (createpolicy + cache_hint), L2::128B / L2::256B prefetch qualifiers
//   depth    tiles whose loads are issued before the current tile is consumed (0: load, wait, consume)
//   modes    all: every column read for every row; skip: f read in full, k1 k2 v only for rows with f in range
//            (+red: the surviving rows add v into a table of 2 words an entry, one RED a word)
//            (+part: the surviving rows become 8-byte tuples {entry index, value} that a CTA stages in shared memory,
//             counting-sorts by bucket (a range of 2^shift entries) and appends as one run per bucket to that bucket's
//             region of a spill area; bucket_reduce_kernel then adds each bucket into its slice of the table in shared
//             memory, one CTA per bucket; a tuple whose bucket region is full takes the REDs)
//   tables   compact: k1 * 8 + k2 (2^20 entries, 16 MB); padded: k1 * 20 + k2 over 163968 x 20 = 3,279,360 entries (52 MB,
//            a third of it live), the layout dense_range gives M2
#include <cstdio>
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <vector>
#include <cuda_runtime.h>
#include <nvml.h>
#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("CUDA %s @%d\n", cudaGetErrorString(e), __LINE__); exit(1); } } while (0)

enum { SH_A = 0, SH_B, SH_C, SH_D };
enum { P_NONE = 0, P_EVICT, P_128, P_256 };
enum { M_ALL = 0, M_SKIP, M_ALL_RED, M_SKIP_RED, M_SKIP_PART };
constexpr unsigned long long PAD_ENTRIES = 163968ULL * 20;
constexpr int ROWS = 128, WARPS = 8, NCOL = 4;

__device__ __forceinline__ uint64_t mix(uint64_t x) { x ^= x >> 33; x *= 0xff51afd7ed558ccdULL; x ^= x >> 33; x *= 0xc4ceb9fe1a85ec53ULL; x ^= x >> 33; return x; }
// f uniform in [0, 1000) per row, or per run of 8 rows; k1 < 2^17, k2 < 8 (dense index k1 * 8 + k2 < 2^20)
__global__ void gen(long long* f, long long* k1, long long* k2, long long* v, size_t n, int runs) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const uint64_t h = mix(i * 0x9E3779B97F4A7C15ULL + 12345);
    f[i] = (long long)(mix((runs ? i / 8 : i) + 777) % 1000); k1[i] = (long long)(h & 0x1FFFF); k2[i] = (long long)((h >> 20) & 7); v[i] = (long long)((h >> 24) % 2000001) - 1000000;
  }
}
// sectors of 4 rows (32 B of an int64 column) and pairs of 8 rows (64 B) that hold a row with f in [lo, hi]
__global__ void count_sectors(const long long* f, size_t n, long long lo, long long hi, unsigned long long* out) {
  unsigned long long s32 = 0, s64 = 0;
  for (size_t g = blockIdx.x * (size_t)blockDim.x + threadIdx.x; g < n / 8; g += (size_t)gridDim.x * blockDim.x) {
    bool a = false, b = false;
    for (int r = 0; r < 4; r++) { a |= f[8 * g + r] >= lo && f[8 * g + r] <= hi; b |= f[8 * g + 4 + r] >= lo && f[8 * g + 4 + r] <= hi; }
    s32 += a + b; s64 += a || b;
  }
  atomicAdd(out, s32); atomicAdd(out + 1, s64);
}

template <int POL> __device__ __forceinline__ void ld2(const long long* p, uint64_t pol, long long& a, long long& b) {
  if (POL == P_NONE) asm volatile("ld.global.nc.L1::no_allocate.v2.b64 {%0,%1}, [%2];" : "=l"(a), "=l"(b) : "l"(p));
  if (POL == P_EVICT) asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.v2.b64 {%0,%1}, [%2], %3;" : "=l"(a), "=l"(b) : "l"(p), "l"(pol));
  if (POL == P_128) asm volatile("ld.global.nc.L1::no_allocate.L2::128B.v2.b64 {%0,%1}, [%2];" : "=l"(a), "=l"(b) : "l"(p));
  if (POL == P_256) asm volatile("ld.global.nc.L1::no_allocate.L2::256B.v2.b64 {%0,%1}, [%2];" : "=l"(a), "=l"(b) : "l"(p));
}
template <int POL> __device__ __forceinline__ void ld1(const long long* p, unsigned on, uint64_t pol, long long& a) {
  if (POL == P_NONE) asm volatile("{\n\t.reg .pred q;\n\tsetp.ne.u32 q, %2, 0;\n\t@q ld.global.nc.L1::no_allocate.b64 %0, [%1];\n\t}" : "+l"(a) : "l"(p), "r"(on));
  if (POL == P_EVICT) asm volatile("{\n\t.reg .pred q;\n\tsetp.ne.u32 q, %2, 0;\n\t@q ld.global.nc.L1::no_allocate.L2::cache_hint.b64 %0, [%1], %3;\n\t}" : "+l"(a) : "l"(p), "r"(on), "l"(pol));
  if (POL == P_128) asm volatile("{\n\t.reg .pred q;\n\tsetp.ne.u32 q, %2, 0;\n\t@q ld.global.nc.L1::no_allocate.L2::128B.b64 %0, [%1];\n\t}" : "+l"(a) : "l"(p), "r"(on));
  if (POL == P_256) asm volatile("{\n\t.reg .pred q;\n\tsetp.ne.u32 q, %2, 0;\n\t@q ld.global.nc.L1::no_allocate.L2::256B.b64 %0, [%1];\n\t}" : "+l"(a) : "l"(p), "r"(on));
}
template <int POL> __device__ __forceinline__ void cpa16(void* s, const void* g, uint64_t pol) {
  const unsigned sa = (unsigned)__cvta_generic_to_shared(s);
  if (POL == P_NONE) asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" :: "r"(sa), "l"(g));
  if (POL == P_EVICT) asm volatile("cp.async.cg.shared.global.L2::cache_hint [%0], [%1], 16, %2;" :: "r"(sa), "l"(g), "l"(pol));
  if (POL == P_128) asm volatile("cp.async.cg.shared.global.L2::128B [%0], [%1], 16;" :: "r"(sa), "l"(g));
  if (POL == P_256) asm volatile("cp.async.cg.shared.global.L2::256B [%0], [%1], 16;" :: "r"(sa), "l"(g));
}

struct Cols { const long long* c[NCOL]; };                          // f, k1, k2, v

// one column of one tile in the mapping of SHAPE (a, b, c): v[j] is row rowof(j) of the tile
template <int SHAPE, int POL> __device__ __forceinline__ void load_col(const long long* p, unsigned lane, uint64_t pol, long long (&v)[4]) {
  if (SHAPE == SH_A) { ld2<POL>(p + 4 * lane, pol, v[0], v[1]); ld2<POL>(p + 4 * lane + 2, pol, v[2], v[3]); }
  if (SHAPE == SH_B) { ld2<POL>(p + 2 * lane, pol, v[0], v[1]); ld2<POL>(p + 64 + 2 * lane, pol, v[2], v[3]); }
  if (SHAPE == SH_C) { for (int j = 0; j < 4; j++) { v[j] = 0; ld1<POL>(p + lane + 32 * j, 1u, pol, v[j]); } }
}

template <int PAD> __device__ __forceinline__ unsigned long long entry_of(long long k1, long long k2) {
  return PAD ? (unsigned long long)k1 * 20 + (unsigned long long)k2 : ((unsigned long long)k1 * 8 + (unsigned long long)k2) & 0xFFFFF;
}

template <int MODE, int PAD = 0> __device__ __forceinline__ void consume(const long long (&f)[4], const long long (&k1)[4], const long long (&k2)[4], const long long (&v)[4], unsigned pass,
                                                        unsigned long long* tab, unsigned long long& acc) {
#pragma unroll
  for (int j = 0; j < 4; j++) {
    const bool on = MODE == M_ALL ? true : ((pass >> j) & 1u);
    if (MODE == M_ALL_RED || MODE == M_SKIP_RED) {
      if (on) { unsigned long long* e = tab + 2 * entry_of<PAD>(k1[j], k2[j]);
                asm volatile("red.global.add.u64 [%0], %1;" :: "l"(e), "l"(v[j]) : "memory"); asm volatile("red.global.add.u64 [%0], %1;" :: "l"(e + 1), "l"(1ULL) : "memory"); }
    } else acc += on ? (unsigned long long)(f[j] ^ k1[j] ^ k2[j] ^ v[j]) : 0ULL;
  }
}

// register-pipelined shapes a, b, c: the loads of tile t + DEPTH are issued before tile t is consumed
template <int SHAPE, int POL, int DEPTH, int MODE, int PAD = 0>
__global__ void __launch_bounds__(256) stream_kernel(Cols cs, long long ntiles, long long lo, unsigned long long span, unsigned long long* tab, unsigned long long* sink) {
  constexpr bool SKIP = MODE == M_SKIP || MODE == M_SKIP_RED;
  constexpr int NB = SKIP ? 1 : NCOL;                               // columns that are pipelined (skip: only f)
  const unsigned lane = threadIdx.x & 31;
  const long long gwarp = (long long)blockIdx.x * WARPS + (threadIdx.x >> 5), nwarps = (long long)gridDim.x * WARPS;
  uint64_t pol = 0; if (POL == P_EVICT) asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
  long long buf[DEPTH + 1][NB][4];
  unsigned long long acc = 0;
#pragma unroll
  for (int d = 0; d < DEPTH; d++) {
    const long long t = gwarp + d * nwarps;
#pragma unroll
    for (int c = 0; c < NB; c++) { for (int j = 0; j < 4; j++) buf[d][c][j] = 0; if (t < ntiles) load_col<SHAPE, POL>(cs.c[c] + t * ROWS, lane, pol, buf[d][c]); }
  }
  for (long long t = gwarp; t < ntiles; t += nwarps) {
    const long long tn = t + DEPTH * nwarps;
#pragma unroll
    for (int c = 0; c < NB; c++) { for (int j = 0; j < 4; j++) buf[DEPTH][c][j] = 0; if (tn < ntiles) load_col<SHAPE, POL>(cs.c[c] + tn * ROWS, lane, pol, buf[DEPTH][c]); }
    unsigned pass = 0;
#pragma unroll
    for (int j = 0; j < 4; j++) pass |= (unsigned)((unsigned long long)(buf[0][0][j] - lo) <= span) << j;
    if (SKIP) {                                                     // shape c only: rows lane + 32 j
      long long k1[4], k2[4], v[4];
#pragma unroll
      for (int j = 0; j < 4; j++) {
        k1[j] = k2[j] = v[j] = 0; const long long r = t * ROWS + lane + 32 * j; const unsigned on = (pass >> j) & 1u;
        ld1<POL>(cs.c[1] + r, on, pol, k1[j]); ld1<POL>(cs.c[2] + r, on, pol, k2[j]); ld1<POL>(cs.c[3] + r, on, pol, v[j]);
      }
      consume<MODE, PAD>(buf[0][0], k1, k2, v, pass, tab, acc);
    } else consume<MODE>(buf[0][0], buf[0][NB > 1 ? 1 : 0], buf[0][NB > 2 ? 2 : 0], buf[0][NB > 3 ? 3 : 0], pass, tab, acc);
#pragma unroll
    for (int d = 0; d < DEPTH; d++)
#pragma unroll
      for (int c = 0; c < NB; c++)
#pragma unroll
        for (int j = 0; j < 4; j++) buf[d][c][j] = buf[d + 1][c][j];
  }
  if (acc == 0x123456789ULL) sink[0] = acc;
}

// shape d: cp.async ring of DEPTH + 1 tiles per warp in shared memory (4 columns x 128 rows x 8 B = 4 KB a tile)
template <int POL, int DEPTH, int MODE>
__global__ void __launch_bounds__(256) cpasync_kernel(Cols cs, long long ntiles, long long lo, unsigned long long span, unsigned long long* tab, unsigned long long* sink) {
  extern __shared__ long long smem[];
  const unsigned lane = threadIdx.x & 31;
  long long* ring = smem + (threadIdx.x >> 5) * (DEPTH + 1) * NCOL * ROWS;
  const long long gwarp = (long long)blockIdx.x * WARPS + (threadIdx.x >> 5), nwarps = (long long)gridDim.x * WARPS;
  uint64_t pol = 0; if (POL == P_EVICT) asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
  auto issue = [&](long long t, int stage) {
    if (t < ntiles)
      for (int c = 0; c < NCOL; c++)
        for (int i = 0; i < 2; i++) { const int ch = lane + 32 * i; cpa16<POL>(ring + (stage * NCOL + c) * ROWS + 2 * ch, cs.c[c] + t * ROWS + 2 * ch, pol); }
    asm volatile("cp.async.commit_group;");
  };
  unsigned long long acc = 0;
  for (int d = 0; d < DEPTH; d++) issue(gwarp + d * nwarps, d);
  int stage = 0;
  for (long long t = gwarp; t < ntiles; t += nwarps) {
    issue(t + DEPTH * nwarps, (stage + DEPTH) % (DEPTH + 1));
    asm volatile("cp.async.wait_group %0;" :: "n"(DEPTH));
    __syncwarp();
    long long x[NCOL][4];
    for (int c = 0; c < NCOL; c++) for (int j = 0; j < 4; j++) x[c][j] = ring[(stage * NCOL + c) * ROWS + lane + 32 * j];
    unsigned pass = 0;
    for (int j = 0; j < 4; j++) pass |= (unsigned)((unsigned long long)(x[0][j] - lo) <= span) << j;
    consume<MODE>(x[0], x[1], x[2], x[3], pass, tab, acc);
    __syncwarp();
    stage = (stage + 1) % (DEPTH + 1);
  }
  asm volatile("cp.async.wait_all;");
  if (acc == 0x123456789ULL) sink[0] = acc;
}

// skip+part: the filter-first stream of shape c (evict_first, the next tile's f in flight); the warps of a CTA walk their tiles
// in lockstep so that the CTA can flush its staging area between two rounds
struct Part {
  unsigned long long* spill;    // nb regions of cap tuples
  unsigned* cursor;             // nb append cursors (they may run past cap: those tuples took the direct RED)
  unsigned cap;
  int shift, idx_bits, nb, stage;
};
constexpr int PART_NB_MAX = 1024;

__device__ __forceinline__ void red_pair(unsigned long long* tab, unsigned long long e, long long v) {
  asm volatile("red.global.add.u64 [%0], %1;" :: "l"(tab + 2 * e), "l"(v) : "memory"); asm volatile("red.global.add.u64 [%0], %1;" :: "l"(tab + 2 * e + 1), "l"(1ULL) : "memory");
}

// counting sort of the n staged tuples by bucket, one global reservation per (flush, bucket), one contiguous run per bucket
__device__ void part_flush(const Part& p, unsigned long long* tab, const unsigned long long* stage, uint16_t* order, unsigned* s_cnt, unsigned* s_off, unsigned* s_dst,
                           unsigned* s_warp, unsigned n) {
  const unsigned t = threadIdx.x; const unsigned long long imask = (1ULL << p.idx_bits) - 1;
  for (unsigned i = t; i < n; i += 256) atomicAdd(&s_cnt[(unsigned)((stage[i] & imask) >> p.shift)], 1u);
  __syncthreads();
  constexpr int K = PART_NB_MAX / 256;                               // buckets t*K .. t*K + K - 1
  unsigned c[K], sum = 0;
#pragma unroll
  for (int k = 0; k < K; k++) { c[k] = t * K + k < (unsigned)p.nb ? s_cnt[t * K + k] : 0u; sum += c[k]; }
  unsigned x = sum;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) { const unsigned y = __shfl_up_sync(0xffffffffu, x, o); if ((t & 31) >= (unsigned)o) x += y; }
  if ((t & 31) == 31) s_warp[t >> 5] = x;
  __syncthreads();
  unsigned before = x - sum;
  for (unsigned w = 0; w < (t >> 5); w++) before += s_warp[w];
#pragma unroll
  for (int k = 0; k < K; k++) if (t * K + k < (unsigned)p.nb) {
    s_off[t * K + k] = before; s_dst[t * K + k] = c[k] ? atomicAdd(&p.cursor[t * K + k], c[k]) : 0u; before += c[k];
  }
  __syncthreads();
  for (unsigned i = t; i < n; i += 256) order[atomicAdd(&s_off[(unsigned)((stage[i] & imask) >> p.shift)], 1u)] = (uint16_t)i;
  __syncthreads();
  for (unsigned i = t; i < n; i += 256) {
    const unsigned long long v = stage[order[i]]; const unsigned b = (unsigned)((v & imask) >> p.shift);
    const unsigned at = s_dst[b] + (i - (s_off[b] - s_cnt[b]));
    if (at < p.cap) p.spill[(size_t)b * p.cap + at] = v;
    else red_pair(tab, v & imask, (long long)v >> p.idx_bits);        // bucket region full
  }
  __syncthreads();
  for (unsigned b = t; b < (unsigned)p.nb; b += 256) s_cnt[b] = 0;
}

template <int PAD>
__global__ void __launch_bounds__(256) part_kernel(Cols cs, long long ntiles, long long lo, unsigned long long span, unsigned long long* tab, Part p) {
  extern __shared__ unsigned long long psmem[];
  unsigned long long* stage = psmem;                                 // p.stage tuples in arrival order
  unsigned* s_cnt = (unsigned*)(stage + p.stage); unsigned* s_off = s_cnt + p.nb; unsigned* s_dst = s_off + p.nb;
  uint16_t* order = (uint16_t*)(s_dst + p.nb);                      // their positions in bucket order
  __shared__ unsigned s_warp[WARPS], s_n;
  const unsigned lane = threadIdx.x & 31, t = threadIdx.x;
  const long long nwarps = (long long)gridDim.x * WARPS;
  const uint64_t pol = [] { uint64_t q; asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(q)); return q; }();
  const long long vmax = (1LL << (63 - p.idx_bits)) - 1;
  for (unsigned b = t; b < (unsigned)p.nb; b += 256) s_cnt[b] = 0;
  if (t == 0) s_n = 0;
  __syncthreads();
  long long f[4];
  const long long t0 = (long long)blockIdx.x * WARPS + (t >> 5);
  for (int j = 0; j < 4; j++) { f[j] = 0; ld1<P_EVICT>(cs.c[0] + t0 * ROWS + lane + 32 * j, t0 < ntiles, pol, f[j]); }
  for (long long round = (long long)blockIdx.x * WARPS; round < ntiles; round += nwarps) {
    const long long tile = round + (t >> 5), tn = tile + nwarps;
    unsigned pass = 0;
#pragma unroll
    for (int j = 0; j < 4; j++) pass |= (unsigned)(tile < ntiles && (unsigned long long)(f[j] - lo) <= span) << j;
    long long k1[4], k2[4], v[4];
#pragma unroll
    for (int j = 0; j < 4; j++) {
      k1[j] = k2[j] = v[j] = 0; const long long r = tile * ROWS + lane + 32 * j; const unsigned on = (pass >> j) & 1u;
      ld1<P_EVICT>(cs.c[1] + r, on, pol, k1[j]); ld1<P_EVICT>(cs.c[2] + r, on, pol, k2[j]); ld1<P_EVICT>(cs.c[3] + r, on, pol, v[j]);
    }
#pragma unroll
    for (int j = 0; j < 4; j++) { f[j] = 0; ld1<P_EVICT>(cs.c[0] + tn * ROWS + lane + 32 * j, tn < ntiles, pol, f[j]); }
    unsigned m[4]; unsigned tot = 0;
#pragma unroll
    for (int j = 0; j < 4; j++) {
      const bool on = (pass >> j) & 1u, fits = v[j] >= -vmax - 1 && v[j] <= vmax;
      if (on && !fits) red_pair(tab, entry_of<PAD>(k1[j], k2[j]), v[j]);
      m[j] = __ballot_sync(0xffffffffu, on && fits); tot += __popc(m[j]);
    }
    unsigned base = 0;
    if (lane == 0 && tot) base = atomicAdd(&s_n, tot);
    base = __shfl_sync(0xffffffffu, base, 0);
#pragma unroll
    for (int j = 0; j < 4; j++) {
      if ((m[j] >> lane) & 1u) stage[base + __popc(m[j] & ((1u << lane) - 1))] = entry_of<PAD>(k1[j], k2[j]) | ((unsigned long long)v[j] << p.idx_bits);
      base += __popc(m[j]);
    }
    // the warp whose run ends last knows the fill level; s_n itself may already be bumped by a warp of the next round
    if (__syncthreads_or(lane == 0 && base > (unsigned)p.stage - WARPS * ROWS) || round + nwarps >= ntiles) {
      part_flush(p, tab, stage, order, s_cnt, s_off, s_dst, s_warp, s_n);
      if (t == 0) s_n = 0;
      __syncthreads();
    }
  }
}

// one CTA per bucket: the bucket's 2^shift entries in shared memory ({count, sum low 32, sum high 32} as 32-bit words: a 64-bit
// shared atomicAdd is a CAS loop on sm_90a), its tuples added with shared atomics, the touched entries added into the table
__global__ void __launch_bounds__(1024) bucket_reduce_kernel(Part p, unsigned long long* tab, unsigned long long nent) {
  extern __shared__ unsigned rsmem[];
  const unsigned E = 1u << p.shift, b = blockIdx.x, t = threadIdx.x;
  unsigned* cnt = rsmem; unsigned* lo = cnt + E; unsigned* hi = lo + E;
  for (unsigned i = t; i < 3 * E; i += blockDim.x) rsmem[i] = 0;
  const unsigned n = min(p.cursor[b], p.cap);
  __syncthreads();
  const unsigned long long* in = p.spill + (size_t)b * p.cap; const unsigned long long imask = (1ULL << p.idx_bits) - 1;
  for (unsigned i = t; i < n; i += blockDim.x) {
    const unsigned long long x = in[i]; const unsigned e = (unsigned)(x & imask) & (E - 1); const long long v = (long long)x >> p.idx_bits;
    atomicAdd(&cnt[e], 1u);
    const unsigned old = atomicAdd(&lo[e], (unsigned)v);
    const unsigned h = (unsigned)((unsigned long long)v >> 32) + ((old + (unsigned)v) < old ? 1u : 0u);
    if (h) atomicAdd(&hi[e], h);
  }
  __syncthreads();
  if (t == 0) p.cursor[b] = 0;
  for (unsigned i = t; i < E; i += blockDim.x) {
    const unsigned long long e = (unsigned long long)b * E + i;
    if (e < nent && cnt[i]) { ulonglong2* w = (ulonglong2*)(tab + 2 * e); ulonglong2 x = *w; x.x += lo[i] | ((unsigned long long)hi[i] << 32); x.y += cnt[i]; *w = x; }
  }
}

static Cols g_cols; static size_t g_n; static unsigned long long *g_tab, *g_sink; static int g_sms;
static const char* SHN[] = {"a 2x128b@32B", "b 128b contig", "c 8B l+32j", "d cp.async"};
static const char* PON[] = {"plain", "evict_first", "L2::128B", "L2::256B"};
static const char* MON[] = {"all", "skip", "all+red", "skip+red", "skip+part"};

template <class K> static void timed(K kernel, int ctas, size_t smem, double sel, const char* what, int shape, int pol, int depth, int mode, int runs) {
  const long long ntiles = (long long)(g_n / ROWS);
  const long long lo = 0; const unsigned long long span = (unsigned long long)(sel * 1000) - 1;
  if (smem) CK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  int per_sm = 0; CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, 256, smem));
  if (per_sm < ctas) { printf("%-14s %-14s %-12s depth=%d ctas/SM=%d  -- only %d CTAs/SM fit\n", what, SHN[shape], PON[pol], depth, ctas, per_sm); return; }
  cudaEvent_t a, b; CK(cudaEventCreate(&a)); CK(cudaEventCreate(&b));
  float best = 1e9;
  for (int it = 0; it < 6; it++) {
    CK(cudaEventRecord(a)); kernel<<<g_sms * ctas, 256, smem>>>(g_cols, ntiles, lo, span, g_tab, g_sink); CK(cudaEventRecord(b));
    CK(cudaEventSynchronize(b)); CK(cudaGetLastError());
    float ms; CK(cudaEventElapsedTime(&ms, a, b)); if (it > 0 && ms < best) best = ms;
  }
  printf("%-14s %-14s %-12s %-9s depth=%d ctas/SM=%d sel=%.2f%s  %7.3f ms  %6.3f TB/s of 32 B/row  %.1f Grows/s\n", what, SHN[shape], PON[pol], MON[mode], depth, ctas, sel,
         runs ? " runs8" : "      ", best, 32.0 * g_n / (best * 1e-3) / 1e12, g_n / (best * 1e-3) / 1e9);
  CK(cudaEventDestroy(a)); CK(cudaEventDestroy(b));
}
template <int SH, int POL, int D, int M, int PAD = 0> static void st(int ctas, double sel, const char* what, int runs = 0) { timed(stream_kernel<SH, POL, D, M, PAD>, ctas, 0, sel, what, SH, POL, D, M, runs); }

// skip+part followed by bucket_reduce_kernel, against skip+red on the same table; checks that both leave the same table
template <int PAD> static void part(double sel, int shift, int stage) {
  const unsigned long long nent = PAD ? PAD_ENTRIES : 1ULL << 20;
  const int idx_bits = PAD ? 22 : 20, nb = (int)((nent + (1ULL << shift) - 1) >> shift);
  const long long ntiles = (long long)(g_n / ROWS), lo = 0; const unsigned long long span = (unsigned long long)(sel * 1000) - 1;
  const int live = (int)((((PAD ? 20ULL : 8ULL) << 17) + (1ULL << shift) - 1) >> shift);   // buckets that hold a key of the generator
  Part p; p.shift = shift; p.idx_bits = idx_bits; p.nb = nb; p.stage = stage; p.cap = (unsigned)(g_n * sel / live * 1.1) + 4096;
  CK(cudaMalloc(&p.spill, (size_t)nb * p.cap * 8)); CK(cudaMalloc(&p.cursor, nb * 4)); CK(cudaMemset(p.cursor, 0, nb * 4));
  const size_t sm1 = (size_t)stage * 10 + (size_t)nb * 12, sm2 = (size_t)12 << shift;
  CK(cudaFuncSetAttribute(part_kernel<PAD>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm1));
  CK(cudaFuncSetAttribute(bucket_reduce_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm2));
  int per_sm = 0; CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, part_kernel<PAD>, 256, sm1)); per_sm = per_sm > 4 ? 4 : per_sm;
  int per_sm2 = 0; CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm2, bucket_reduce_kernel, 1024, sm2));
  auto run = [&] { part_kernel<PAD><<<g_sms * per_sm, 256, sm1>>>(g_cols, ntiles, lo, span, g_tab, p); };
  auto reduce = [&] { bucket_reduce_kernel<<<nb, 1024, sm2>>>(p, g_tab, nent); };
  // same table from both forms
  std::vector<unsigned long long> ref(2 * nent), got(2 * nent);
  CK(cudaMemset(g_tab, 0, nent * 16)); stream_kernel<SH_C, P_EVICT, 1, M_SKIP_RED, PAD><<<g_sms * 4, 256>>>(g_cols, ntiles, lo, span, g_tab, g_sink);
  CK(cudaMemcpy(ref.data(), g_tab, nent * 16, cudaMemcpyDeviceToHost));
  CK(cudaMemset(g_tab, 0, nent * 16)); run();
  std::vector<unsigned> cur(nb); CK(cudaMemcpy(cur.data(), p.cursor, nb * 4, cudaMemcpyDeviceToHost));
  unsigned long long placed = 0, over = 0; unsigned mx = 0;
  for (unsigned c : cur) { placed += c < p.cap ? c : p.cap; over += c > p.cap ? c - p.cap : 0; mx = c > mx ? c : mx; }
  reduce(); CK(cudaMemcpy(got.data(), g_tab, nent * 16, cudaMemcpyDeviceToHost)); CK(cudaGetLastError());
  size_t bad = 0; for (size_t i = 0; i < 2 * nent; i++) bad += got[i] != ref[i];
  cudaEvent_t a, m, b; CK(cudaEventCreate(&a)); CK(cudaEventCreate(&m)); CK(cudaEventCreate(&b));
  float best = 1e9, b1 = 0, b2 = 0;
  for (int it = 0; it < 6; it++) {
    CK(cudaEventRecord(a)); run(); CK(cudaEventRecord(m)); reduce(); CK(cudaEventRecord(b)); CK(cudaEventSynchronize(b)); CK(cudaGetLastError());
    float t1, t2; CK(cudaEventElapsedTime(&t1, a, m)); CK(cudaEventElapsedTime(&t2, m, b));
    if (it > 0 && t1 + t2 < best) { best = t1 + t2; b1 = t1; b2 = t2; }
  }
  printf("part   %-7s shift=%d (%d buckets) stage=%d: %zu B smem, %d CTAs/SM; reduce %zu B, %d CTAs/SM  sel=%.2f  %7.3f ms = %.3f partition + %.3f reduce"
         "  tuples %llu in runs, %llu by RED (bucket full, max bucket %u of %u)  mismatching words %zu\n",
         PAD ? "padded" : "compact", shift, nb, stage, sm1, per_sm, sm2, per_sm2, sel, best, b1, b2, placed, over, mx, p.cap, bad);
  CK(cudaEventDestroy(a)); CK(cudaEventDestroy(m)); CK(cudaEventDestroy(b)); CK(cudaFree(p.spill)); CK(cudaFree(p.cursor));
}
template <int POL, int D, int M> static void ca(int ctas, double sel, const char* what, int runs = 0) {
  timed(cpasync_kernel<POL, D, M>, ctas, (size_t)WARPS * (D + 1) * NCOL * ROWS * 8, sel, what, SH_D, POL, D, M, runs);
}

int main(int argc, char** argv) {
  g_n = (argc > 1) ? strtoull(argv[1], 0, 10) : (size_t)1 << 28;
  cudaDeviceProp prop; CK(cudaGetDeviceProperties(&prop, 0)); g_sms = prop.multiProcessorCount;
  unsigned plim = 0; nvmlDevice_t dev;
  if (nvmlInit() == NVML_SUCCESS && nvmlDeviceGetHandleByIndex(0, &dev) == NVML_SUCCESS) nvmlDeviceGetPowerManagementLimit(dev, &plim);
  printf("card: %s, %d SMs, power limit %.0f W; 4 int64 columns x %zu rows (%.2f GB), best of 5 after a warm-up\n", prop.name, g_sms, plim / 1000.0, g_n, 32.0 * g_n / 1e9);
  long long* c[NCOL]; for (int i = 0; i < NCOL; i++) CK(cudaMalloc(&c[i], g_n * 8));
  for (int i = 0; i < NCOL; i++) g_cols.c[i] = c[i];
  CK(cudaMalloc(&g_tab, PAD_ENTRIES * 16)); CK(cudaMemset(g_tab, 0, PAD_ENTRIES * 16)); CK(cudaMalloc(&g_sink, 64));
  unsigned long long* d_cnt; CK(cudaMalloc(&d_cnt, 16));
  gen<<<g_sms * 8, 256>>>(c[0], c[1], c[2], c[3], g_n, 0); CK(cudaDeviceSynchronize());
  const bool only_part = argc > 2 && !strcmp(argv[2], "part");
  if (!only_part) {

  printf("\n== 1. read ceiling per load shape and L2 policy (all rows, all columns, no prefetch, 4 CTAs/SM)\n");
  st<SH_A, P_NONE, 0, M_ALL>(4, 1, "ceiling"); st<SH_A, P_EVICT, 0, M_ALL>(4, 1, "ceiling"); st<SH_A, P_128, 0, M_ALL>(4, 1, "ceiling"); st<SH_A, P_256, 0, M_ALL>(4, 1, "ceiling");
  st<SH_B, P_NONE, 0, M_ALL>(4, 1, "ceiling"); st<SH_B, P_EVICT, 0, M_ALL>(4, 1, "ceiling"); st<SH_B, P_128, 0, M_ALL>(4, 1, "ceiling"); st<SH_B, P_256, 0, M_ALL>(4, 1, "ceiling");
  st<SH_C, P_NONE, 0, M_ALL>(4, 1, "ceiling"); st<SH_C, P_EVICT, 0, M_ALL>(4, 1, "ceiling"); st<SH_C, P_128, 0, M_ALL>(4, 1, "ceiling"); st<SH_C, P_256, 0, M_ALL>(4, 1, "ceiling");
  ca<P_NONE, 1, M_ALL>(4, 1, "ceiling"); ca<P_EVICT, 1, M_ALL>(4, 1, "ceiling"); ca<P_128, 1, M_ALL>(4, 1, "ceiling"); ca<P_256, 1, M_ALL>(4, 1, "ceiling");

  printf("\n== 2. latency hiding: tiles prefetched per warp x CTAs per SM (evict_first)\n");
  for (int ctas = 2; ctas <= 4; ctas++) {
    st<SH_A, P_EVICT, 0, M_ALL>(ctas, 1, "prefetch"); st<SH_A, P_EVICT, 1, M_ALL>(ctas, 1, "prefetch"); st<SH_A, P_EVICT, 2, M_ALL>(ctas, 1, "prefetch");
    st<SH_C, P_EVICT, 0, M_ALL>(ctas, 1, "prefetch"); st<SH_C, P_EVICT, 1, M_ALL>(ctas, 1, "prefetch"); st<SH_C, P_EVICT, 2, M_ALL>(ctas, 1, "prefetch");
    ca<P_EVICT, 0, M_ALL>(ctas, 1, "prefetch"); ca<P_EVICT, 1, M_ALL>(ctas, 1, "prefetch"); ca<P_EVICT, 2, M_ALL>(ctas, 1, "prefetch");
  }

  printf("\n== 3. sector skipping: f in full, k1 k2 v only for rows with f in range (shape c, evict_first, filter of the next tile in flight)\n");
  const double sels[] = {0.01, 0.05, 0.2, 0.5, 1.0};
  for (int runs = 0; runs <= 1; runs++) {
    gen<<<g_sms * 8, 256>>>(c[0], c[1], c[2], c[3], g_n, runs); CK(cudaDeviceSynchronize());
    for (double s : sels) {
      unsigned long long h[2]; CK(cudaMemset(d_cnt, 0, 16)); count_sectors<<<g_sms * 8, 256>>>(c[0], g_n, 0, (long long)(s * 1000) - 1, d_cnt);
      CK(cudaMemcpy(h, d_cnt, 16, cudaMemcpyDeviceToHost));
      printf("sectors: sel=%.2f%s  32-byte sectors holding a survivor %.3f -> %.1f B/row; 64-byte pairs %.3f -> %.1f B/row\n", s, runs ? " runs8" : "", h[0] / (g_n / 4.0),
             8 + 24.0 * h[0] / (g_n / 4.0), h[1] / (g_n / 8.0), 8 + 24.0 * h[1] / (g_n / 8.0));
      st<SH_C, P_EVICT, 1, M_ALL>(4, s, "skip?", runs); st<SH_C, P_EVICT, 1, M_SKIP>(4, s, "skip?", runs); st<SH_C, P_EVICT, 1, M_SKIP>(3, s, "skip?", runs);
    }
  }
  gen<<<g_sms * 8, 256>>>(c[0], c[1], c[2], c[3], g_n, 0); CK(cudaDeviceSynchronize());

  printf("\n== 4. with the dense-table REDs of the survivors (2^20 entries x 2 words, L2-resident), sel = 0.2\n");
  st<SH_A, P_EVICT, 0, M_ALL_RED>(4, 0.2, "red"); st<SH_C, P_EVICT, 1, M_ALL_RED>(4, 0.2, "red");
  st<SH_C, P_EVICT, 1, M_SKIP_RED>(4, 0.2, "red"); st<SH_C, P_NONE, 1, M_SKIP_RED>(4, 0.2, "red"); st<SH_C, P_EVICT, 1, M_SKIP_RED>(3, 0.2, "red");
  }

  printf("\n== 5. survivors bucketed into a spill area and reduced per bucket in shared memory (skip+part) against their REDs (skip+red)\n");
  for (double s : {0.2, 0.5}) {
    st<SH_C, P_EVICT, 1, M_SKIP>(4, s, "stream"); st<SH_C, P_EVICT, 1, M_SKIP_RED, 0>(4, s, "red compact"); st<SH_C, P_EVICT, 1, M_SKIP_RED, 1>(4, s, "red padded");
    for (int shift : {12, 13}) for (int stage : {3072, 4096, 4608}) { part<0>(s, shift, stage); part<1>(s, shift, stage); }
  }
  return 0;
}
