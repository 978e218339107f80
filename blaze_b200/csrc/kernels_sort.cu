// SortExec on the GPU (SURVEY.md §8(f) rank 4): order-preserving key normalisation + stable LSD radix sort of
// (key, row) pairs + gather.
//
// Reference (datafusion-ext-plans/src/sort_exec.rs): every batch is sorted by its arrow-row encoded keys (:626-678), the
// sorted blocks are merged by a loser tree (:896-1027), `fetch` keeps the first rows (:650,946-960).  Row encoding makes a
// memcmp-comparable byte string per row: per key column a NULL marker that sorts first or last, then the value big-endian
// with the sign bit flipped (floats: IEEE totalOrder bits), all bytes inverted for descending columns.  Here the same
// order is produced column by column: the least significant key column first, each as a 64-bit normalised word (the
// same transform, as an integer instead of bytes) sorted by a STABLE radix sort, then a one-digit pass on its NULL rank;
// digits on which every row agrees are skipped (one histogram kernel finds them for all eight digits at once), so an
// int32 or date key costs four passes and a dictionary-like key one or two.  Ties keep their arrival order (the
// reference's order among equal keys is unspecified: unstable sort for short keys, sort_exec.rs:637-651).
#include <cuda_runtime.h>
#include <stdint.h>

#include <algorithm>

#include "kernels_sort.cuh"

namespace b200q {

namespace {

constexpr int SB = 256, S_ITEMS = 16, S_TILE = SB * S_ITEMS, S_WARPS = SB / 32;

int sgrid(int64_t n, int per_block = SB * 4) {
  int dev = 0, sms = 132; cudaGetDevice(&dev); cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  return (int)std::max<int64_t>(1, std::min<int64_t>((n + per_block - 1) / per_block, (int64_t)sms * 8));
}

// keys[i] = normalised word of row idx[i] (idx null: row i); nullrank[i] = 0 / 1 so that ascending order puts NULLs where asked
__global__ void __launch_bounds__(SB) sort_normalise_kernel(const SortKeyCol k, const uint32_t* __restrict__ idx, long long n, unsigned long long* __restrict__ keys, uint8_t* __restrict__ nullrank) {
  for (long long i = blockIdx.x * (long long)SB + threadIdx.x; i < n; i += (long long)gridDim.x * SB) {
    const long long r = idx ? idx[i] : i;
    bool valid;
    const unsigned long long w = sort_normalise_word(k, r, &valid);
    keys[i] = w;
    if (nullrank) nullrank[i] = valid ? (k.nulls_first ? 1 : 0) : (k.nulls_first ? 0 : 1);
  }
}

// hist[d * 256 + b] = rows whose digit d of the key is b (all 8 digits in one pass), hist[8 * 256 + r] = rows with null rank r
__global__ void __launch_bounds__(SB) sort_digit_hist_kernel(const unsigned long long* __restrict__ keys, const uint8_t* __restrict__ nullrank, long long n, unsigned long long* hist) {
  __shared__ unsigned s[9 * 256];
  for (int i = threadIdx.x; i < 9 * 256; i += SB) s[i] = 0;
  __syncthreads();
  for (long long i = blockIdx.x * (long long)SB + threadIdx.x; i < n; i += (long long)gridDim.x * SB) {
    const unsigned long long k = keys[i];
#pragma unroll
    for (int d = 0; d < 8; d++) atomicAdd(&s[d * 256 + (unsigned)((k >> (8 * d)) & 255)], 1u);
    if (nullrank) atomicAdd(&s[8 * 256 + nullrank[i]], 1u);
  }
  __syncthreads();
  for (int i = threadIdx.x; i < 9 * 256; i += SB) if (s[i]) atomicAdd(hist + i, (unsigned long long)s[i]);
}

__device__ __forceinline__ unsigned digit_of(const unsigned long long* keys, const uint8_t* nullrank, long long i, int shift) {
  return shift < 0 ? (unsigned)nullrank[i] : (unsigned)((keys[i] >> shift) & 255);
}

// counts[b * ntiles + tile] = rows of the tile with digit b
__global__ void __launch_bounds__(SB) sort_tile_hist_kernel(const unsigned long long* __restrict__ keys, const uint8_t* __restrict__ nullrank, long long n, int shift, int32_t* __restrict__ counts, long long ntiles) {
  __shared__ unsigned s[256];
  for (long long tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    s[threadIdx.x] = 0;
    __syncthreads();
    const long long t0 = tile * S_TILE;
    for (int j = threadIdx.x; j < S_TILE; j += SB) if (t0 + j < n) atomicAdd(&s[digit_of(keys, nullrank, t0 + j, shift)], 1u);
    __syncthreads();
    counts[(long long)threadIdx.x * ntiles + tile] = (int32_t)s[threadIdx.x];
    __syncthreads();
  }
}

// stable scatter: a warp owns 512 consecutive rows of the tile, 32 at a time; rows with the same digit keep their order.  The rows are first
// placed in digit order in SHARED memory and leave it as contiguous runs (one run per digit and tile): a warp's stores fall on a handful of
// sectors instead of one sector per lane (ncu of the direct form: 30 sectors per store request, 14 % DRAM).
constexpr size_t S_STAGE_BYTES = (size_t)S_TILE * (8 + 4 + 1);
__global__ void __launch_bounds__(SB, 3) sort_scatter_kernel(const unsigned long long* __restrict__ keys, const uint8_t* __restrict__ nullrank, const uint32_t* __restrict__ idx, long long n, int shift,
                                                             const int32_t* __restrict__ offs, long long ntiles, unsigned long long* __restrict__ okeys, uint8_t* __restrict__ onull, uint32_t* __restrict__ oidx) {
#ifdef B200Q_EMULATED_DEVICE                                                 // tools/emu: blocks run one at a time, shared memory is a static array
  static unsigned long long stage_words[(S_STAGE_BYTES + 7) / 8];
  unsigned char* stage = (unsigned char*)stage_words;
#else
  extern __shared__ __align__(16) unsigned char stage[];
#endif
  unsigned long long* s_key = (unsigned long long*)stage; uint32_t* s_idx = (uint32_t*)(s_key + S_TILE); uint8_t* s_null = (uint8_t*)(s_idx + S_TILE);
  __shared__ unsigned s_cnt[S_WARPS][256];
  __shared__ unsigned s_lstart[256], s_gbase[256], s_wsum[S_WARPS];
  const unsigned lane = threadIdx.x & 31, warp = threadIdx.x >> 5, lt = (1u << lane) - 1;
  for (long long tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    for (int i = threadIdx.x; i < S_WARPS * 256; i += SB) (&s_cnt[0][0])[i] = 0;
    __syncthreads();
    const long long t0 = tile * S_TILE, w0 = t0 + (long long)warp * (S_ITEMS * 32);
    unsigned rank[S_ITEMS]; unsigned dig[S_ITEMS];
#pragma unroll
    for (int r = 0; r < S_ITEMS; r++) {
      const long long i = w0 + r * 32 + lane;
      const bool live = i < n;
      const unsigned d = live ? digit_of(keys, nullrank, i, shift) : 256u;        // 256: a digit no live row has
      unsigned peers = __ballot_sync(0xFFFFFFFFu, live);
#pragma unroll
      for (int b = 0; b < 9; b++) { const unsigned bal = __ballot_sync(0xFFFFFFFFu, (d >> b) & 1); peers &= ((d >> b) & 1) ? bal : ~bal; }
      unsigned base = 0;
      if (live) base = s_cnt[warp][d];
      __syncwarp();
      if (live && (peers & lt) == 0) s_cnt[warp][d] = base + __popc(peers);         // the first lane of the group advances the counter
      __syncwarp();
      dig[r] = d; rank[r] = base + __popc(peers & lt);
    }
    __syncthreads();
    {   // digit = threadIdx.x: exclusive prefix over the warps; then the digit's start inside the tile (block scan) and its global base
      unsigned run = 0;
      for (int w = 0; w < S_WARPS; w++) { const unsigned c = s_cnt[w][threadIdx.x]; s_cnt[w][threadIdx.x] = run; run += c; }
      unsigned inc = run;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) { const unsigned y = __shfl_up_sync(0xFFFFFFFFu, inc, o); if (lane >= (unsigned)o) inc += y; }
      if (lane == 31) s_wsum[warp] = inc;
      __syncthreads();
      unsigned wbase = 0;
      for (unsigned w = 0; w < warp; w++) wbase += s_wsum[w];
      s_lstart[threadIdx.x] = wbase + inc - run;
      s_gbase[threadIdx.x] = (unsigned)offs[(long long)threadIdx.x * ntiles + tile];
    }
    __syncthreads();
#pragma unroll
    for (int r = 0; r < S_ITEMS; r++) {
      const long long i = w0 + r * 32 + lane;
      if (i < n) {
        const unsigned p = s_lstart[dig[r]] + s_cnt[warp][dig[r]] + rank[r];
        s_key[p] = keys[i]; s_idx[p] = idx[i];
        if (onull) s_null[p] = nullrank[i];
      }
    }
    __syncthreads();
    const unsigned rows = (unsigned)min((long long)S_TILE, n - t0);
    for (unsigned p = threadIdx.x; p < rows; p += SB) {
      const unsigned long long k = s_key[p];
      const unsigned nr = onull ? s_null[p] : 0u;
      const unsigned d = shift < 0 ? nr : (unsigned)((k >> shift) & 255);
      const unsigned dst = s_gbase[d] + (p - s_lstart[d]);
      okeys[dst] = k; oidx[dst] = s_idx[p];
      if (onull) onull[dst] = (uint8_t)nr;
    }
    __syncthreads();
  }
}

__global__ void __launch_bounds__(SB) iota_kernel(uint32_t* idx, long long n) {
  for (long long i = blockIdx.x * (long long)SB + threadIdx.x; i < n; i += (long long)gridDim.x * SB) idx[i] = (uint32_t)i;
}

}  // namespace

int launch_sort_iota(uint32_t* d_idx, int64_t n, cudaStream_t s) {
  if (n <= 0) return 0;
  iota_kernel<<<sgrid(n), SB, 0, s>>>(d_idx, n);
  return 1;
}
int launch_sort_normalise(const SortKeyCol& k, const uint32_t* d_idx, int64_t n, unsigned long long* d_keys, uint8_t* d_nullrank, cudaStream_t s) {
  if (n <= 0) return 0;
  sort_normalise_kernel<<<sgrid(n), SB, 0, s>>>(k, d_idx, n, d_keys, d_nullrank);
  return 1;
}
int launch_sort_digit_hist(const unsigned long long* d_keys, const uint8_t* d_nullrank, int64_t n, unsigned long long* d_hist, cudaStream_t s) {
  if (n <= 0) return 0;
  sort_digit_hist_kernel<<<sgrid(n, SB * 16), SB, 0, s>>>(d_keys, d_nullrank, n, d_hist);
  return 1;
}
int64_t sort_num_tiles(int64_t n) { return (n + S_TILE - 1) / S_TILE; }
int launch_sort_pass(const unsigned long long* d_keys, const uint8_t* d_nullrank, const uint32_t* d_idx, int64_t n, int shift, int32_t* d_counts, int32_t* d_offs, int32_t* d_block_sums,
                     unsigned long long* d_okeys, uint8_t* d_onull, uint32_t* d_oidx, cudaStream_t s) {
  if (n <= 0) return 0;
  const int64_t ntiles = sort_num_tiles(n);
  const int grid = (int)std::max<int64_t>(1, std::min<int64_t>(ntiles, (int64_t)sgrid(n, 1) ));
  sort_tile_hist_kernel<<<grid, SB, 0, s>>>(d_keys, d_nullrank, n, shift, d_counts, ntiles);
  int launches = 1 + launch_exclusive_scan_i32(d_counts, d_offs, 256 * ntiles, d_block_sums, s);
#ifndef B200Q_EMULATED_DEVICE
  cudaFuncSetAttribute(sort_scatter_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)S_STAGE_BYTES);      // per device: cheap, idempotent
#endif
  sort_scatter_kernel<<<grid, SB, S_STAGE_BYTES, s>>>(d_keys, d_nullrank, d_idx, n, shift, d_offs, ntiles, d_okeys, d_onull, d_oidx);
  return launches + 1;
}

}  // namespace b200q
