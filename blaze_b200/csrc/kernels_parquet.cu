// Parquet column-chunk decode on the GPU (SURVEY.md §8(f) rank 3).  The host frames the pages (parquet_meta.cc: Thrift headers,
// Snappy, run tables); these kernels expand a whole column chunk — any mix of PLAIN and dictionary-encoded pages — in one pass:
// every row finds its run by binary search over the chunk's run table (a few hundred entries, L1-resident), unpacks its
// dictionary index or reads its PLAIN value, and writes the Arrow value (narrowing INT32 -> int8 / int16, sign-extending
// INT32 / INT64 / big-endian FIXED_LEN_BYTE_ARRAY decimals to 128 bits).  Definition levels (max level 1) become the validity
// bytes; an exclusive scan of them gives every non-NULL row the ordinal of its stored value.
#include <cuda_runtime.h>
#include <stdint.h>

#include <algorithm>

#include "kernels_parquet.cuh"

namespace b200q {

namespace {

constexpr int PB = 256;
int pgrid(int64_t n) {
  int dev = 0, sms = 132; cudaGetDevice(&dev); cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  return (int)std::max<int64_t>(1, std::min<int64_t>((n + PB * 4 - 1) / (PB * 4), (int64_t)sms * 8));
}

__device__ __forceinline__ int find_run(const PqDevRun* __restrict__ runs, int n, uint32_t pos) {
  int lo = 0, hi = n - 1;                                             // last run whose start <= pos
  while (lo < hi) { const int mid = (lo + hi + 1) >> 1; if (__ldg(&runs[mid].start) <= pos) lo = mid; else hi = mid - 1; }
  return lo;
}
// The positions of a warp's 32 consecutive rows are monotone, so ONE binary search (for lane 0's position) serves the warp; lanes whose position
// lies beyond that run walk forward (at most 31 runs start inside 32 positions).
__device__ __forceinline__ int find_run_warp(const PqDevRun* __restrict__ runs, int n, uint32_t pos) {
  int ri = 0;
  const uint32_t first = __shfl_sync(0xffffffffu, pos, 0);
  if ((threadIdx.x & 31) == 0) ri = find_run(runs, n, first);
  ri = __shfl_sync(0xffffffffu, ri, 0);
  while (ri + 1 < n && __ldg(&runs[ri + 1].start) <= pos) ri++;
  return ri;
}
// 8 bytes from any address: two aligned loads and a funnel shift (buffers are allocated 256-byte aligned and padded by 16 bytes)
__device__ __forceinline__ unsigned long long ld_unaligned_u64(const uint8_t* p) {
  const uintptr_t a = (uintptr_t)p; const unsigned long long* q = (const unsigned long long*)(a & ~(uintptr_t)7); const int sh = (int)(a & 7) * 8;
  const unsigned long long w0 = __ldg(q);
  if (sh == 0) return w0;
  return (w0 >> sh) | (__ldg(q + 1) << (64 - sh));
}
__device__ __forceinline__ uint32_t ld_unaligned_u32(const uint8_t* p) {
  const uintptr_t a = (uintptr_t)p; const unsigned long long* q = (const unsigned long long*)(a & ~(uintptr_t)7); const int sh = (int)(a & 7) * 8;
  const unsigned long long w0 = __ldg(q);
  if (sh <= 32) return (uint32_t)(w0 >> sh);
  return (uint32_t)((w0 >> sh) | (__ldg(q + 1) << (64 - sh)));
}
__device__ __forceinline__ unsigned long long read_bits(const uint8_t* __restrict__ bytes, unsigned long long bit, int bw) {
  if (bw == 0) return 0;                                              // bw <= 32
  return (ld_unaligned_u64(bytes + (bit >> 3)) >> (bit & 7)) & ((1ull << bw) - 1);      // 7 + 32 bits of the 64 loaded
}

__global__ void __launch_bounds__(PB) pq_levels_kernel(const uint8_t* __restrict__ bytes, const PqDevRun* __restrict__ runs, int n_runs, long long n_rows, uint8_t* __restrict__ valid) {
  const long long gw = (blockIdx.x * (long long)PB + threadIdx.x) >> 5, nw = ((long long)gridDim.x * PB) >> 5; const unsigned lane = threadIdx.x & 31;
  for (long long base = gw * 32; base < n_rows; base += nw * 32) {
    const long long r = base + lane; const bool in = r < n_rows;
    const uint32_t pos = (uint32_t)(in ? r : n_rows - 1);
    const int ri = find_run_warp(runs, n_runs, pos);
    if (!in) continue;
    const unsigned long long off = __ldg(&runs[ri].off_or_value);
    valid[r] = __ldg(&runs[ri].kind) == PQR_RLE ? (uint8_t)(off != 0) : (uint8_t)read_bits(bytes, off + (unsigned long long)(pos - __ldg(&runs[ri].start)), 1);
  }
}

__global__ void __launch_bounds__(PB) pq_decode_kernel(const PqDecodeSpec sp, const uint8_t* __restrict__ valid, const int32_t* __restrict__ ordinal, long long n_rows, void* out, int* err) {
  const long long gw = (blockIdx.x * (long long)PB + threadIdx.x) >> 5, nw = ((long long)gridDim.x * PB) >> 5; const unsigned lane = threadIdx.x & 31;
  for (long long base = gw * 32; base < n_rows; base += nw * 32) {
    const long long r = base + lane; const bool in = r < n_rows; const long long rr = in ? r : n_rows - 1;
    const bool ok = in && (valid ? valid[rr] != 0 : true);
    const uint32_t o = ordinal ? (uint32_t)ordinal[rr] : (uint32_t)rr;      // the exclusive count of stored values: monotone in r, defined for NULL rows too
    const int ri = find_run_warp(sp.value_runs, sp.n_value_runs, o);
    if (!in) continue;
    unsigned long long lo = 0, hi = 0;                                // the stored value (low / high 64 bits)
    if (ok) {
      const uint32_t k = o - __ldg(&sp.value_runs[ri].start);
      const int kind = __ldg(&sp.value_runs[ri].kind), bw = __ldg(&sp.value_runs[ri].bw);
      const unsigned long long off = __ldg(&sp.value_runs[ri].off_or_value);
      const uint8_t* src;
      if (kind == PQR_PLAIN) {
        if (sp.src_width == 0) { const unsigned long long bit = off * 8 + k; lo = (sp.bytes[bit >> 3] >> (bit & 7)) & 1; src = nullptr; }
        else src = sp.bytes + off + (unsigned long long)k * sp.src_width;
      } else {
        const unsigned long long idx = kind == PQR_RLE ? off : read_bits(sp.bytes, off + (unsigned long long)k * bw, bw);
        if (sp.src_width == 0) { lo = idx & 1; src = nullptr; }                                     // RLE-encoded Booleans (data page v2)
        else if (idx >= (unsigned long long)sp.dict_count) { atomicOr(err, 1); src = nullptr; }
        else src = sp.dict + idx * sp.src_width;
      }
      if (src) {
        if (sp.out_kind == PQO_DEC_FROM_FLBA) {                       // big-endian two's complement of src_width bytes
          const bool neg = src[0] & 0x80;
          lo = hi = neg ? ~0ull : 0ull;
          for (int i = 0; i < sp.src_width; i++) { hi = (hi << 8) | (lo >> 56); lo = (lo << 8) | src[i]; }
        } else if (sp.src_width == 4) { lo = (unsigned long long)(long long)(int32_t)ld_unaligned_u32(src); hi = (long long)lo < 0 ? ~0ull : 0; }
        else { lo = ld_unaligned_u64(src); hi = (long long)lo < 0 ? ~0ull : 0; }
      }
    }
    switch (sp.out_kind) {
      case PQO_I8: ((int8_t*)out)[r] = (int8_t)lo; break;
      case PQO_I16: ((int16_t*)out)[r] = (int16_t)lo; break;
      case PQO_I32: ((int32_t*)out)[r] = (int32_t)lo; break;
      case PQO_I64: ((unsigned long long*)out)[r] = lo; break;
      case PQO_BOOL_BYTES: ((uint8_t*)out)[r] = (uint8_t)(lo & 1); break;
      default: ((unsigned long long*)out)[2 * r] = lo; ((unsigned long long*)out)[2 * r + 1] = hi; break;
    }
  }
}

}  // namespace

int launch_pq_levels(const uint8_t* bytes, const PqDevRun* runs, int n_runs, int64_t n_rows, uint8_t* valid, cudaStream_t s) {
  if (n_rows <= 0) return 0;
  pq_levels_kernel<<<pgrid(n_rows), PB, 0, s>>>(bytes, runs, n_runs, n_rows, valid);
  return 1;
}
int launch_pq_decode(const PqDecodeSpec& sp, const uint8_t* valid, const int32_t* ordinal, int64_t n_rows, void* out, int* d_err, cudaStream_t s) {
  if (n_rows <= 0) return 0;
  pq_decode_kernel<<<pgrid(n_rows), PB, 0, s>>>(sp, valid, ordinal, n_rows, out, d_err);
  return 1;
}

}  // namespace b200q
