// The BLOOM_FILTER aggregate on the device (agg/bloom_filter.rs + spark_bloom_filter.rs).  The bit array (at most 2^31 bits,
// Spark caps it at 2^26 = 8 MiB) stays in L2 while the rows stream past: a put is k atomicOrs on 64-bit words.
#include "hash.cuh"
#include "kernels_bloom.cuh"

namespace b200q {

namespace {

constexpr int BLOOM_BLOCK = 256;

unsigned grid_of(int64_t n) {
  const int64_t b = (n + BLOOM_BLOCK - 1) / BLOOM_BLOCK;
  return (unsigned)(b < 1 ? 1 : b > 65535 * 16 ? 65535 * 16 : b);
}

__global__ void __launch_bounds__(BLOOM_BLOCK) bloom_put_kernel(const DevCol col, uint8_t phys, long long n, unsigned long long* __restrict__ bits,
                                                                int32_t bit_size, int32_t k) {
  for (long long i = blockIdx.x * (long long)BLOOM_BLOCK + threadIdx.x; i < n; i += (long long)gridDim.x * BLOOM_BLOCK) {
    if (col.validity) { const unsigned long long bi = (unsigned long long)i + col.bit_offset; if (!((__ldg(col.validity + (bi >> 3)) >> (bi & 7)) & 1)) continue; }
    long long v;
    switch (phys) {
      case PH_I8: v = __ldg((const signed char*)col.values + i); break;
      case PH_I16: v = __ldg((const short*)col.values + i); break;
      case PH_I32: v = __ldg((const int*)col.values + i); break;
      default: v = __ldg((const long long*)col.values + i); break;
    }
    const int32_t h1 = mm3_hash_long(v, 0), h2 = mm3_hash_long(v, h1);
    for (int32_t j = 1; j <= k; j++) {
      int32_t c = (int32_t)((uint32_t)h1 + (uint32_t)j * (uint32_t)h2);   // i32 wrapping
      if (c < 0) c = ~c;                                                  // flip all bits if negative
      const uint32_t b = (uint32_t)(c % bit_size);
      atomicOr(bits + (b >> 6), 1ULL << (b & 63));
    }
  }
}

__device__ __forceinline__ unsigned long long load_be64(const uint8_t* p) {
  unsigned long long v = 0;
#pragma unroll
  for (int j = 0; j < 8; j++) v = (v << 8) | p[j];
  return v;
}

__global__ void __launch_bounds__(BLOOM_BLOCK) bloom_merge_kernel(const uint8_t* __restrict__ src, unsigned long long* __restrict__ bits, long long nwords) {
  for (long long i = blockIdx.x * (long long)BLOOM_BLOCK + threadIdx.x; i < nwords; i += (long long)gridDim.x * BLOOM_BLOCK)
    bits[i] |= load_be64(src + 8 * i);
}

__global__ void __launch_bounds__(BLOOM_BLOCK) bloom_popcount_kernel(const unsigned long long* __restrict__ bits, long long nwords, unsigned long long* count) {
  unsigned long long c = 0;
  for (long long i = blockIdx.x * (long long)BLOOM_BLOCK + threadIdx.x; i < nwords; i += (long long)gridDim.x * BLOOM_BLOCK) {
    const unsigned long long w = bits[i];
    c += __popc((unsigned)w) + __popc((unsigned)(w >> 32));
  }
  for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
  if ((threadIdx.x & 31) == 0 && c) atomicAdd(count, c);
}

__global__ void __launch_bounds__(BLOOM_BLOCK) bloom_fold_kernel(const unsigned long long* __restrict__ bits, long long nwords, unsigned long long* out, long long shrunk) {
  for (long long i = blockIdx.x * (long long)BLOOM_BLOCK + threadIdx.x; i < nwords; i += (long long)gridDim.x * BLOOM_BLOCK) {
    unsigned long long x = bits[i];
    if (!x) continue;
    if (shrunk >= 64) { atomicOr(out + (i & (shrunk / 64 - 1)), x); continue; }
    const unsigned long long mask = (1ULL << shrunk) - 1;                // shrunk < 64: every bit lands in word 0
    unsigned long long r = 0;
    for (int j = 0; j < 64; j += (int)shrunk) r |= (x >> j) & mask;
    atomicOr(out, r);
  }
}

__global__ void __launch_bounds__(BLOOM_BLOCK) bloom_write_kernel(const unsigned long long* __restrict__ bits, long long nwords, uint8_t* __restrict__ dst) {
  for (long long i = blockIdx.x * (long long)BLOOM_BLOCK + threadIdx.x; i < nwords; i += (long long)gridDim.x * BLOOM_BLOCK) {
    const unsigned long long v = bits[i];
#pragma unroll
    for (int j = 0; j < 8; j++) dst[8 * i + j] = (uint8_t)(v >> (56 - 8 * j));
  }
}

}  // namespace

int launch_bloom_put(const DevCol& col, uint8_t phys, int64_t n, unsigned long long* bits, int32_t bit_size, int32_t k, cudaStream_t s) {
  if (n <= 0) return 0;
  bloom_put_kernel<<<grid_of(n), BLOOM_BLOCK, 0, s>>>(col, phys, n, bits, bit_size, k);
  return 1;
}
int launch_bloom_merge(const uint8_t* src_be, unsigned long long* bits, int64_t nwords, cudaStream_t s) {
  bloom_merge_kernel<<<grid_of(nwords), BLOOM_BLOCK, 0, s>>>(src_be, bits, nwords);
  return 1;
}
int launch_bloom_popcount(const unsigned long long* bits, int64_t nwords, unsigned long long* count, cudaStream_t s) {
  bloom_popcount_kernel<<<grid_of(nwords), BLOOM_BLOCK, 0, s>>>(bits, nwords, count);
  return 1;
}
int launch_bloom_fold(const unsigned long long* bits, int64_t nwords, unsigned long long* out, int64_t shrunk, cudaStream_t s) {
  bloom_fold_kernel<<<grid_of(nwords), BLOOM_BLOCK, 0, s>>>(bits, nwords, out, shrunk);
  return 1;
}
int launch_bloom_write(const unsigned long long* bits, int64_t nwords, uint8_t* dst, cudaStream_t s) {
  bloom_write_kernel<<<grid_of(nwords), BLOOM_BLOCK, 0, s>>>(bits, nwords, dst);
  return 1;
}

}  // namespace b200q
