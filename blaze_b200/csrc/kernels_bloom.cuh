// Launchers of the BLOOM_FILTER aggregate kernels (kernels_bloom.cu): SparkBloomFilter put_long / put_all / shrink_to_fit /
// write_to (datafusion-ext-commons/src/spark_bloom_filter.rs, spark_bit_array.rs) over a device-resident bit array of 64-bit words.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "vm.h"

namespace b200q {

// put_long of every valid row of an Int8..Int64 column (phys PH_I8..PH_I64): k atomicOrs into bits[0, bit_size / 64)
int launch_bloom_put(const DevCol& col, uint8_t phys, int64_t n, unsigned long long* bits, int32_t bit_size, int32_t k, cudaStream_t s);
// bits[i] |= the i-th big-endian 8-byte word at src (any alignment): SparkBitArray::put_all of a serialized filter's words
int launch_bloom_merge(const uint8_t* src_be, unsigned long long* bits, int64_t nwords, cudaStream_t s);
// *count += the number of set bits (count zeroed by the caller)
int launch_bloom_popcount(const unsigned long long* bits, int64_t nwords, unsigned long long* count, cudaStream_t s);
// shrink_to_fit's fold: bit i of `bits` -> bit i mod `shrunk` of `out` (out zeroed, max(1, shrunk / 64) words; shrunk a power of two
// smaller than 64 * nwords)
int launch_bloom_fold(const unsigned long long* bits, int64_t nwords, unsigned long long* out, int64_t shrunk, cudaStream_t s);
// the words as big-endian i64 (SparkBitArray::write_to after its length) into dst
int launch_bloom_write(const unsigned long long* bits, int64_t nwords, uint8_t* dst, cudaStream_t s);

}  // namespace b200q
