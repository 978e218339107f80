// Descriptors and launchers of the SortExec kernels (kernels_sort.cu).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "kernels.cuh"

namespace b200q {

struct SortKeyCol {
  const void* values;                 // contiguous column of the concatenated input
  const uint8_t* valid_bytes;         // one byte per row, null: no NULLs (or see valid_bits)
  uint8_t phys;                       // PhysKind
  uint8_t descending, nulls_first;
  uint8_t dec_word;                   // decimal128: 0 = low word, 1 = high word
  uint32_t bit_offset;                // of valid_bits
  unsigned long long mask;            // all-ones over the type's width (keeps `~w` of a descending key inside it)
  const uint8_t* valid_bits;          // used when valid_bytes is null: an Arrow bitmap (bit r + bit_offset), null: no NULLs
};

// the order-preserving 64-bit word of row r of key column k (0 for a NULL row); *valid says whether the row is non-NULL.
// Ascending (null rank, word) is the column's order under k.descending / k.nulls_first, with null rank
// valid ? (nulls_first ? 1 : 0) : (nulls_first ? 0 : 1).  Shared by the sort and the sort-merge join.
__device__ __forceinline__ unsigned long long sort_normalise_word(const SortKeyCol& k, long long r, bool* valid) {
  bool ok = true;
  if (k.valid_bytes) ok = k.valid_bytes[r] != 0;
  else if (k.valid_bits) { const unsigned long long bi = (unsigned long long)r + k.bit_offset; ok = (k.valid_bits[bi >> 3] >> (bi & 7)) & 1; }
  *valid = ok;
  unsigned long long w = 0;
  if (!ok) return 0;
  switch (k.phys) {
    case PH_BOOL: w = ((const uint8_t*)k.values)[r] ? 1 : 0; break;       // the stage hands Boolean keys over as bytes
    case PH_I8: w = (uint8_t)(((const int8_t*)k.values)[r] ^ 0x80); break;
    case PH_I16: w = (uint16_t)(((const int16_t*)k.values)[r] ^ 0x8000); break;
    case PH_I32: w = (uint32_t)(((const int32_t*)k.values)[r]) ^ 0x80000000u; break;
    case PH_I64: w = (unsigned long long)(((const long long*)k.values)[r]) ^ 0x8000000000000000ull; break;
    case PH_F32: { const uint32_t b = ((const uint32_t*)k.values)[r]; w = (b & 0x80000000u) ? (uint32_t)~b : (b | 0x80000000u); break; }
    case PH_F64: { const unsigned long long b = ((const unsigned long long*)k.values)[r]; w = (b >> 63) ? ~b : (b | 0x8000000000000000ull); break; }
    default: {                                                         // decimal128: word 0 = low (unsigned), word 1 = high (signed)
      const unsigned long long* p = (const unsigned long long*)k.values + 2 * r;
      w = k.dec_word ? (p[1] ^ 0x8000000000000000ull) : p[0];
      break;
    }
  }
  if (k.descending) w = ~w & k.mask;
  return w;
}

int launch_sort_iota(uint32_t* d_idx, int64_t n, cudaStream_t s);
int launch_sort_normalise(const SortKeyCol& k, const uint32_t* d_idx, int64_t n, unsigned long long* d_keys, uint8_t* d_nullrank, cudaStream_t s);
// d_hist: 9 x 256 counters (zeroed): digits 0..7 of the keys, then the NULL ranks
int launch_sort_digit_hist(const unsigned long long* d_keys, const uint8_t* d_nullrank, int64_t n, unsigned long long* d_hist, cudaStream_t s);
int64_t sort_num_tiles(int64_t n);
// one stable pass on digit `shift / 8` (shift < 0: on the NULL rank): (keys, nullrank, idx) -> (okeys, onull, oidx)
// d_counts / d_offs: 256 * sort_num_tiles(n) + 1 int32 each, d_block_sums: scan_num_blocks(256 * tiles) int32
int launch_sort_pass(const unsigned long long* d_keys, const uint8_t* d_nullrank, const uint32_t* d_idx, int64_t n, int shift, int32_t* d_counts, int32_t* d_offs, int32_t* d_block_sums,
                     unsigned long long* d_okeys, uint8_t* d_onull, uint32_t* d_oidx, cudaStream_t s);

}  // namespace b200q
