// Spark's hash functions on the device: the murmur3_x86_32 rounds (hash/mur.rs:19-87) used by the shuffle partitioner, the
// multi-GPU exchange and the bloom filters, and XXH64 (hash/xxhash.rs) as XxHash64 uses it.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace b200q {

__device__ __forceinline__ uint32_t rotl32(uint32_t x, int r) { return (x << r) | (x >> (32 - r)); }
__device__ __forceinline__ uint32_t mm3_mix_k1(uint32_t k1) { k1 *= 0xcc9e2d51u; k1 = rotl32(k1, 15); k1 *= 0x1b873593u; return k1; }
__device__ __forceinline__ uint32_t mm3_mix_h1(uint32_t h1, uint32_t k1) { h1 ^= k1; h1 = rotl32(h1, 13); return h1 * 5 + 0xe6546b64u; }
__device__ __forceinline__ uint32_t mm3_fmix(uint32_t h1, uint32_t len) { h1 ^= len; h1 ^= h1 >> 16; h1 *= 0x85ebca6bu; h1 ^= h1 >> 13; h1 *= 0xc2b2ae35u; h1 ^= h1 >> 16; return h1; }

// spark_compatible_murmur3_hash_long (hash/mur.rs): the 8 little-endian bytes of v as two 4-byte blocks
__device__ __forceinline__ int32_t mm3_hash_long(int64_t v, int32_t seed) {
  uint32_t h1 = mm3_mix_h1((uint32_t)seed, mm3_mix_k1((uint32_t)(uint64_t)v));
  h1 = mm3_mix_h1(h1, mm3_mix_k1((uint32_t)((uint64_t)v >> 32)));
  return (int32_t)mm3_fmix(h1, 8);
}

constexpr uint64_t XXH_P1 = 0x9E3779B185EBCA87ULL, XXH_P2 = 0xC2B2AE3D27D4EB4FULL, XXH_P3 = 0x165667B19E3779F9ULL,
                   XXH_P4 = 0x85EBCA77C2B2AE63ULL, XXH_P5 = 0x27D4EB2F165667C5ULL;
__device__ __forceinline__ uint64_t rotl64(uint64_t x, int r) { return (x << r) | (x >> (64 - r)); }
__device__ __forceinline__ uint64_t xxh64_round(uint64_t acc, uint64_t in) { acc += in * XXH_P2; return rotl64(acc, 31) * XXH_P1; }
__device__ __forceinline__ uint64_t xxh64_merge(uint64_t h, uint64_t acc) { h ^= xxh64_round(0, acc); return h * XXH_P1 + XXH_P4; }
__device__ __forceinline__ uint64_t xxh64_avalanche(uint64_t h) {
  h ^= h >> 33; h *= XXH_P2; h ^= h >> 29; h *= XXH_P3; h ^= h >> 32; return h;
}
// the tail of XXH64 after the stripes: 8-byte words, one 4-byte word, single bytes
__device__ __forceinline__ uint64_t xxh64_word8(uint64_t h, uint64_t w) { h ^= xxh64_round(0, w); return rotl64(h, 27) * XXH_P1 + XXH_P4; }
__device__ __forceinline__ uint64_t xxh64_word4(uint64_t h, uint32_t w) { h ^= (uint64_t)w * XXH_P1; return rotl64(h, 23) * XXH_P2 + XXH_P3; }
__device__ __forceinline__ uint64_t xxh64_byte(uint64_t h, uint8_t b) { h ^= (uint64_t)b * XXH_P5; return rotl64(h, 11) * XXH_P1; }

// XXH64 of a 4-byte int / an 8-byte long (its little-endian bytes), Spark's hashInt / hashLong
__device__ __forceinline__ uint64_t xxh64_int(uint32_t v, uint64_t seed) { return xxh64_avalanche(xxh64_word4(seed + XXH_P5 + 4, v)); }
__device__ __forceinline__ uint64_t xxh64_long(uint64_t v, uint64_t seed) { return xxh64_avalanche(xxh64_word8(seed + XXH_P5 + 8, v)); }

__device__ __forceinline__ uint64_t xxh_ld64(const uint8_t* p) { uint64_t v = 0; for (int i = 7; i >= 0; i--) v = (v << 8) | p[i]; return v; }
__device__ __forceinline__ uint32_t xxh_ld32(const uint8_t* p) { return (uint32_t)p[0] | (uint32_t)p[1] << 8 | (uint32_t)p[2] << 16 | (uint32_t)p[3] << 24; }

// XXH64 of n bytes (hash/xxhash.rs xxhash64); byte loads, since Utf8 data carries no alignment
__device__ __forceinline__ uint64_t xxh64_bytes(const uint8_t* p, uint32_t n, uint64_t seed) {
  uint64_t h;
  uint32_t i = 0;
  if (n >= 32) {
    uint64_t a1 = seed + XXH_P1 + XXH_P2, a2 = seed + XXH_P2, a3 = seed, a4 = seed - XXH_P1;
    for (; i + 32 <= n; i += 32) {
      a1 = xxh64_round(a1, xxh_ld64(p + i)); a2 = xxh64_round(a2, xxh_ld64(p + i + 8));
      a3 = xxh64_round(a3, xxh_ld64(p + i + 16)); a4 = xxh64_round(a4, xxh_ld64(p + i + 24));
    }
    h = rotl64(a1, 1) + rotl64(a2, 7) + rotl64(a3, 12) + rotl64(a4, 18);
    h = xxh64_merge(h, a1); h = xxh64_merge(h, a2); h = xxh64_merge(h, a3); h = xxh64_merge(h, a4);
  } else {
    h = seed + XXH_P5;
  }
  h += n;
  for (; i + 8 <= n; i += 8) h = xxh64_word8(h, xxh_ld64(p + i));
  if (i + 4 <= n) { h = xxh64_word4(h, xxh_ld32(p + i)); i += 4; }
  for (; i < n; i++) h = xxh64_byte(h, p[i]);
  return xxh64_avalanche(h);
}

}  // namespace b200q
