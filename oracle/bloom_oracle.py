"""Spark's runtime bloom filters restated in Python for the tests: XXH64 as Spark's XxHash64 uses it, murmur3 `hash_long`,
SparkBitArray and SparkBloomFilter.  Paths are relative to the reference's native-engine/.

Every value is a Python int wrapped to the Rust width it has there, so the oracle is exact and shares no code with the
device kernels."""
from __future__ import annotations

import struct
from typing import Iterable, List, Optional

M64 = (1 << 64) - 1
M32 = (1 << 32) - 1


def _i64(v: int) -> int:
    v &= M64
    return v - (1 << 64) if v >> 63 else v


def _i32(v: int) -> int:
    v &= M32
    return v - (1 << 32) if v >> 31 else v


# ---- XXH64: datafusion-ext-commons/src/hash/xxhash.rs ----------------------------------------------------------------
P1, P2, P3, P4, P5 = 0x9E3779B185EBCA87, 0xC2B2AE3D27D4EB4F, 0x165667B19E3779F9, 0x85EBCA77C2B2AE63, 0x27D4EB2F165667C5


def _rotl64(x: int, r: int) -> int:
    return ((x << r) | (x >> (64 - r))) & M64


def _round(acc: int, inp: int) -> int:                       # xxh64_round
    return (_rotl64((acc + inp * P2) & M64, 31) * P1) & M64


def _merge(h: int, acc: int) -> int:                         # xxh64_merge_round
    return ((h ^ _round(0, acc)) * P1 + P4) & M64


def _avalanche(h: int) -> int:                               # xxh64_avalanche
    h ^= h >> 33
    h = (h * P2) & M64
    h ^= h >> 29
    h = (h * P3) & M64
    return h ^ (h >> 32)


def xxhash64(data: bytes, seed: int) -> int:
    """spark_compatible_xxhash64_hash(data, seed) -> i64 (xxhash.rs:24-95)"""
    seed &= M64
    n, i = len(data), 0
    if n >= 32:
        a = [(seed + P1 + P2) & M64, (seed + P2) & M64, seed, (seed - P1) & M64]
        while n - i >= 32:
            for j in range(4):
                a[j] = _round(a[j], int.from_bytes(data[i + 8 * j:i + 8 * j + 8], "little"))
            i += 32
        h = (_rotl64(a[0], 1) + _rotl64(a[1], 7) + _rotl64(a[2], 12) + _rotl64(a[3], 18)) & M64
        for x in a:
            h = _merge(h, x)
    else:
        h = (seed + P5) & M64
    h = (h + n) & M64
    while n - i >= 8:
        h ^= _round(0, int.from_bytes(data[i:i + 8], "little"))
        h = (_rotl64(h, 27) * P1 + P4) & M64
        i += 8
    if n - i >= 4:
        h ^= (int.from_bytes(data[i:i + 4], "little") * P1) & M64
        h = (_rotl64(h, 23) * P2 + P3) & M64
        i += 4
    while i < n:
        h ^= (data[i] * P5) & M64
        h = (_rotl64(h, 11) * P1) & M64
        i += 1
    return _i64(_avalanche(h))


def value_bytes(v, type_name: str) -> bytes:
    """the bytes XxHash64 hashes for one value (datafusion-ext-commons/src/spark_hash.rs:84-195): Bool (as a u32 0/1), Int8,
    Int16, Int32 and Date32 as a 4-byte little-endian int; Int64 and Timestamp as an 8-byte long; Utf8 as its UTF-8 bytes"""
    if type_name in ("bool", "int8", "int16", "int32", "date32"):
        return struct.pack("<i", int(v))
    if type_name in ("int64", "timestamp[us]"):
        return struct.pack("<q", int(v))
    if type_name == "utf8":
        return v.encode() if isinstance(v, str) else bytes(v)
    raise ValueError(f"XxHash64 over {type_name} is not restated here")


def spark_xxhash64(columns: List[list], type_names: List[str]) -> List[int]:
    """XxHash64(children, 42) per row (datafusion-ext-functions/src/spark_hash.rs spark_xxhash64 + create_xxhash64_hashes):
    h = 42, then h = xxhash64(child, h) per child in order; a NULL (None) child leaves h; never NULL"""
    n = len(columns[0]) if columns else 0
    out = []
    for r in range(n):
        h = 42
        for col, tn in zip(columns, type_names):
            if col[r] is not None:
                h = xxhash64(value_bytes(col[r], tn), h)
        out.append(h)
    return out


# ---- murmur3: datafusion-ext-commons/src/hash/mur.rs -------------------------------------------------------------------
def _rotl32(x: int, r: int) -> int:
    return ((x << r) | (x >> (32 - r))) & M32


def _mix_k1(k1: int) -> int:
    k1 = (k1 * 0xcc9e2d51) & M32
    return (_rotl32(k1, 15) * 0x1b873593) & M32


def _mix_h1(h1: int, k1: int) -> int:
    h1 = _rotl32(h1 ^ k1, 13)
    return (h1 * 5 + 0xe6546b64) & M32


def _fmix(h1: int, n: int) -> int:
    h1 ^= n
    h1 ^= h1 >> 16
    h1 = (h1 * 0x85ebca6b) & M32
    h1 ^= h1 >> 13
    h1 = (h1 * 0xc2b2ae35) & M32
    return h1 ^ (h1 >> 16)


def hash_long(v: int, seed: int) -> int:
    """spark_compatible_murmur3_hash_long (mur.rs hash_long) -> i32"""
    v &= M64
    h1 = _mix_h1(seed & M32, _mix_k1(v & M32))
    h1 = _mix_h1(h1, _mix_k1(v >> 32))
    return _i32(_fmix(h1, 8))


# ---- SparkBitArray: datafusion-ext-commons/src/spark_bit_array.rs ------------------------------------------------------
class SparkBitArray:
    def __init__(self, words: List[int]):
        self.words = [w & M64 for w in words]

    @classmethod
    def with_num_bits(cls, num_bits: int) -> "SparkBitArray":          # new_with_num_bits
        if not 0 < num_bits <= 0x7FFFFFFF:
            raise ValueError(f"num_bits {num_bits} out of range")
        return cls([0] * ((num_bits + 63) // 64))

    def bit_size(self) -> int:
        return 64 * len(self.words)

    def set(self, i: int) -> None:
        self.words[i >> 6] |= 1 << (i & 63)

    def get(self, i: int) -> bool:
        return bool((self.words[i >> 6] >> (i & 63)) & 1)

    def put_all(self, other: "SparkBitArray") -> None:
        if len(self.words) != len(other.words):
            raise ValueError("bit arrays of different sizes")
        self.words = [a | b for a, b in zip(self.words, other.words)]

    def true_count(self) -> int:
        return sum(bin(w).count("1") for w in self.words)

    def write_to(self) -> bytes:                                       # big-endian i32 length, big-endian i64 words
        return struct.pack(">i", len(self.words)) + b"".join(struct.pack(">Q", w) for w in self.words)


# ---- SparkBloomFilter: datafusion-ext-commons/src/spark_bloom_filter.rs ------------------------------------------------
class SparkBloomFilter:
    def __init__(self, num_hash_functions: int, bits: SparkBitArray):
        self.k = num_hash_functions
        self.bits = bits

    @staticmethod
    def optimal_num_of_hash_functions(n: int, m: int) -> int:
        """max(1, round(m / n * ln 2)); Rust's f64::round rounds half away from zero"""
        import math
        x = m / n * math.log(2.0)
        return max(1, int(math.floor(x + 0.5)) if x >= 0 else -int(math.floor(-x + 0.5)))

    @classmethod
    def with_expected_num_items(cls, expected: int, num_bits: int) -> "SparkBloomFilter":
        return cls(cls.optimal_num_of_hash_functions(expected, num_bits), SparkBitArray.with_num_bits(num_bits))

    def _indexes(self, v: int) -> Iterable[int]:
        h1 = hash_long(v, 0)
        h2 = hash_long(v, h1)
        bit_size = _i32(self.bits.bit_size())
        for i in range(1, self.k + 1):
            c = _i32(h1 + i * h2)
            if c < 0:
                c = ~c                                                  # flip all the bits
            yield c % bit_size

    def put_long(self, v: int) -> None:
        for b in self._indexes(v):
            self.bits.set(b)

    def might_contain_long(self, v: int) -> bool:
        return all(self.bits.get(b) for b in self._indexes(v))

    def put_all(self, other: "SparkBloomFilter") -> None:
        if self.k != other.k:
            raise ValueError("bloom filters with different num_hash_functions")
        self.bits.put_all(other.bits)

    def shrink_to_fit(self) -> None:
        num_bits = self.bits.bit_size()
        shrunk = 1 << (max(1, self.k * self.bits.true_count() * 2) - 1).bit_length()   # next_power_of_two
        if shrunk >= num_bits:
            return
        nb = SparkBitArray.with_num_bits(shrunk)
        for i in range(num_bits):
            if self.bits.get(i):
                nb.set(i % shrunk)
        self.bits = nb

    def write_to(self) -> bytes:
        return struct.pack(">ii", 1, self.k) + self.bits.write_to()

    @classmethod
    def read_from(cls, data: bytes) -> "SparkBloomFilter":
        version, k, n = struct.unpack(">iii", data[:12])
        if version != 1:
            raise ValueError(f"unsupported version: {version}")
        words = [struct.unpack(">Q", data[12 + 8 * i:20 + 8 * i])[0] for i in range(n)]
        return cls(k, SparkBitArray(words))


def might_contain(filter_bytes: Optional[bytes], values: List[Optional[int]]) -> List[Optional[bool]]:
    """BloomFilterMightContain over Int8..Int64 values as this project evaluates it (bloom_filter_might_contain.rs): a NULL
    filter is False for every row; a NULL value is NULL (Spark's semantics; the reference probes the NULL slot instead)"""
    if filter_bytes is None:
        return [False] * len(values)
    bf = SparkBloomFilter.read_from(filter_bytes)
    return [None if v is None else bf.might_contain_long(int(v)) for v in values]


def frozen_row(bf: Optional[SparkBloomFilter]) -> bytes:
    """AccBloomFilterColumn::freeze_to_rows (datafusion-ext-plans/src/agg/bloom_filter.rs): [0] for None, else [1] ++ write_to"""
    return b"\x00" if bf is None else b"\x01" + bf.write_to()


def bloom_agg(values_per_batch: List[List[Optional[int]]], estimated_num_items: int, num_bits: int) -> Optional[SparkBloomFilter]:
    """AggBloomFilter::partial_update over the pushed batches (agg/bloom_filter.rs): None until a batch arrives; the filter is then
    created (optimal k) and every non-NULL value put"""
    bf = None
    for vals in values_per_batch:
        if not vals:
            continue
        if bf is None:
            bf = SparkBloomFilter.with_expected_num_items(estimated_num_items, num_bits)
        for v in vals:
            if v is not None:
                bf.put_long(int(v))
    return bf


def final_bytes(bf: Optional[SparkBloomFilter]) -> Optional[bytes]:
    """final_merge: shrink_to_fit then write_to; None stays NULL"""
    if bf is None:
        return None
    c = SparkBloomFilter(bf.k, SparkBitArray(list(bf.bits.words)))
    c.shrink_to_fit()
    return c.write_to()
