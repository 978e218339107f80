// Descriptors and launchers of the ShuffleWriterExec kernels (kernels_shuffle.cu): hash partition + batch_serde encode.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "kernels.cuh"

namespace b200q {

constexpr int SHUF_MAX_COLS = 32;
constexpr int SHUF_MAX_PARTS = 4096;        // partition counters live in shared memory
constexpr int SHUF_TILE = 4096;             // rows ranked and staged per CTA step

// One column of the batch being written.  Wire layout of a record of m rows (datafusion-ext-commons/src/io/batch_serde.rs:66-77,
// 264-306, 530-551): varint(m), then per column: one byte `has null buffer` (varint 0/1), ceil(m/8) validity bytes when it
// is 1, then the values: bit-packed for Boolean, raw for 1-byte types, otherwise `width` byte PLANES of m bytes each.
struct ShufCol {
  const void* values;                       // advanced by the Arrow offset (byte-addressable types)
  const uint8_t* validity;                  // may be null for a nullable column that carries no bitmap: every bit is written as 1
  uint32_t bit_offset;                      // Arrow offset for validity / Boolean values
  uint8_t width;                            // 0: Boolean (bits), else 1, 2, 4, 8, 16 bytes
  uint8_t nullable;                         // the field is nullable: the record carries a validity bitmap for it
  uint8_t tma;                              // set by the launcher: the column's tiles are staged by cp.async.bulk (16-byte aligned, width 1/2/4/8)
  uint8_t varlen;                           // Binary: width 4 (the int32 length planes), `values` = the data base the offsets index
  uint32_t k8, kw;                          // columns before this one take k8 * ceil(m/8) + kw * m bytes (+ one flag byte each)
};

struct ShufSpec {
  int32_t ncols, num_partitions, batch_size, nkeys;
  uint32_t tot_k8, tot_kw;                  // record of m rows = varint_len(m) + ncols + tot_k8 * ceil(m/8) + tot_kw * m bytes
  int8_t key_col[8];                        // hash partitioning: indices (into col[]) of the key columns, in hash order
  uint8_t key_phys[8];
  ShufCol col[SHUF_MAX_COLS];
};

__host__ __device__ inline uint32_t shuf_varint_len(unsigned long long m) { uint32_t l = 1; while (m >= 128) { m >>= 7; l++; } return l; }
__host__ __device__ inline unsigned long long shuf_record_bytes(const ShufSpec& sp, unsigned long long m) {
  return shuf_varint_len(m) + (unsigned long long)sp.ncols + (unsigned long long)sp.tot_k8 * ((m + 7) >> 3) + (unsigned long long)sp.tot_kw * m;
}
// bytes of partition holding t rows: records of batch_size rows, the last one shorter
__host__ __device__ inline unsigned long long shuf_partition_bytes(const ShufSpec& sp, unsigned long long t) {
  if (t == 0) return 0;
  const unsigned long long B = (unsigned long long)sp.batch_size, nrec = (t + B - 1) / B;
  return (nrec - 1) * shuf_record_bytes(sp, B) + shuf_record_bytes(sp, t - (nrec - 1) * B);
}

// pids[i] = pmod(murmur3(key columns of row i, seed 42), P) as u16 and counts[p] += 1 (shuffle/mod.rs:163-188); nkeys == 0: every row -> partition 0
int launch_shuffle_pids(const ShufSpec& sp, int64_t n, uint16_t* d_pids, unsigned long long* d_counts /* P, zeroed */, cudaStream_t s);
// part_off[p] = byte offset of partition p in the encoded buffer (P + 1 entries), cursors[p] = 0, record headers + flag bytes written
int launch_shuffle_layout(const ShufSpec& sp, const unsigned long long* d_counts, unsigned long long* d_part_off, unsigned long long* d_cursors, uint8_t* d_out, cudaStream_t s);
// scatter + encode: every value lands in its byte planes
int launch_shuffle_encode(const ShufSpec& sp, const uint16_t* d_pids, int64_t n, const unsigned long long* d_counts, const unsigned long long* d_part_off,
                          unsigned long long* d_cursors, uint8_t* d_out, cudaStream_t s);

// ---- batches with Binary columns (batch_serde.rs:595-619 + write_offsets :217-240): after the `has null buffer` byte and the
// validity bytes, a Binary column of a record of m rows is its m int32 lengths as 4 byte planes (a NULL row has length 0), then
// the bytes of its rows in row order.  A record's size now depends on the data, so the layout is computed in passes over
// positions assigned once: sorted position q of the chunk = partition-major order, row perm[q] of the input.
constexpr int SHUF_MAX_VARLEN = SHUF_MAX_COLS;
struct ShufVarlen {
  int32_t nb;                               // Binary columns
  uint32_t B;                               // rows per record (the last record of a partition holds the rest)
  long long n, R;                           // rows and records of the chunk
  int8_t col[SHUF_MAX_VARLEN];              // column index of the k-th Binary column, ascending
  const int32_t* offsets[SHUF_MAX_VARLEN];  // its Arrow offsets, advanced by the Arrow offset (offsets[0] may be > 0)
  // device work arrays of the chunk
  uint32_t* perm;                           // n: sorted position -> input row (null when P = 1: the identity)
  uint32_t* lens;                           // nb * n: data bytes of every sorted position per Binary column
  unsigned long long* doff;                 // nb * (n + 1): exclusive prefix of `lens` (64-bit: a chunk may carry > 4 GiB)
  const unsigned long long* row_start;      // P + 1: first sorted position of every partition
  const unsigned long long* rec_start;      // P + 1: first record of every partition
  unsigned long long* rec_size;             // R: encoded bytes of every record
  unsigned long long* rec_off;              // R + 1: byte offset of every record in the chunk's buffer
  unsigned long long* sums;                 // scan block sums: shuffle_varlen_scan_blocks(max(n, R)) entries
  unsigned* err;                            // bit 0: one record holds more than INT32_MAX bytes of Binary data
};
int64_t shuffle_varlen_scan_blocks(int64_t n);
// totals[k] += data bytes of the non-NULL rows of Binary column k (input order; totals zeroed)
int launch_shuffle_varlen_bytes(const ShufSpec& sp, const ShufVarlen& vl, unsigned long long* d_totals, cudaStream_t s);
// with row_start / rec_start uploaded and d_out zeroed where bits are OR-ed in: ranks the rows (P > 1), scans the lengths, sizes and
// places the records (part_off, P + 1 entries), writes headers, fixed-width planes, length planes and the Binary bytes
int launch_shuffle_varlen_encode(const ShufSpec& sp, const ShufVarlen& vl, const uint16_t* d_pids, const unsigned long long* d_counts,
                                 unsigned long long* d_cursors, unsigned long long* d_part_off, uint8_t* d_out, cudaStream_t s);

}  // namespace b200q
