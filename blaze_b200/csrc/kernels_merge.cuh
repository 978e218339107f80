// Descriptors and launchers of the sort-merge join kernels (kernels_merge.cu): key normalisation with the sortedness check,
// the merge-path co-ranking of a left batch against the right side, counts, a 64-bit scan, and the emission of the
// (left row, right row) index pairs in output order.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "kernels_sort.cuh"

namespace b200q {

// the normalised join keys of one side, one entry per row: up to two order words and one flag byte
//   flags bit 0 / bit 1: null rank of key 0 / key 1 (SortKeyCol order), bit 2: some key is NULL (the row never matches)
// rows compare as the tuple (null rank 0, w0, null rank 1, w1): the order both sides must be sorted in
struct MergeKeys {
  const unsigned long long* w0;
  const unsigned long long* w1;        // null with one key
  const uint8_t* flags;
};
constexpr uint8_t SMJ_ANY_NULL = 4;

// the last row of the previous batch of one side, kept on the device between batches
struct SmjCarry { unsigned long long w0, w1; uint32_t flags, has; };
// what the host reads back after the normalise pass of a left batch
struct SmjStatus { unsigned long long rb0, rb1; uint32_t unsorted, _pad; };

// keys[0..nkeys) of rows 0..n) -> w0 / w1 / flags; sets st->unsorted when a row sorts before its predecessor (row 0: before
// *carry when carry->has); then *carry = row n - 1
int launch_smj_normalise(const SortKeyCol* keys, int nkeys, int64_t n, unsigned long long* w0, unsigned long long* w1, uint8_t* flags,
                         SmjCarry* d_carry, SmjStatus* d_status, cudaStream_t s);
// st->rb0 = right rows before left row 0, st->rb1 = right rows up to and including left row n - 1's key (rows [0, m))
int launch_smj_bounds(const MergeKeys& left, int64_t n, const MergeKeys& right, int64_t m, SmjStatus* d_status, cudaStream_t s);
// merge path of left rows [0, n) against right rows [rb0, rb1): lo[i] / hi[i] = first / one past the last right row with
// left row i's key (absolute right row numbers); pr[r - rb0] = left rows whose key is <= right row r's key
int launch_smj_merge(const MergeKeys& left, int64_t n, const MergeKeys& right, int64_t rb0, int64_t rb1, uint32_t* lo, uint32_t* hi, uint32_t* pr, cudaStream_t s);
// counts[i] = output rows of left row i for the join type (protobuf JoinType numbering)
int launch_smj_counts(const MergeKeys& left, int64_t n, const uint32_t* lo, const uint32_t* hi, int join_type, unsigned long long* counts, cudaStream_t s);
// matched[r] = 1 for right rows r in [rb0, rb1) whose key some left row of the batch has
int launch_smj_mark(const MergeKeys& left, const MergeKeys& right, int64_t rb0, int64_t rb1, const uint32_t* pr, uint8_t* matched, cudaStream_t s);
// flags[w] = 1 when right row s0 + w (w < nw) is unmatched
int launch_smj_unmatched(const uint8_t* matched, int64_t s0, int64_t nw, unsigned long long* flags, cudaStream_t s);
// exclusive scan of n u64 -> out[0..n] (out[n] = total); d_tmp: smj_scan_tmp_words(n) words
int64_t smj_scan_tmp_words(int64_t n);
int launch_smj_scan(const unsigned long long* in, unsigned long long* out, int64_t n, unsigned long long* d_tmp, cudaStream_t s);

// one output chunk [o0, o1): the pairs of the left rows (pidx = left row, bidx = right row or JOIN_NIL; bidx / exists may be
// null) and of the settled unmatched right rows [s0, s0 + nw) (pidx = JOIN_NIL).  Output position of left row i:
// L[i] + U[lo[i] - s0]; of unmatched right row r: L[p] + U[r - s0] with p = r < rb0 ? 0 : pr[r - rb0] (U null: 0)
struct SmjEmit {
  int64_t n;                           // left rows
  const uint32_t* lo; const uint32_t* hi; const uint8_t* lflags;
  const unsigned long long* L;         // n + 1
  const unsigned long long* U;         // nw + 1, or null
  int64_t s0, nw, rb0;
  const uint32_t* pr; const uint8_t* matched;
  int64_t o0, o1;
  uint32_t* pidx; uint32_t* bidx; uint8_t* exists;
};
int launch_smj_emit(const SmjEmit& e, cudaStream_t s);

}  // namespace b200q
