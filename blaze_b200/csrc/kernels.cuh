// Kernel-side data structures shared between kernels.cu and the host runtime.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "vm.h"

namespace b200q {

constexpr int AGG_MAX_KEYS = 8;
constexpr int AGG_MAX_ACC = 16;
constexpr int AGG_MAX_ROW_WORDS = 24;       // per-row scratch words produced by the VM (keys + agg args)
constexpr int AGG_MAX_SLOT_WORDS = 32;

// accumulator update kinds (one 64-bit word each, except the DEC ones: lo,hi)
enum AccKind : uint8_t {
  ACC_ADD_I64 = 0,    // wrapping i64 add of the argument (AggSum over integers, sum.rs:103-109; count merge count.rs:128-149)
  ACC_ADD_F64,        // f64 add
  ACC_ADD_DEC,        // i128 add, two words, carry propagated through the returning atomic on the low word
  ACC_COUNT,          // += 1 when every listed argument is valid (count.rs:100-124)
  ACC_MIN_I64, ACC_MAX_I64,
  ACC_MIN_F64, ACC_MAX_F64,   // stored as IEEE totalOrder keys so integer atomics apply
  ACC_MIN_DEC, ACC_MAX_DEC,   // 128-bit CAS loop
  // FIRST / FIRST_IGNORES_NULL (first.rs, first_ignores_null.rs): the value of the eligible row with the smallest arrival
  // ordinal.  `oword` holds that ordinal (identity ~0, "not set"); the value word(s) and the value's validity bit (`vbit`,
  // 0xFF: never NULL) are written together with it under the slot lock.  Eligible rows:
  ACC_FIRST,          // every row (nargs 1), or a row whose second argument (the merged `#flag` column) is non-zero (nargs 2)
  ACC_FIRST_VALID,    // a row whose argument is valid
};
__host__ __device__ inline bool acc_is_first(uint8_t kind) { return kind == ACC_FIRST || kind == ACC_FIRST_VALID; }

struct AccOp {
  uint8_t kind;
  uint8_t word;        // word offset inside the accumulator entry
  uint8_t vbit;        // bit in the slot header's flags marking "accumulator has a value" (0xFF: always valid)
  uint8_t nargs;       // arguments (ACC_COUNT may have 0..4; others exactly 1, ACC_FIRST 1 or 2)
  uint8_t arg_out[4];  // VM output index of each argument
  uint8_t oword;       // ACC_FIRST*: word of the arrival ordinal (ACC_FIRST accumulators of one aggregate share it)
  uint8_t nwords;      // ACC_FIRST*: value words (2 for decimal128, else 1)
};

// The table is split in two arrays indexed by the slot number (tools/microbench/probes.cu compares the layouts: a probe
// load followed by a RED on the SAME sector is slower than probing one array and RED-ing another, because the read
// copies the L2 keeps of a line must be invalidated by every atomic on it):
//   key entry  = [hdr][key words...]           kstride words, probed with plain loads, written once at insertion
//   acc entry  = [accumulator words...]        astride words, only ever touched by RED/ATOM
//   hdr low 32 bits : tag  (0 empty, 1 locked, else 0x80000000|fingerprint — cf. agg_hash_map.rs:228-234)
//   hdr high 32 bits: flags (bits 0..15 accumulator-valid bits, bits 16..31 key-is-NULL bits)
struct AggLayout {
  int32_t nkeys, nkw, nacc, kstride, astride, nouts;
  uint8_t key_out[AGG_MAX_KEYS];     // VM output index of key k
  uint8_t key_word[AGG_MAX_KEYS];    // first word of key k inside the key entry (>= 1)
  uint8_t key_nwords[AGG_MAX_KEYS];  // 1, or 2 for decimal128
  uint8_t out_word[VM_MAX_OUT];      // VM output index -> word in the per-row scratch buffer
  AccOp acc[AGG_MAX_ACC];
  uint64_t init[AGG_MAX_SLOT_WORDS]; // initial accumulator entry (identities)
  uint32_t init_flags;               // accumulator-valid bits set at insertion (accumulators with vbit == 0xFF have none)
};

// Grouping sets of an ExpandExec fused into the aggregate: every row is evaluated once by the VM, then inserted once per set.
// One descriptor per set lives in device memory next to the program; the key entry layout (AggLayout) is shared by all sets.
constexpr int AGG_MAX_SETS = 64;
constexpr uint8_t AGG_KEY_CONST = 0xFF;   // key_out: the key is a constant of the set (key_const words, or NULL in key_null)
constexpr uint8_t AGG_NO_ARG = 0xFF;
struct AggSetDesc {
  uint8_t key_out[AGG_MAX_KEYS];          // VM output of key k in this set, or AGG_KEY_CONST
  uint8_t acc_arg[AGG_MAX_ACC][4];        // VM output of each argument of accumulator j in this set (AGG_NO_ARG: none)
  uint32_t key_null;                      // constant keys that are NULL in this set
  uint32_t acc_skip;                      // accumulators this set never updates (an argument is a NULL literal)
  uint64_t key_const[AGG_MAX_KEYS * 2];   // words of the constant keys, at their position in the key entry (key_word - 1)
};

struct AggTable {
  unsigned long long* keys;       // capacity * kstride words
  unsigned long long* accs;       // capacity * astride words
  uint64_t capacity;        // any size: slot = mulhi64(hash, capacity), linear probing with wrap-around
  uint64_t max_groups;      // load limit: inserts beyond it are deferred (table grown by the host, rows replayed)
  unsigned long long* counters;   // [0] ngroups, [1] ndeferred, [2] (int) error flags
  uint32_t* deferred;       // row indices that could not be inserted (with grouping sets: row * nsets + set)
};

// emit descriptors: one per output column
enum EmitKind : uint8_t {
  EMIT_KEY = 0,        // key k, cast back to its physical type
  EMIT_ACC_VALUE,      // accumulator word(s) as a value of `phys` (valid iff its vbit is set / always)
  EMIT_AVG_F64,        // sum(word)/count(word2) -> f64            (avg.rs:166-171)
  EMIT_AVG_DEC,        // i128 sum div_euclid count -> decimal128   (avg.rs:158-165)
  EMIT_FIRST_VALUE,    // FIRST value: valid iff the ordinal (word2) is set and the value's vbit is set (or vbit == 0xFF)
  EMIT_FIRST_FLAG,     // FIRST `#flag` state column: int8 1 iff the ordinal (word2) is set
};
struct EmitCol {
  uint8_t kind, phys, word, word2;   // word: offset in the key entry (EMIT_KEY) or in the accumulator entry
  uint8_t vbit;        // 0xFF: always valid
  uint8_t key;         // key index for EMIT_KEY
  uint8_t sum_is_f64;  // EMIT_AVG_F64: the sum word holds an f64 (else i64)
  uint8_t is_order_key;// value is stored as a totalOrder key (f64 min/max): decode on emit
  void* values;
  uint8_t* valid_bytes;  // one byte per row (packed to bits by pack_valid_kernel), null for non-nullable columns
};
constexpr int EMIT_MAX_COLS = 40;
struct EmitTable { int32_t ncols; EmitCol col[EMIT_MAX_COLS]; };

// frozen-row (reference Binary accumulator column) field descriptors
// FZ_BOOL (AccBooleanColumn, acc.rs:180-207): one byte, 0 = NULL, else 1 + value.  With `valid` it is a Boolean value;
// without, it is FIRST's flag over an int8 0/1 column (set: byte 2; any non-zero byte reads back as set)
enum FrozenKind : uint8_t { FZ_PRIM = 0, FZ_COUNT = 1, FZ_BOOL = 2 };
struct FrozenField {
  uint8_t kind;        // FZ_PRIM: [u8 valid][LE value if valid] (acc.rs:335-346); FZ_COUNT: varint (count.rs:193-203); FZ_BOOL above
  uint8_t width;       // value bytes of FZ_PRIM (1,2,4,8,16)
  uint8_t phys;        // physical type of the state column
  uint8_t _pad;
  const void* values;      // freeze: state column values;      unfreeze: output
  const uint8_t* valid;    // freeze: validity bytes or null;   unfreeze: output validity bytes
};
constexpr int FROZEN_MAX_FIELDS = 32;
struct FrozenTable { int32_t nfields; FrozenField f[FROZEN_MAX_FIELDS]; };

// launchers (kernels.cu); every launcher returns the number of kernels it launched
int launch_filter_project(const VmProgram* d_prog, const ColTable& cols, const OutTable& outs, int nouts, int64_t n,
                          bool has_filters, unsigned long long* d_tile_status, unsigned long long* d_scratch /*[0]=tile ctr,[1]=out count,[2]=err*/,
                          cudaStream_t s);
int64_t filter_project_num_tiles(int64_t n);

// lean FilterExec/ProjectExec kernel: non-null int64 columns, `col cmp literal` conjuncts, projections that are a
// column or `column (+|-|*) column|literal`
struct LeanFpSpec {
  int32_t nfilt, nout;
  struct { int8_t col; uint8_t op; uint8_t _pad[6]; long long lit; } filt[4];
  struct { uint8_t kind; int8_t a; int8_t b; uint8_t _pad[5]; long long lit; } out[8];   // kind 0: col a; 1: a+b 2: a-b 3: a*b (b<0: literal)
};
int launch_filter_project_lean(const ColTable& cols, int ncols /*1..4, every one referenced*/, const LeanFpSpec& sp, long long* const* out_values, int64_t n,
                               void* d_work /* filter_project_lean_scratch_bytes(n) bytes, zeroed */, unsigned long long* d_scratch, cudaStream_t s);
int64_t filter_project_lean_scratch_bytes(int64_t n);

// ord_base: rows the op fed to the aggregate before this batch; row i of the batch has the arrival ordinal ord_base + i (FIRST)
int launch_agg_update(const VmProgram* d_prog, const ColTable& cols, const AggLayout& lay, const AggTable& tab, int64_t row_begin, int64_t n,
                      const uint32_t* d_row_list /*replay of deferred rows, or null*/, uint64_t ord_base, cudaStream_t s);
// grouping sets: d_row_list entries (and the deferred entries it writes) are row * nsets + set; n counts rows, or list entries.
// The arrival ordinal of (row, set) is (ord_base + row) * nsets + set
int launch_agg_update_sets(const VmProgram* d_prog, const ColTable& cols, const AggLayout& lay, const AggTable& tab, int64_t row_begin, int64_t n,
                           const uint32_t* d_row_list, const AggSetDesc* d_sets, int nsets, uint64_t ord_base, cudaStream_t s);
int launch_agg_rehash(const AggLayout& lay, const AggTable& old_tab, const AggTable& new_tab, cudaStream_t s);
int launch_agg_emit(const AggLayout& lay, const AggTable& tab, const EmitTable& emit, unsigned long long* d_out_count, cudaStream_t s);
// n (<= 32) words from device memory into pinned host memory (cudaMallocHost: addressable from the device at the same address), in
// stream order and without a copy-engine operation: a D2H copy between two kernels of a stream leaves a bubble before the next one
int launch_copy_words_to_host(const unsigned long long* src, unsigned long long* pinned_dst, int n, cudaStream_t s);
int launch_pack_valid(const uint8_t* bytes, uint32_t* bits, int64_t n, cudaStream_t s);
int launch_frozen_lengths(const FrozenTable& ft, int64_t n, int32_t* lengths, cudaStream_t s);
int launch_exclusive_scan_i32(const int32_t* in, int32_t* out /* n+1 entries */, int64_t n, int32_t* d_block_sums, cudaStream_t s);
int launch_frozen_write(const FrozenTable& ft, int64_t n, const int32_t* offsets, uint8_t* data, cudaStream_t s);
int launch_frozen_read(const FrozenTable& ft, int64_t n, const int32_t* offsets, int64_t offsets_base, const uint8_t* data, int* d_err, cudaStream_t s);
int launch_murmur3_partition(const ColTable& cols, const uint8_t* phys, int ncols, int64_t n, int32_t num_partitions, uint32_t* out, cudaStream_t s);
int64_t scan_num_blocks(int64_t n);

// variable-width (Utf8 / Binary) column gather: output row i is source row sel[i] (sel null: row i).  `src` is a DevCol whose
// `offsets` are already advanced by the Arrow offset.  Pass 1 writes the lengths, the gathered validity bits (when `out_valid`)
// and adds the total byte count to *d_total; pass 2 (after launch_exclusive_scan_i32 of the lengths) copies the bytes.
int launch_varlen_lengths(const DevCol& src, const uint32_t* sel, int64_t m, int32_t* lengths, uint32_t* out_valid, unsigned long long* d_total, cudaStream_t s);
int launch_varlen_copy(const DevCol& src, const uint32_t* sel, int64_t m, const int32_t* out_offsets, uint8_t* out_data, cudaStream_t s);

// IpcReaderExec decode (ipc_source.cu drives them): batch_serde records -> coalesced columns
constexpr int IPC_TILE = 1024;                 // rows of one (record, column) tile of ipc_decode_fixed_kernel
constexpr int IPC_COPY_PIECE = 32768;          // bytes of one piece of ipc_decode_bytes_kernel
struct IpcFixedJob { const uint8_t* src; uint8_t* dst; int64_t rows; int32_t width; int32_t _pad; };   // src: `width` planes; dst: the record's first output value
struct IpcTile { int32_t job; int32_t row0; };
struct IpcBitCol { uint32_t* dst; const uint8_t* const* src; };   // src: per record, its bitmap in the stream, or null (all bits set)
struct IpcCopy { const uint8_t* src; uint8_t* dst; int64_t len; };
int launch_ipc_decode_fixed(const IpcFixedJob* jobs, const IpcTile* tiles, int64_t ntiles, cudaStream_t s);
int launch_ipc_decode_bits(const IpcBitCol* cols, int ncols, const int64_t* rec_row /* nrec + 1 output row starts */, int64_t nrec, int64_t rows, cudaStream_t s);
int launch_ipc_decode_bytes(const IpcCopy* copies, int64_t n, cudaStream_t s);

}  // namespace b200q
