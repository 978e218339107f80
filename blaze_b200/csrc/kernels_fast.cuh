// Descriptors of the specialised HashAgg update kernels (kernels_fast.cu).
#pragma once
#include <cstddef>

#include "kernels.cuh"

namespace b200q {

enum FastAccKind : uint8_t { FAST_ACC_ADD = 0, FAST_ACC_COUNT = 1 };   // COUNT with col < 0 is COUNT(*)

// the `col cmp literal` conjuncts on one column merged into one closed interval: a row passes iff (u64)(x - lo) <= span
struct FilterInterval { int8_t col; uint8_t phys; uint8_t _pad[6]; long long lo; unsigned long long span; };

struct FastSpec {
  int32_t nkeys, nacc, nfilt, dense;
  int32_t lean, hot_cache;                                // lean: all referenced columns are aligned non-null int64 (set per launch); hot_cache: skewed keys (experimental)
  int8_t key_col[2]; uint8_t key_phys[2];                 // program column slots / physical kinds of the key columns
  struct { uint8_t kind; int8_t col; uint8_t phys; uint8_t vbit; uint8_t word; uint8_t _pad[3]; } acc[2];
  struct { int8_t col; uint8_t phys; uint8_t op; uint8_t _pad[5]; long long lit; } filt[4];
  // the same conjuncts merged per column (tile kernels): a row passes iff it lies in every interval
  int32_t nfcol;                                          // -1: the conjuncts cannot be merged (a `!=` term or more than 2 columns): a dense table takes the row kernels
  int32_t filt_never;                                     // the merged intervals are empty: no row passes
  FilterInterval frange[2];
  long long dense_base;                                   // DENSE: entry index = key0 - dense_base                      (one key)
  unsigned long long dense_cap;                           // entries of dense_stride words
  long long dense_base1;                                  //        entry index = (key0 - dense_base) * dense_r1 + (key1 - dense_base1)   (two keys),
                                                          //        or (key1 - dense_base1) * dense_cap0 + (key0 - dense_base) with dense_key0_minor
  unsigned long long dense_r1, dense_cap0;                // key1 - dense_base1 < dense_r1, key0 - dense_base < dense_cap0; dense_cap = dense_cap0 * dense_r1
  unsigned long long* dense_tab;
  int8_t dense_stride;                                    // 2 or 4 words per entry (= lanes that update one entry in one instruction)
  int8_t dense_word_src[4];                               // per entry word: -1 row counter (+1), -2 padding (+0), j accumulator j, 2+j valid arguments of accumulator j
  uint8_t dense_presence_word;                            // word that is non-zero iff the entry holds a group
  uint8_t dense_key0_minor;                               // two keys: key0 varies fastest in the entry index (set when key1 has the shorter span)
  uint8_t _pad1;
  unsigned long long* sink;                               // FAST_SINK_WARPS x 4 words: per-warp scratch sector for no-op REDs
};
constexpr int FAST_SINK_WARPS = 4096;

// per emit column: which dense word holds the value and which (count) word validates it
struct DenseEmitMap { uint8_t word[EMIT_MAX_COLS]; uint8_t valid_word[EMIT_MAX_COLS]; };

// entry of the two-key offsets d0 < dense_cap0, d1 < dense_r1
__device__ __forceinline__ unsigned long long dense_entry2(const FastSpec& fs, unsigned long long d0, unsigned long long d1) {
  return fs.dense_key0_minor ? d1 * fs.dense_cap0 + d0 : d0 * fs.dense_r1 + d1;
}
// dense entry index of a row; false: outside the dense range (the row goes to a hashed slot)
template <int NK>
__device__ __forceinline__ bool dense_index_of(const FastSpec& fs, long long k0, long long k1, unsigned long long& idx) {
  const unsigned long long d0 = (unsigned long long)(k0 - fs.dense_base);
  if (NK == 1) { idx = d0; return d0 < fs.dense_cap; }
  const unsigned long long d1 = (unsigned long long)(k1 - fs.dense_base1);
  idx = dense_entry2(fs, d0, d1);
  return d0 < fs.dense_cap0 && d1 < fs.dense_r1;
}

// ---------------------------------------------------------------------------------------------------
// WIDE tile aggregates (kernels_tile.cu, round 2): the accumulator kinds the specialised family did not cover — f64
// SUM / AVG, decimal128 SUM / AVG, integer and f64 MIN / MAX, any mix of up to 4 of them over at most two argument
// columns — on a DENSE table whose entry words all take the SAME RED flavour, so that one instruction still updates the
// G (2, 4 or 8) words of 32 / G rows:
//   TF_ADD_U64  SUM(int) | COUNT | decimal128 SUM kept carry-free as three words (low 32 bits, middle 32 bits, high 64
//               bits: 64-bit wrapping adds of 32-bit pieces cannot lose a carry for 2^31 rows; the host normalises the
//               pieces before that and before the emit)
//   TF_ADD_F64  SUM(f64) | SUM(TryCast(int -> f64)) (= Spark AVG(long)) | COUNT kept as an exact f64 integer
//   TF_MIN_S64  MIN(x) | MAX(x) kept as MIN(~x) | presence / valid-argument marks kept as MIN(0) (identity INT64_MAX);
//               f64 values enter as IEEE totalOrder keys
// NULL / out-of-range keys fall back to the hashed table with the generic accumulator updates of AggLayout.
// ---------------------------------------------------------------------------------------------------
enum TileFlavour : uint8_t { TF_ADD_U64 = 0, TF_ADD_F64 = 1, TF_MIN_S64 = 2 };
// identity of a flavour's RED: the fill of every dense word and the value a gated-off lane adds.  f64 words start at -0.0,
// the identity of IEEE addition (-0.0 + x == x for every x): a group whose values are all -0.0 sums to -0.0, as the
// reference's store-the-first-value-then-add does, where +0.0 would turn it into +0.0.  Marks and counts are therefore
// tested as doubles under TF_ADD_F64 (tw_marked), not as integers
__host__ __device__ constexpr unsigned long long tile_identity(int flavour) {
  return flavour == TF_MIN_S64 ? 0x7FFFFFFFFFFFFFFFULL : flavour == TF_ADD_F64 ? 0x8000000000000000ULL : 0ULL;
}
enum TileArgCvt : uint8_t { TC_NONE = 0, TC_I2F = 1 /* integer -> f64 bits */, TC_ORDER = 2 /* f64 bits -> totalOrder key */ };
enum TileRecon : uint8_t { TR_COPY = 0 /* slot word = dense word */, TR_NOT = 1 /* ~dense word (a maximum kept as the minimum of the complement) */,
                           TR_F2I = 2 /* count kept as f64 */, TR_DEC3 = 3 /* three carry-free pieces -> {lo, hi} */ };
struct TileWord {                                         // value a lane adds to its entry word: (((srcsel ? v1 : v0) >> sh) & msk) ^ inv, or cst; gated by a pk bit
  uint8_t srcsel;                                         // 0: argument register v0, 1: v1, 2: the constant cst
  uint8_t sh;                                             // 0 or 32
  uint8_t gate;                                           // pk bit that must be set: 28 / 29 = argument 0 / 1 is not NULL, 30 = always
  uint8_t _pad[5];
  unsigned long long msk, inv, cst;
};
struct TileAggSpec {
  int32_t nkeys, nargs, nfcol, filt_never, nacc, G, flavour, arg_is_dec;
  int8_t key_col[2]; uint8_t key_phys[2];
  int8_t arg_col[2]; uint8_t arg_phys[2]; uint8_t arg_cvt[2]; uint8_t arg_values[2];      // arg_values: 0 = only the validity is needed (COUNT(col))
  FilterInterval frange[2];
  long long dense_base, dense_base1;
  unsigned long long dense_cap, dense_r1, dense_cap0;
  unsigned long long* dense_tab;
  unsigned long long* sink;
  unsigned long long dec_mul;                             // decimal argument: 10^(scale increase) of the TryCast below the SUM / AVG (Spark AVG(decimal(p,s)) accumulates at (p+4, s+4)); 1: none
  TileWord word[8];
  uint8_t presence_word, dec_word /* first of the three decimal pieces, 0xFF: none */, _pad2[6];
  struct { int8_t arg; uint8_t recon; uint8_t w0; uint8_t valid_word; uint8_t lay_acc; uint8_t _pad[3]; } acc[4];
};
// the kernels take both descriptors by value as launch parameters: a change of size or interval offset must be deliberate
static_assert(sizeof(FastSpec) == 232 && offsetof(FastSpec, frange) == 120, "FastSpec layout");
static_assert(sizeof(TileAggSpec) == 456 && offsetof(TileAggSpec, frange) == 48, "TileAggSpec layout");

int launch_agg_tile_wide(const ColTable& cols, const TileAggSpec& ts, const AggLayout& lay, const AggTable& tab, int64_t row_begin, int64_t n, cudaStream_t s);
int launch_tile_wide_init(const TileAggSpec& ts, cudaStream_t s);                       // identities of the dense entries
int launch_tile_wide_count(const TileAggSpec& ts, unsigned long long* d_out, cudaStream_t s);
int launch_tile_wide_normalise(const TileAggSpec& ts, cudaStream_t s);                  // carry the decimal pieces (no-op without a decimal SUM)
int launch_tile_wide_emit(const TileAggSpec& ts, const AggLayout& lay, const EmitTable& emit, unsigned long long* d_out_count, cudaStream_t s);

int launch_agg_tile_dense(const ColTable& cols, const FastSpec& fs, const AggLayout& lay, const AggTable& tab, int64_t row_begin, int64_t n, cudaStream_t s);
int launch_agg_fast_update(const ColTable& cols, const FastSpec& fs, const AggLayout& lay, const AggTable& tab, int64_t row_begin, int64_t n, cudaStream_t s);
int launch_key_skew_probe(const DevCol* key_cols, const uint8_t* phys, int nkeys, int64_t n, unsigned* d_hist /* 65536 + 1 words, zeroed */, cudaStream_t s);
int launch_key_range(const DevCol& col, int phys, int64_t n, long long* d_out, cudaStream_t s);
int launch_agg_emit_dense(const FastSpec& fs, const EmitTable& emit, const DenseEmitMap& map, unsigned long long* d_out_count, cudaStream_t s);
int launch_dense_count(const FastSpec& fs, unsigned long long* d_out, cudaStream_t s);

}  // namespace b200q
