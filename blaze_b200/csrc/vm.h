// Expression bytecode shared by the host compiler (compile.cc) and the device interpreter (vm.cuh).
//
// One program evaluates, per input row: the conjuncts of the fused FilterExec chain (VM_FILTER after
// each — CachedExprsEvaluator::filter_impl, cached_exprs_evaluator.rs:90-136), then the projections /
// grouping keys / aggregate arguments (VM_OUT).  It is a typed stack machine: every value is one
// 64-bit slot (ints/bool/date/timestamp sign-extended to i64; f32/f64 as an f64) or two slots
// (decimal128 lo,hi; a Utf8 string {byte pointer, length}) plus one validity bit per slot (a two-slot
// value's validity is the bit of its first slot).  There is no control flow: CASE compiles to
// VM_SELECT, so R rows per thread run in lockstep and the program counter is warp-uniform.
#pragma once
#include <cstdint>

namespace b200q {

enum VmOp : uint8_t {
  VM_END = 0,
  VM_LOAD_COL,        // a = PhysKind, b = column slot                 -> push 1|2
  VM_LOAD_LIT,        // a = bit0 null, bit1 two-slot; c = pool index   -> push 1|2
  VM_ADD_I, VM_SUB_I, VM_MUL_I, VM_DIV_I, VM_MOD_I,         // a = bit width (8/16/32/64), wrapping
  VM_ADD_F, VM_SUB_F, VM_MUL_F, VM_DIV_F, VM_MOD_F,         // a = 1: round the result to f32
  VM_ADD_DEC, VM_SUB_DEC,                                   // c = pool{lmul lo,hi, rmul lo,hi}
  VM_CMP_I, VM_CMP_F, VM_CMP_DEC,                           // a = CmpOp
  VM_AND, VM_OR, VM_NOT,
  VM_IS_NULL, VM_IS_NOT_NULL,                               // a = slots of the operand
  VM_BIT_AND, VM_BIT_OR, VM_BIT_XOR,
  VM_NEG_I, VM_NEG_F, VM_NEG_DEC,                           // a = bit width for NEG_I
  VM_CAST_I_I,        // a = target bits; NULL on overflow (arrow safe cast)
  VM_CAST_I_F,        // a = 1: to f32
  VM_CAST_F_I,        // a = target bits; Rust `as`: truncate, saturate, NaN -> 0 (commons cast.rs:54-95)
  VM_CAST_F_F32,      // round to f32
  VM_CAST_I_BOOL, VM_CAST_F_BOOL,
  VM_CAST_I_DEC,      // c = pool{mul lo,hi, limit lo,hi}
  VM_CAST_DEC_DEC,    // a = 0 none / 1 scale down (round half away) / 2 scale up; c = pool{factor lo,hi, limit lo,hi}
  VM_CAST_DEC_I,      // a = target bits; c = pool{div lo,hi}
  VM_CAST_DEC_F,      // a = 1: to f32; c = pool{double divisor}
  VM_CAST_F_DEC,      // c = pool{double mul, limit lo,hi}
  VM_UNSCALED,        // decimal -> i64 (low 64 bits)         spark_unscaled_value.rs:24-42
  VM_MAKE_DEC,        // i64 -> decimal, no range check       spark_make_decimal.rs:24-58
  VM_CHECK_OVERFLOW,  // a = 0 same scale / 1 down (half up) / 2 up (wrapping mul); c = pool{factor lo,hi, limit lo,hi}; b=1: identity
  VM_NULL_IF_ZERO_I, VM_NULL_IF_ZERO_F, VM_NULL_IF_ZERO_DEC,
  VM_NULLIFY,         // a = value slots: pops bool m, value v -> v with validity cleared where m is true
  VM_NORM_NAN_ZERO,   // a = 1: f32
  VM_SELECT,          // a = value slots: pops else, then, cond -> (cond valid && true) ? then : else
  VM_IN_LIST,         // a = bits: 0-1 kind (0 int,1 float,2 dec,3 utf8), bit2 negated, bit3 list has a NULL item; b = count; c = pool index
  VM_FILTER,          // pops bool: row stays alive iff valid && true (null -> false, :518-520)
  VM_COMPACT,         // FilterExec/ProjectExec kernel only: all predicates done, compute output positions
  VM_OUT,             // a = OutKind, b = output index: pops the value
  // Utf8 (operands are {pointer, length} pairs; byte loops run inside one instruction, the pc stays warp-uniform)
  VM_CMP_STR,         // a = CmpOp: unsigned byte-lexicographic, a proper prefix sorts first (arrow Utf8 cmp)
  VM_STARTS_WITH, VM_ENDS_WITH, VM_CONTAINS,               // pops pattern, string -> bool; an empty pattern matches
  VM_CAST_STR_I,      // a = target bits: Spark UTF8String.toLong/toInt (commons cast.rs:287-361); NULL on bad input
  VM_LOAD_STR,        // b = column slot: pushes {pointer into the data, length} of a Utf8 column
  VM_OUT_SEL,         // b = output index: the source row of the (surviving) row, for the variable-width gathers
  // Spark's runtime bloom filters (only the generic VM kernels run programs that use these)
  VM_XXHASH64,        // a = PhysKind of the operand: pops value, i64 seed -> xxhash64(value, seed); a NULL value leaves the seed
  VM_BLOOM_PROBE,     // c = pool{device address of the bit words, bit size, k}: pops an i64 -> might_contain_long; NULL stays NULL
};

enum PhysKind : uint8_t { PH_BOOL = 0, PH_I8, PH_I16, PH_I32, PH_I64, PH_F32, PH_F64, PH_DEC128, PH_STR,
                          PH_SEL };   // VM_OUT_SEL's output: the u32 source row of each surviving row
enum CmpOp : uint8_t { CMP_EQ = 0, CMP_NE, CMP_LT, CMP_LE, CMP_GT, CMP_GE };

struct VmInstr { uint8_t op, a; uint16_t b; uint32_t c; };
static_assert(sizeof(VmInstr) == 8, "VmInstr must be 8 bytes");

constexpr int VM_MAX_CODE = 384;
constexpr int VM_MAX_POOL = 256;
constexpr int VM_MAX_DEPTH = 16;
constexpr int VM_MAX_COLS = 32;     // distinct input columns referenced by one program
constexpr int VM_MAX_OUT = 32;      // outputs (projection columns, or key words + agg args)
constexpr int VM_MAX_STR_POOL = 4096;   // bytes of Utf8 literals, patterns and IN-list items per program

struct VmProgram {
  uint32_t n_code, n_pool, n_filters, max_depth;
  VmInstr code[VM_MAX_CODE];
  uint64_t pool[VM_MAX_POOL];
  // Utf8 constants: the pool holds {device address into str_pool, length} pairs for them (relocated at upload)
  uint32_t n_str, _pad;
  uint8_t str_pool[VM_MAX_STR_POOL];
};

// One input column as seen by a kernel launch (Arrow buffers; `validity` may be null).
struct DevCol {
  const void* values;        // already advanced by the Arrow offset for byte-addressable types
  const uint8_t* validity;   // bit-packed, LSB first
  uint32_t bit_offset;       // Arrow offset for validity (and for bit-packed bool values)
  uint32_t _pad;
  const int32_t* offsets;    // Utf8 / Binary: Arrow offsets advanced by the Arrow offset; they index `values` (the data base)
};
struct ColTable { DevCol col[VM_MAX_COLS]; };

// outputs of the FilterExec / ProjectExec kernel
struct OutTable {
  void* values[VM_MAX_OUT];
  uint32_t* validity[VM_MAX_OUT];   // pre-zeroed bitmaps, or null when the column is non-nullable
  uint8_t phys[VM_MAX_OUT];
};

}  // namespace b200q
