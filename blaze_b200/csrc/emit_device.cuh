// Emission of one group's output columns (typed results / state columns), shared by the hashed-table emit kernel
// (kernels.cu) and the dense-table emit kernels (kernels_fast.cu, kernels_tile.cu): the caller presents the group as a
// key entry [hdr][key words...], an accumulator entry in AggLayout word order and the header flags.
#pragma once
#include "kernels.cuh"
#include "vm.cuh"

namespace b200q {

// AVG results from (sum, count != 0): f64 division, and i128::checked_div_euclid for decimals (avg.rs:158-165)
__device__ __forceinline__ double avg_f64_final(double sum, long long cnt) { return sum / __ll2double_rn(cnt); }
__device__ __forceinline__ i128_t avg_dec_final(i128_t sum, long long cnt) {
  i128_t q = sum / cnt; const i128_t r = sum % cnt;
  if (r < 0) q += cnt > 0 ? -1 : 1;
  return q;
}

__device__ __forceinline__ void emit_store(const EmitCol& c, unsigned long long at, uint64_t lo, uint64_t hi, bool valid) {
  if (c.valid_bytes) c.valid_bytes[at] = valid ? 1 : 0;
  switch (c.phys) {
    case PH_BOOL: ((uint8_t*)c.values)[at] = lo != 0; break;          // bytes; packed to bits by pack_valid_kernel
    case PH_I8: ((int8_t*)c.values)[at] = (int8_t)lo; break;
    case PH_I16: ((int16_t*)c.values)[at] = (int16_t)lo; break;
    case PH_I32: ((int32_t*)c.values)[at] = (int32_t)lo; break;
    case PH_I64: case PH_F64: ((uint64_t*)c.values)[at] = lo; break;
    case PH_F32: ((float*)c.values)[at] = (float)as_f64(lo); break;
    default: ((uint64_t*)c.values)[2 * at] = lo; ((uint64_t*)c.values)[2 * at + 1] = hi; break;
  }
}


__device__ __forceinline__ void emit_row_columns(const EmitTable& emit, unsigned long long at, const unsigned long long* ke, const unsigned long long* slot, unsigned flags) {
  for (int c = 0; c < emit.ncols; c++) {
      const EmitCol ec = emit.col[c];
      switch (ec.kind) {
        case EMIT_KEY: {
          const bool valid = !((flags >> (16 + ec.key)) & 1);
          emit_store(ec, at, ke[ec.word], ec.phys == PH_DEC128 ? ke[ec.word + 1] : 0, valid);
          break;
        }
        case EMIT_ACC_VALUE: {
          const bool valid = ec.vbit == 0xFF ? true : ((flags >> ec.vbit) & 1);
          uint64_t lo = slot[ec.word];
          if (ec.is_order_key) lo = (uint64_t)total_order_key(lo);               // the key transform is an involution
          emit_store(ec, at, valid ? lo : 0, (valid && ec.phys == PH_DEC128) ? slot[ec.word + 1] : 0, valid);
          break;
        }
        case EMIT_AVG_F64: {
          const long long cnt = (long long)slot[ec.word2];
          const bool valid = (ec.vbit == 0xFF ? true : ((flags >> ec.vbit) & 1)) && cnt != 0;
          const double sum = ec.sum_is_f64 ? as_f64(slot[ec.word]) : __ll2double_rn((long long)slot[ec.word]);
          emit_store(ec, at, valid ? f64_bits(avg_f64_final(sum, cnt)) : 0, 0, valid);
          break;
        }
        case EMIT_FIRST_VALUE: {
          const bool valid = slot[ec.word2] != ~0ULL && (ec.vbit == 0xFF || ((flags >> ec.vbit) & 1));
          emit_store(ec, at, valid ? slot[ec.word] : 0, (valid && ec.phys == PH_DEC128) ? slot[ec.word + 1] : 0, valid);
          break;
        }
        case EMIT_FIRST_FLAG: emit_store(ec, at, slot[ec.word2] != ~0ULL ? 1 : 0, 0, true); break;
        default: {   // EMIT_AVG_DEC: i128::checked_div_euclid(sum, count) (avg.rs:158-165)
          const long long cnt = (long long)slot[ec.word2];
          const bool valid = (ec.vbit == 0xFF ? true : ((flags >> ec.vbit) & 1)) && cnt != 0;
          const i128_t q = valid ? avg_dec_final(mk128(slot[ec.word], slot[ec.word + 1]), cnt) : 0;
          emit_store(ec, at, lo64(q), hi64(q), valid);
          break;
        }
      }
    }
}

}  // namespace b200q
