// Device interpreter of the expression bytecode (vm.h).  R rows per thread run in lockstep, so the
// program counter and stack pointer are warp-uniform: instruction fetches are shared-memory
// broadcasts and the (local-memory) stack accesses are perfectly coalesced.
//
// Semantics follow the reference (DataFusion 49 / arrow-rs 55.2 as the reference pins them), restated for the tests in oracle/blaze_oracle.py:
// expression evaluation as used by CachedExprsEvaluator (cached_exprs_evaluator.rs:90-166).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "hash.cuh"
#include "vm.h"

namespace b200q {

typedef __int128 i128_t;
typedef unsigned __int128 u128_t;

#define B200Q_ERR_FLAG_DIV_ZERO 1
#define B200Q_ERR_FLAG_OVERFLOW 2

__device__ __forceinline__ i128_t mk128(uint64_t lo, uint64_t hi) { return (i128_t)(((u128_t)hi << 64) | (u128_t)lo); }
__device__ __forceinline__ uint64_t lo64(i128_t v) { return (uint64_t)v; }
__device__ __forceinline__ uint64_t hi64(i128_t v) { return (uint64_t)((u128_t)v >> 64); }
__device__ __forceinline__ int64_t sext(int64_t v, int bits) { int s = 64 - bits; return (v << s) >> s; }
__device__ __forceinline__ int64_t total_order_key(uint64_t b) { int64_t x = (int64_t)b; return x ^ ((x >> 63) & 0x7FFFFFFFFFFFFFFFLL); }
__device__ __forceinline__ double as_f64(uint64_t b) { return __longlong_as_double((long long)b); }
__device__ __forceinline__ uint64_t f64_bits(double d) { return (uint64_t)__double_as_longlong(d); }

// correctly rounded i128 -> f64 (Rust `i128 as f64`)
__device__ __forceinline__ double i128_to_double(i128_t v) {
  bool neg = v < 0;
  u128_t m = neg ? (u128_t)(-(v + 1)) + 1 : (u128_t)v;
  uint64_t h = (uint64_t)(m >> 64), l = (uint64_t)m;
  double d;
  if (h == 0) d = __ull2double_rn(l);
  else {
    int lz = __clzll((long long)h);                 // h != 0
    int shift = 64 - lz;                            // bits to drop so that the top 64 bits remain
    uint64_t top = (uint64_t)(m >> shift);
    u128_t dropped = m & ((((u128_t)1) << shift) - 1);
    if (dropped != 0) top |= 1;                     // sticky bit: 64 -> 53 bit rounding stays exact
    d = ldexp(__ull2double_rn(top), shift);
  }
  return neg ? -d : d;
}

// f64 (already integral, finite) -> i128; *ok=false when out of range
__device__ __forceinline__ i128_t double_to_i128(double r, bool* ok) {
  *ok = true;
  double a = fabs(r);
  if (a < 9.2e18) return (i128_t)(long long)r;
  if (!(a < 1.7014118346046923e38)) { *ok = false; return 0; }
  int e; double fr = frexp(a, &e);                   // a = fr * 2^e, fr in [0.5,1)
  uint64_t mant = (uint64_t)ldexp(fr, 64);           // top 64 bits
  u128_t m = e >= 64 ? ((u128_t)mant << (e - 64)) : ((u128_t)mant >> (64 - e));
  return r < 0 ? -(i128_t)m : (i128_t)m;
}

// overflow-checked i128 arithmetic (the __builtin_*_overflow intrinsics are host-only under nvcc)
__device__ __forceinline__ bool mul_of(i128_t a, i128_t f /* > 0 */, i128_t* r) {
  const i128_t mx = (i128_t)((~(u128_t)0) >> 1), mn = -mx - 1;
  *r = (i128_t)((u128_t)a * (u128_t)f);
  return a > mx / f || a < mn / f;
}
__device__ __forceinline__ bool add_of(i128_t a, i128_t b, i128_t* r) {
  *r = (i128_t)((u128_t)a + (u128_t)b);
  return (b >= 0) ? (*r < a) : (*r > a);
}
__device__ __forceinline__ bool sub_of(i128_t a, i128_t b, i128_t* r) {
  *r = (i128_t)((u128_t)a - (u128_t)b);
  return (b >= 0) ? (*r > a) : (*r < a);
}

// ---- Utf8 helpers: {pointer, length} operands, bytes compared as uint8_t ----
__device__ __forceinline__ int str_cmp(const uint8_t* a, uint32_t la, const uint8_t* b, uint32_t lb) {
  const uint32_t m = la < lb ? la : lb;
  for (uint32_t i = 0; i < m; i++) { const int d = (int)a[i] - (int)b[i]; if (d) return d; }
  return la == lb ? 0 : (la < lb ? -1 : 1);                      // a proper prefix sorts first
}
__device__ __forceinline__ bool str_eq(const uint8_t* a, uint32_t la, const uint8_t* b, uint32_t lb) {
  if (la != lb) return false;
  for (uint32_t i = 0; i < la; i++) if (a[i] != b[i]) return false;
  return true;
}
__device__ __forceinline__ bool str_contains(const uint8_t* s, uint32_t ls, const uint8_t* p, uint32_t lp) {
  if (lp > ls) return false;
  for (uint32_t i = 0; i + lp <= ls; i++) if (str_eq(s + i, lp, p, lp)) return true;
  return false;
}
// Spark UTF8String.toLong / toInt as the reference ports it (commons cast.rs:287-361): no trimming, optional sign (a lone sign is
// NULL), digits accumulated negatively and checked against the target width, a '.' ends the integral part and may only be
// followed by digits, which are dropped; any other byte or an overflow is NULL.
__device__ __forceinline__ bool str_to_int(const uint8_t* s, uint32_t n, int bits, int64_t* out) {
  if (n == 0) return false;
  const bool neg = s[0] == '-';
  uint32_t i = 0;
  if (neg || s[0] == '+') { i = 1; if (n == 1) return false; }
  const int64_t mn = bits == 64 ? INT64_MIN : -(1LL << (bits - 1)), stop = mn / 10;
  int64_t r = 0;
  while (i < n) {
    const uint8_t b = s[i++];
    if (b == '.') break;
    if (b < '0' || b > '9') return false;
    if (r < stop) return false;
    r = sext((int64_t)((uint64_t)r * 10u - (uint64_t)(b - '0')), bits);   // wraps like the target type
    if (r > 0) return false;
  }
  for (; i < n; i++) if (s[i] < '0' || s[i] > '9') return false;
  if (!neg) { r = sext((int64_t)(0 - (uint64_t)r), bits); if (r < 0) return false; }
  *out = r;
  return true;
}
#define STRP(x) ((const uint8_t*)(uintptr_t)(x))

struct NullSink { template <class... A> __device__ void out(A...) {} };

#define VALID(r, i) ((vm[r] >> (i)) & 1u)
#define SETV(r, i, ok) vm[r] = (vm[r] & ~(1u << (i))) | ((uint32_t)((ok) ? 1u : 0u) << (i))
#define FORR _Pragma("unroll") for (int r = 0; r < R; r++)

// The Utf8 instructions (VM_CMP_STR, VM_STARTS_WITH / ENDS_WITH / CONTAINS, VM_CAST_STR_I, VM_IN_LIST kind 3).  Returns the new
// stack pointer.
template <int R>
__device__ __forceinline__ int vm_str(const VmInstr in, const uint64_t* __restrict__ pool, uint64_t (&st)[VM_MAX_DEPTH][R], uint32_t (&vm)[R], int sp) {
  switch (in.op) {
    case VM_CMP_STR: {
      sp -= 3;
      FORR {
        const bool ok = VALID(r, sp - 1) && VALID(r, sp + 1);
        const int c = ok ? str_cmp(STRP(st[sp - 1][r]), (uint32_t)st[sp][r], STRP(st[sp + 1][r]), (uint32_t)st[sp + 2][r]) : 0;
        bool v;
        switch (in.a) { case CMP_EQ: v = c == 0; break; case CMP_NE: v = c != 0; break; case CMP_LT: v = c < 0; break;
                        case CMP_LE: v = c <= 0; break; case CMP_GT: v = c > 0; break; default: v = c >= 0; }
        st[sp - 1][r] = v; SETV(r, sp - 1, ok);
      }
      return sp;
    }
    case VM_STARTS_WITH: case VM_ENDS_WITH: case VM_CONTAINS: {
      sp -= 3;
      FORR {
        const bool ok = VALID(r, sp - 1);
        const uint8_t* s = STRP(st[sp - 1][r]); const uint32_t ls = (uint32_t)st[sp][r];
        const uint8_t* p = STRP(st[sp + 1][r]); const uint32_t lp = (uint32_t)st[sp + 2][r];
        bool v = false;
        if (ok) {
          if (in.op == VM_CONTAINS) v = str_contains(s, ls, p, lp);
          else v = lp <= ls && str_eq(in.op == VM_STARTS_WITH ? s : s + (ls - lp), lp, p, lp);
        }
        st[sp - 1][r] = v; SETV(r, sp - 1, ok);
      }
      return sp;
    }
    case VM_CAST_STR_I: {
      sp -= 1;
      FORR {
        int64_t v = 0;
        const bool ok = VALID(r, sp - 1) && str_to_int(STRP(st[sp - 1][r]), (uint32_t)st[sp][r], in.a, &v);
        st[sp - 1][r] = ok ? (uint64_t)v : 0; SETV(r, sp - 1, ok);
      }
      return sp;
    }
    default: {                     // VM_IN_LIST over Utf8
      const bool neg = in.a & 4, has_null = in.a & 8;
      const int ix = sp - 2;
      FORR {
        bool found = false;
        if (VALID(r, ix)) for (int k = 0; k < in.b && !found; k++) found = str_eq(STRP(st[ix][r]), (uint32_t)st[ix + 1][r], STRP(pool[in.c + 2 * k]), (uint32_t)pool[in.c + 2 * k + 1]);
        const bool ok = VALID(r, ix) && (found || !has_null);
        st[ix][r] = found != neg; SETV(r, ix, ok);
      }
      return ix + 1;
    }
  }
}

// VM_XXHASH64 (spark_hash.rs create_xxhash64_hashes: Bool / Int8 / Int16 / Int32 / Date32 hash as a 4-byte int, Int64 /
// Timestamp as an 8-byte long, Utf8 over its bytes) and VM_BLOOM_PROBE (SparkBloomFilter::might_contain_long).  Returns the new
// stack pointer.
template <int R>
__device__ __forceinline__ int vm_bloom(const VmInstr in, const uint64_t* __restrict__ pool, uint64_t (&st)[VM_MAX_DEPTH][R], uint32_t (&vm)[R], int sp) {
  if (in.op == VM_XXHASH64) {
    const int is = sp - (in.a == PH_STR ? 3 : 2);   // the seed; the value above it
    FORR {
      uint64_t h = st[is][r];
      if (VALID(r, is + 1)) {
        const uint64_t v = st[is + 1][r];
        if (in.a == PH_STR) h = xxh64_bytes(STRP(v), (uint32_t)st[is + 2][r], h);
        else if (in.a == PH_I64) h = xxh64_long(v, h);
        else h = xxh64_int((uint32_t)v, h);
      }
      st[is][r] = h;
    }
    return is + 1;
  }
  const uint64_t* __restrict__ bits = (const uint64_t*)(uintptr_t)pool[in.c];
  const int32_t bit_size = (int32_t)pool[in.c + 1], k = (int32_t)pool[in.c + 2];
  FORR {
    bool v = false;
    if (VALID(r, sp - 1)) {
      const int64_t x = (int64_t)st[sp - 1][r];
      const int32_t h1 = mm3_hash_long(x, 0), h2 = mm3_hash_long(x, h1);
      v = true;
      for (int32_t i = 1; i <= k && v; i++) {
        int32_t c = (int32_t)((uint32_t)h1 + (uint32_t)i * (uint32_t)h2);   // i32 wrapping
        if (c < 0) c = ~c;                                                  // flip all bits if negative
        const uint32_t b = (uint32_t)(c % bit_size);
        v = (__ldg(bits + (b >> 6)) >> (b & 63)) & 1;
      }
    }
    st[sp - 1][r] = v;
  }
  return sp;
}

// Runs from `pc` until VM_END (returns -1) or VM_COMPACT (returns the pc after it).
template <int R, class Sink>
__device__ __forceinline__ int vm_run(const VmInstr* __restrict__ code, const uint64_t* __restrict__ pool, int pc,
                                      const ColTable& cols, const long long (&row)[R], const bool (&inb)[R],
                                      bool (&alive)[R], int* __restrict__ err, Sink& sink) {
  uint64_t st[VM_MAX_DEPTH][R];
  uint32_t vm[R];
  int sp = 0;
#pragma unroll
  for (int r = 0; r < R; r++) vm[r] = 0;

  while (true) {
    const VmInstr in = code[pc++];
    switch (in.op) {
      case VM_END: return -1;
      case VM_COMPACT: return pc;
      case VM_LOAD_COL: {
        const DevCol c = cols.col[in.b];
        FORR {
          uint64_t lo = 0, hi = 0; bool ok = false;
          if (inb[r]) {
            const long long i = row[r];
            ok = true;
            if (c.validity) { const unsigned long long bi = (unsigned long long)i + c.bit_offset; ok = (__ldg(c.validity + (bi >> 3)) >> (bi & 7)) & 1; }
            switch (in.a) {
              case PH_BOOL: { const unsigned long long bi = (unsigned long long)i + c.bit_offset; lo = (__ldg((const uint8_t*)c.values + (bi >> 3)) >> (bi & 7)) & 1; break; }
              case PH_I8: lo = (uint64_t)(int64_t)__ldg((const int8_t*)c.values + i); break;
              case PH_I16: lo = (uint64_t)(int64_t)__ldg((const int16_t*)c.values + i); break;
              case PH_I32: lo = (uint64_t)(int64_t)__ldg((const int32_t*)c.values + i); break;
              case PH_I64: lo = (uint64_t)__ldg((const long long*)c.values + i); break;
              case PH_F32: lo = f64_bits((double)__ldg((const float*)c.values + i)); break;
              case PH_F64: lo = (uint64_t)__ldg((const long long*)c.values + i); break;
              default: lo = (uint64_t)__ldg((const long long*)c.values + 2 * i); hi = (uint64_t)__ldg((const long long*)c.values + 2 * i + 1); break;
            }
          }
          st[sp][r] = lo; SETV(r, sp, ok);
          if (in.a == PH_DEC128) st[sp + 1][r] = hi;
        }
        sp += in.a == PH_DEC128 ? 2 : 1;
        break;
      }
      case VM_LOAD_STR: {          // Utf8 column -> {pointer into the data, length}
        const DevCol c = cols.col[in.b];
        FORR {
          uint64_t p = 0, len = 0; bool ok = false;
          if (inb[r]) {
            const long long i = row[r];
            ok = true;
            if (c.validity) { const unsigned long long bi = (unsigned long long)i + c.bit_offset; ok = (__ldg(c.validity + (bi >> 3)) >> (bi & 7)) & 1; }
            const int32_t o0 = __ldg(c.offsets + i), o1 = __ldg(c.offsets + i + 1);
            p = (uint64_t)(uintptr_t)((const uint8_t*)c.values + o0); len = (uint64_t)(uint32_t)(o1 - o0);
          }
          st[sp][r] = p; st[sp + 1][r] = len; SETV(r, sp, ok);
        }
        sp += 2;
        break;
      }
      case VM_LOAD_LIT: {
        const uint64_t lo = pool[in.c], hi = pool[in.c + 1];
        const bool ok = !(in.a & 1);
        FORR { st[sp][r] = lo; SETV(r, sp, ok); if (in.a & 2) st[sp + 1][r] = hi; }
        sp += (in.a & 2) ? 2 : 1;
        break;
      }
      case VM_ADD_I: case VM_SUB_I: case VM_MUL_I: case VM_DIV_I: case VM_MOD_I: {
        sp -= 1;
        FORR {
          const int64_t a = (int64_t)st[sp - 1][r], b = (int64_t)st[sp][r];
          const bool ok = VALID(r, sp - 1) && VALID(r, sp);
          int64_t v = 0;
          if (in.op == VM_ADD_I) v = (int64_t)((uint64_t)a + (uint64_t)b);
          else if (in.op == VM_SUB_I) v = (int64_t)((uint64_t)a - (uint64_t)b);
          else if (in.op == VM_MUL_I) v = (int64_t)((uint64_t)a * (uint64_t)b);
          else if (ok) {
            // arrow div_checked / mod_checked: errors only on evaluated (alive) valid slots
            const int64_t mn = in.a == 64 ? INT64_MIN : -(1LL << (in.a - 1));
            if (b == 0) { if (alive[r]) atomicOr(err, B200Q_ERR_FLAG_DIV_ZERO); }
            else if (a == mn && b == -1) { if (alive[r]) atomicOr(err, B200Q_ERR_FLAG_OVERFLOW); }
            else v = in.op == VM_DIV_I ? a / b : a % b;
          }
          st[sp - 1][r] = (uint64_t)sext(v, in.a); SETV(r, sp - 1, ok);
        }
        break;
      }
      case VM_ADD_F: case VM_SUB_F: case VM_MUL_F: case VM_DIV_F: case VM_MOD_F: {
        sp -= 1;
        FORR {
          const double a = as_f64(st[sp - 1][r]), b = as_f64(st[sp][r]);
          double v;
          if (in.a) {   // f32 arithmetic done in f32 (operands are exact widenings)
            const float fa = (float)a, fb = (float)b; float fv;
            if (in.op == VM_ADD_F) fv = __fadd_rn(fa, fb); else if (in.op == VM_SUB_F) fv = __fsub_rn(fa, fb);
            else if (in.op == VM_MUL_F) fv = __fmul_rn(fa, fb); else if (in.op == VM_DIV_F) fv = __fdiv_rn(fa, fb); else fv = fmodf(fa, fb);
            v = (double)fv;
          } else {
            if (in.op == VM_ADD_F) v = __dadd_rn(a, b); else if (in.op == VM_SUB_F) v = __dsub_rn(a, b);
            else if (in.op == VM_MUL_F) v = __dmul_rn(a, b); else if (in.op == VM_DIV_F) v = __ddiv_rn(a, b); else v = fmod(a, b);
          }
          st[sp - 1][r] = f64_bits(v); SETV(r, sp - 1, VALID(r, sp - 1) && VALID(r, sp));
        }
        break;
      }
      case VM_ADD_DEC: case VM_SUB_DEC: {
        // arrow-arith decimal_op: rescale both sides, checked i128 arithmetic (error on overflow)
        const i128_t lm = mk128(pool[in.c], pool[in.c + 1]), rm = mk128(pool[in.c + 2], pool[in.c + 3]);
        sp -= 2;
        FORR {
          const bool ok = VALID(r, sp - 2) && VALID(r, sp);
          i128_t v = 0;
          if (ok) {
            const i128_t a = mk128(st[sp - 2][r], st[sp - 1][r]), b = mk128(st[sp][r], st[sp + 1][r]);
            i128_t x, y; bool of = mul_of(a, lm, &x) | mul_of(b, rm, &y);
            of |= in.op == VM_ADD_DEC ? add_of(x, y, &v) : sub_of(x, y, &v);
            if (of) { v = 0; if (alive[r]) atomicOr(err, B200Q_ERR_FLAG_OVERFLOW); }
          }
          st[sp - 2][r] = lo64(v); st[sp - 1][r] = hi64(v); SETV(r, sp - 2, ok);
        }
        break;
      }
      case VM_CMP_I: case VM_CMP_F: {
        sp -= 1;
        FORR {
          int64_t a = (int64_t)st[sp - 1][r], b = (int64_t)st[sp][r];
          if (in.op == VM_CMP_F) { a = total_order_key((uint64_t)a); b = total_order_key((uint64_t)b); }   // arrow cmp: IEEE totalOrder
          bool v;
          switch (in.a) { case CMP_EQ: v = a == b; break; case CMP_NE: v = a != b; break; case CMP_LT: v = a < b; break;
                          case CMP_LE: v = a <= b; break; case CMP_GT: v = a > b; break; default: v = a >= b; }
          st[sp - 1][r] = v; SETV(r, sp - 1, VALID(r, sp - 1) && VALID(r, sp));
        }
        break;
      }
      case VM_CMP_DEC: {
        sp -= 3;
        FORR {
          const i128_t a = mk128(st[sp - 1][r], st[sp][r]), b = mk128(st[sp + 1][r], st[sp + 2][r]);
          bool v;
          switch (in.a) { case CMP_EQ: v = a == b; break; case CMP_NE: v = a != b; break; case CMP_LT: v = a < b; break;
                          case CMP_LE: v = a <= b; break; case CMP_GT: v = a > b; break; default: v = a >= b; }
          st[sp - 1][r] = v; SETV(r, sp - 1, VALID(r, sp - 1) && VALID(r, sp + 1));
        }
        break;
      }
      case VM_AND: case VM_OR: {   // Kleene
        sp -= 1;
        FORR {
          const bool lv = VALID(r, sp - 1), rv = VALID(r, sp), l = st[sp - 1][r] != 0, rr = st[sp][r] != 0;
          bool v, ok;
          if (in.op == VM_AND) { const bool lf = lv && !l, rf = rv && !rr; ok = (lv && rv) || lf || rf; v = lv && rv && l && rr; }
          else { const bool lt = lv && l, rt = rv && rr; ok = (lv && rv) || lt || rt; v = lt || rt; }
          st[sp - 1][r] = v; SETV(r, sp - 1, ok);
        }
        break;
      }
      case VM_NOT: FORR { st[sp - 1][r] = st[sp - 1][r] == 0; } break;
      case VM_IS_NULL: case VM_IS_NOT_NULL: {
        sp -= in.a - 1;
        FORR { const bool ok = VALID(r, sp - 1); st[sp - 1][r] = (in.op == VM_IS_NULL) ? !ok : ok; SETV(r, sp - 1, true); }
        break;
      }
      case VM_BIT_AND: case VM_BIT_OR: case VM_BIT_XOR: {
        sp -= 1;
        FORR {
          const uint64_t a = st[sp - 1][r], b = st[sp][r];
          st[sp - 1][r] = in.op == VM_BIT_AND ? (a & b) : in.op == VM_BIT_OR ? (a | b) : (a ^ b);
          SETV(r, sp - 1, VALID(r, sp - 1) && VALID(r, sp));
        }
        break;
      }
      case VM_NEG_I: FORR { st[sp - 1][r] = (uint64_t)sext((int64_t)(0 - st[sp - 1][r]), in.a); } break;   // neg_wrapping
      case VM_NEG_F: FORR { st[sp - 1][r] ^= 0x8000000000000000ULL; } break;
      case VM_NEG_DEC: FORR { const i128_t v = (i128_t)(0 - (u128_t)mk128(st[sp - 2][r], st[sp - 1][r])); st[sp - 2][r] = lo64(v); st[sp - 1][r] = hi64(v); } break;
      case VM_CAST_I_I: {
        FORR {
          const int64_t v = (int64_t)st[sp - 1][r];
          const bool fits = sext(v, in.a) == v;
          if (!fits) { st[sp - 1][r] = 0; SETV(r, sp - 1, false); }
        }
        break;
      }
      case VM_CAST_I_F: FORR { const long long v = (long long)st[sp - 1][r]; st[sp - 1][r] = f64_bits(in.a ? (double)__ll2float_rn(v) : __ll2double_rn(v)); } break;
      case VM_CAST_F_I: {
        FORR {
          const double d = as_f64(st[sp - 1][r]);
          // Rust `as i64`: truncates, saturates, NaN -> 0 (arrow/cast.rs:442-470 test_float_to_int).  cvt.rzi.s64.f64 saturates
          // too but maps NaN to 0x8000000000000000, so NaN is handled here (found by the reference KAT on hardware).
          long long v = d != d ? 0LL : __double2ll_rz(d);
          if (in.a < 64) { const long long mx = (1LL << (in.a - 1)) - 1, mn = -(1LL << (in.a - 1)); v = v > mx ? mx : (v < mn ? mn : v); }
          st[sp - 1][r] = (uint64_t)v;
        }
        break;
      }
      case VM_CAST_F_F32: FORR { st[sp - 1][r] = f64_bits((double)__double2float_rn(as_f64(st[sp - 1][r]))); } break;
      case VM_CAST_I_BOOL: FORR { st[sp - 1][r] = st[sp - 1][r] != 0; } break;
      case VM_CAST_F_BOOL: FORR { st[sp - 1][r] = as_f64(st[sp - 1][r]) != 0.0; } break;
      case VM_CAST_I_DEC: {
        const i128_t mul = mk128(pool[in.c], pool[in.c + 1]), lim = mk128(pool[in.c + 2], pool[in.c + 3]);
        FORR {
          i128_t v; bool ok = VALID(r, sp - 1);
          const bool of = mul_of((i128_t)(int64_t)st[sp - 1][r], mul, &v);
          ok = ok && !of && v > -lim && v < lim;
          if (!ok) v = 0;
          st[sp - 1][r] = lo64(v); st[sp][r] = hi64(v); SETV(r, sp - 1, ok);
        }
        sp += 1;
        break;
      }
      case VM_CAST_DEC_DEC: {
        const i128_t f = mk128(pool[in.c], pool[in.c + 1]), lim = mk128(pool[in.c + 2], pool[in.c + 3]);
        FORR {
          i128_t v = mk128(st[sp - 2][r], st[sp - 1][r]); bool ok = VALID(r, sp - 2);
          if (ok) {
            if (in.a == 1) {          // scale down: round half away from zero (arrow-cast)
              const bool neg = v < 0; u128_t m = neg ? (u128_t)0 - (u128_t)v : (u128_t)v;
              u128_t q = m / (u128_t)f, rem = m % (u128_t)f;
              if (rem * 2 >= (u128_t)f) q += 1;
              v = neg ? -(i128_t)q : (i128_t)q;
            } else if (in.a == 2) { i128_t t; if (mul_of(v, f, &t)) ok = false; v = t; }
            ok = ok && v > -lim && v < lim;
          }
          if (!ok) v = 0;
          st[sp - 2][r] = lo64(v); st[sp - 1][r] = hi64(v); SETV(r, sp - 2, ok);
        }
        break;
      }
      case VM_CAST_DEC_I: {
        const i128_t f = mk128(pool[in.c], pool[in.c + 1]);
        sp -= 1;
        FORR {
          const i128_t q = mk128(st[sp - 1][r], st[sp][r]) / f;       // truncates toward zero
          bool ok = VALID(r, sp - 1);
          const i128_t mx = ((i128_t)1 << (in.a - 1)) - 1, mn = -((i128_t)1 << (in.a - 1));
          ok = ok && q >= mn && q <= mx;
          st[sp - 1][r] = ok ? (uint64_t)(int64_t)q : 0; SETV(r, sp - 1, ok);
        }
        break;
      }
      case VM_CAST_DEC_F: {
        const double div = as_f64(pool[in.c]);
        sp -= 1;
        FORR {
          double d = i128_to_double(mk128(st[sp - 1][r], st[sp][r])) / div;
          if (in.a) d = (double)__double2float_rn(d);
          st[sp - 1][r] = f64_bits(d);
        }
        break;
      }
      case VM_CAST_F_DEC: {
        const double mul = as_f64(pool[in.c]); const i128_t lim = mk128(pool[in.c + 1], pool[in.c + 2]);
        FORR {
          bool ok = VALID(r, sp - 1);
          const double f = as_f64(st[sp - 1][r]) * mul;
          i128_t v = 0;
          if (ok && isfinite(f)) { bool fits; v = double_to_i128(round(f), &fits); ok = fits && v > -lim && v < lim; } else ok = false;
          if (!ok) v = 0;
          st[sp - 1][r] = lo64(v); st[sp][r] = hi64(v); SETV(r, sp - 1, ok);
        }
        sp += 1;
        break;
      }
      case VM_UNSCALED: sp -= 1; break;                                        // low 64 bits stay in place
      case VM_MAKE_DEC: FORR { st[sp][r] = (uint64_t)((int64_t)st[sp - 1][r] >> 63); } sp += 1; break;
      case VM_CHECK_OVERFLOW: {
        // change_precision_round_half_up (spark_check_overflow.rs:84-124)
        if (in.b == 1) break;
        const i128_t f = mk128(pool[in.c], pool[in.c + 1]), lim = mk128(pool[in.c + 2], pool[in.c + 3]);
        FORR {
          i128_t v = mk128(st[sp - 2][r], st[sp - 1][r]); bool ok = VALID(r, sp - 2);
          if (ok) {
            if (in.a == 1) {
              const i128_t dropped = v % f; v = v / f;
              const i128_t ad = dropped < 0 ? -dropped : dropped;
              // release build: `dropped.abs() * 2` wraps, so |dropped| >= 2^126 (a 38-digit scale drop) does not round
              if ((i128_t)((u128_t)ad * 2) >= f) v += dropped < 0 ? -1 : 1;
            } else if (in.a == 2) v = (i128_t)((u128_t)v * (u128_t)f);       // release build: wrapping multiply
            ok = !(v <= -lim || v >= lim);
          }
          if (!ok) v = 0;
          st[sp - 2][r] = lo64(v); st[sp - 1][r] = hi64(v); SETV(r, sp - 2, ok);
        }
        break;
      }
      case VM_NULL_IF_ZERO_I: FORR { if (st[sp - 1][r] == 0) SETV(r, sp - 1, false); } break;
      case VM_NULL_IF_ZERO_F: FORR { if (as_f64(st[sp - 1][r]) == 0.0) SETV(r, sp - 1, false); } break;
      case VM_NULL_IF_ZERO_DEC: FORR { if ((st[sp - 2][r] | st[sp - 1][r]) == 0) SETV(r, sp - 2, false); } break;
      case VM_NULLIFY: {
        sp -= 1;
        FORR { if (VALID(r, sp) && st[sp][r] != 0) SETV(r, sp - in.a, false); }
        break;
      }
      case VM_NORM_NAN_ZERO: {
        FORR {
          double d = as_f64(st[sp - 1][r]);
          if (d != d) d = in.a ? (double)__int_as_float(0x7fc00000) : __longlong_as_double(0x7ff8000000000000LL);
          else if (d == 0.0) d = 0.0;
          st[sp - 1][r] = f64_bits(d);
        }
        break;
      }
      case VM_SELECT: {
        // stack: cond, then[n], else[n]  ->  result[n]
        const int n = in.a, ic = sp - 2 * n - 1, it = ic + 1, ie = it + n;
        FORR {
          const bool c = VALID(r, ic) && st[ic][r] != 0;
          const bool ok = c ? VALID(r, it) : VALID(r, ie);
          st[ic][r] = c ? st[it][r] : st[ie][r];
          if (n == 2) st[ic + 1][r] = c ? st[it + 1][r] : st[ie + 1][r];
          SETV(r, ic, ok);
        }
        sp = ic + n;
        break;
      }
      case VM_IN_LIST: {
        if ((in.a & 3) == 3) { sp = vm_str<R>(in, pool, st, vm, sp); break; }
        const int kind = in.a & 3; const bool neg = in.a & 4, has_null = in.a & 8;
        const int n = kind >= 2 ? 2 : 1, ix = sp - n;
        FORR {
          bool found = false;
          if (kind == 2) { for (int k = 0; k < in.b; k++) found |= pool[in.c + 2 * k] == st[ix][r] && pool[in.c + 2 * k + 1] == st[ix + 1][r]; }
          else if (kind == 1) { const int64_t x = total_order_key(st[ix][r]); for (int k = 0; k < in.b; k++) found |= total_order_key(pool[in.c + k]) == x; }
          else { for (int k = 0; k < in.b; k++) found |= pool[in.c + k] == st[ix][r]; }
          const bool ok = VALID(r, ix) && (found || !has_null);
          st[ix][r] = found != neg; SETV(r, ix, ok);
        }
        sp = ix + 1;
        break;
      }
      case VM_FILTER: {
        sp -= 1;
        FORR { alive[r] = alive[r] && VALID(r, sp) && st[sp][r] != 0; }
        break;
      }
      case VM_OUT: {
        const int n = in.a >= PH_DEC128 ? 2 : 1;
        sp -= n;
        FORR { sink.out(r, (int)in.b, (int)in.a, st[sp][r], n == 2 ? st[sp + 1][r] : 0ULL, (bool)VALID(r, sp)); }
        break;
      }
      case VM_OUT_SEL: FORR { sink.out(r, (int)in.b, (int)PH_SEL, (uint64_t)row[r], 0ULL, true); } break;
      case VM_CMP_STR: case VM_STARTS_WITH: case VM_ENDS_WITH: case VM_CONTAINS: case VM_CAST_STR_I: sp = vm_str<R>(in, pool, st, vm, sp); break;
      case VM_XXHASH64: case VM_BLOOM_PROBE: sp = vm_bloom<R>(in, pool, st, vm, sp); break;
      default: return -1;
    }
  }
#undef STRP
#undef VALID
#undef SETV
#undef FORR
}

}  // namespace b200q
