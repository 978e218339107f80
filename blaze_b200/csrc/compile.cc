// Expression IR -> VM bytecode (see vm.h).  Also the plan-level helpers used when fusing a
// Project(Filter(...)) chain into one program: ProjectExec fuses its child FilterExec
// (project_exec.rs:143-149); on the GPU the whole Filter/Project chain below an Agg fuses the same
// way, so filtered rows never round-trip through HBM.
#include <cmath>
#include <cstddef>
#include <cstring>

#include "../../include/blaze_b200.h"
#include "compile.h"

namespace b200q {

typedef __int128 i128;

static i128 pow10_i128(int n) { i128 v = 1; for (int i = 0; i < n; i++) v *= 10; return v; }
// 10^n as the correctly rounded f64 (i128 -> double rounds once).  libm's pow need not be: glibc 2.39 returns 10^23 one ulp
// high, so the decimal <-> float casts of scale 23 would depend on the host's libm.
static double pow10_f64(int n) { return (double)pow10_i128(n); }

PhysKind phys_of(const DType& t) {
  switch (t.id) {
    case T_BOOL: return PH_BOOL; case T_INT8: return PH_I8; case T_INT16: return PH_I16;
    case T_INT32: case T_DATE32: return PH_I32; case T_INT64: case T_TIMESTAMP_US: return PH_I64;
    case T_FLOAT32: return PH_F32; case T_FLOAT64: return PH_F64; case T_DECIMAL128: return PH_DEC128; case T_UTF8: return PH_STR;
    default: throw PlanError(B200Q_ERR_UNSUPPORTED, "column type " + t.str() + " cannot be evaluated on the device");
  }
}

ExprP substitute(const ExprP& e, const std::vector<ExprP>& cols) {
  if (e->kind == E_COLUMN) {
    if (e->col_index < 0 || (size_t)e->col_index >= cols.size()) throw PlanError(B200Q_ERR_INVALID_PLAN, "column index out of range");
    return cols[e->col_index];
  }
  if (e->children.empty()) return e;
  auto c = std::make_shared<Expr>(*e);
  for (auto& ch : c->children) ch = substitute(ch, cols);
  return c;
}

namespace {

struct Compiler {
  CompiledProgram out;
  int depth = 0;

  VmProgram& p() { return out.prog; }
  void push(int n) { depth += n; if (depth > (int)p().max_depth) p().max_depth = depth; if (depth > VM_MAX_DEPTH) throw PlanError(B200Q_ERR_UNSUPPORTED, "expression too deep for the device evaluator"); }
  void pop(int n) { depth -= n; }
  void emit(VmOp op, uint8_t a = 0, uint16_t b = 0, uint32_t c = 0) {
    if (p().n_code >= VM_MAX_CODE - 1) throw PlanError(B200Q_ERR_UNSUPPORTED, "expression program too long for the device evaluator");
    p().code[p().n_code++] = VmInstr{(uint8_t)op, a, b, c};
  }
  uint32_t pool(std::initializer_list<uint64_t> vals) {
    if (p().n_pool + vals.size() > VM_MAX_POOL) throw PlanError(B200Q_ERR_UNSUPPORTED, "too many constants for the device evaluator");
    uint32_t at = p().n_pool;
    for (auto v : vals) p().pool[p().n_pool++] = v;
    return at;
  }
  static uint64_t lo(i128 v) { return (uint64_t)v; }
  static uint64_t hi(i128 v) { return (uint64_t)(v >> 64); }
  static uint64_t dbits(double d) { uint64_t b; memcpy(&b, &d, 8); return b; }

  int col_slot(int col_index) {
    for (size_t i = 0; i < out.used_cols.size(); i++) if (out.used_cols[i] == col_index) return (int)i;
    if (out.used_cols.size() >= VM_MAX_COLS) throw PlanError(B200Q_ERR_UNSUPPORTED, "too many input columns referenced by one fused pipeline");
    out.used_cols.push_back(col_index);
    return (int)out.used_cols.size() - 1;
  }

  static int slots(const DType& t) { return t.is_decimal() || t.id == T_UTF8 ? 2 : 1; }

  // a Utf8 constant: its bytes go to the program's string pool, the pool gets {offset, length} (relocated to a device address at upload)
  uint32_t str_const(const std::string& v) {
    if (p().n_str + v.size() > (size_t)VM_MAX_STR_POOL)
      throw PlanError(B200Q_ERR_UNSUPPORTED, "string literals of one fused pipeline exceed the " + std::to_string(VM_MAX_STR_POOL) + "-byte literal pool of the device evaluator");
    const uint32_t off = p().n_str;
    if (!v.empty()) memcpy(p().str_pool + off, v.data(), v.size());
    p().n_str += (uint32_t)v.size();
    out.has_strings = true;
    const uint32_t at = pool({off, (uint64_t)v.size()});
    out.str_relocs.push_back(at);
    return at;
  }

  void push_null(int nslots) { emit(VM_LOAD_LIT, (uint8_t)(1 | (nslots == 2 ? 2 : 0)), 0, pool({0, 0})); push(nslots); }

  // compile `e`; when e is an untyped NULL and `want` is given, produce a NULL of `want`'s width
  int expr(const ExprP& e, const DType* want = nullptr) {
    if (e->type.id == T_NULL && e->kind == E_LITERAL) { int n = want ? slots(*want) : 1; push_null(n); return n; }
    switch (e->kind) {
      case E_COLUMN: {
        PhysKind ph = phys_of(e->type);
        if (ph == PH_STR) { out.has_strings = true; emit(VM_LOAD_STR, 0, (uint16_t)col_slot(e->col_index)); push(2); return 2; }
        emit(VM_LOAD_COL, ph, (uint16_t)col_slot(e->col_index)); push(slots(e->type)); return slots(e->type);
      }
      case E_LITERAL: {
        int n = slots(e->type);
        if (e->type.id == T_UTF8) { emit(VM_LOAD_LIT, (uint8_t)((e->lit_null ? 1 : 0) | 2), 0, str_const(e->lit_str)); push(2); return 2; }
        emit(VM_LOAD_LIT, (uint8_t)((e->lit_null ? 1 : 0) | (n == 2 ? 2 : 0)), 0, pool({e->lit_lo, e->lit_hi})); push(n); return n;
      }
      case E_BINARY: case E_SC_AND: case E_SC_OR: return binary(e);
      case E_IS_NULL: case E_IS_NOT_NULL: {
        int n = expr(e->children[0]);
        emit(e->kind == E_IS_NULL ? VM_IS_NULL : VM_IS_NOT_NULL, (uint8_t)n); pop(n); push(1); return 1;
      }
      case E_NOT: expr(e->children[0]); emit(VM_NOT); return 1;
      case E_NEGATIVE: {
        const DType& t = e->type; int n = expr(e->children[0]);
        if (t.is_decimal()) emit(VM_NEG_DEC); else if (t.is_float()) emit(VM_NEG_F, t.id == T_FLOAT32); else emit(VM_NEG_I, (uint8_t)t.int_bits());
        return n;
      }
      case E_CAST: case E_TRY_CAST: return cast(e);
      case E_CASE: return case_(e);
      case E_IN_LIST: return in_list(e);
      case E_SCALAR_FN: return scalar_fn(e);
      case E_BLOOM: return bloom(e);
      case E_STR_MATCH: {
        expr(e->children[0]);
        emit(VM_LOAD_LIT, 2, 0, str_const(e->lit_str)); push(2);
        static const VmOp ops[] = {VM_STARTS_WITH, VM_ENDS_WITH, VM_CONTAINS};
        emit(ops[e->str_match]); pop(4); push(1); return 1;
      }
    }
    throw PlanError(B200Q_ERR_UNSUPPORTED, "unsupported expression kind");
  }

  int binary(const ExprP& e) {
    const ExprP &l = e->children[0], &r = e->children[1];
    BinOp op = e->op;
    if (op == OP_AND || op == OP_OR) { expr(l); expr(r); emit(op == OP_AND ? VM_AND : VM_OR); pop(2); push(1); return 1; }
    const DType& t = l->type;
    if (op >= OP_EQ && op <= OP_GE) {
      int n = expr(l); expr(r);
      uint8_t c = (uint8_t)(op - OP_EQ);   // OP_EQ..OP_GE map to CMP_EQ,NE,LT,LE,GT,GE in the same order
      if (t.id == T_UTF8) emit(VM_CMP_STR, c); else if (t.is_decimal()) emit(VM_CMP_DEC, c); else if (t.is_float()) emit(VM_CMP_F, c); else emit(VM_CMP_I, c);
      pop(2 * n); push(1); return 1;
    }
    if (op >= OP_BIT_AND) { expr(l); expr(r); emit(op == OP_BIT_AND ? VM_BIT_AND : op == OP_BIT_OR ? VM_BIT_OR : VM_BIT_XOR); pop(2); push(1); return 1; }
    if (t.is_decimal()) {
      expr(l); expr(r);
      i128 lm = pow10_i128(e->type.scale - l->type.scale), rm = pow10_i128(e->type.scale - r->type.scale);
      emit(op == OP_PLUS ? VM_ADD_DEC : VM_SUB_DEC, 0, 0, pool({lo(lm), hi(lm), lo(rm), hi(rm)})); pop(4); push(2); return 2;
    }
    expr(l); expr(r);
    if (t.is_float()) {
      static const VmOp f[] = {VM_ADD_F, VM_SUB_F, VM_MUL_F, VM_DIV_F, VM_MOD_F};
      emit(f[op - OP_PLUS], t.id == T_FLOAT32);
    } else {
      static const VmOp f[] = {VM_ADD_I, VM_SUB_I, VM_MUL_I, VM_DIV_I, VM_MOD_I};
      emit(f[op - OP_PLUS], (uint8_t)t.int_bits());
    }
    pop(2); push(1); return 1;
  }

  int cast(const ExprP& e) {
    const DType from = e->children[0]->type, to = e->type;
    if (from.id == T_NULL) { push_null(slots(to)); return slots(to); }       // cast of an untyped NULL
    int n = expr(e->children[0]);
    if (from == to) return n;                                                 // commons cast.rs:41
    if (from.id == T_UTF8 && to.is_integer() && e->kind == E_TRY_CAST) { emit(VM_CAST_STR_I, (uint8_t)to.int_bits()); pop(2); push(1); return 1; }
    auto ii = [](const DType& t) { return t.is_integer() || t.id == T_DATE32 || t.id == T_TIMESTAMP_US; };
    i128 lim = to.is_decimal() ? pow10_i128(to.precision) : 0;
    if (ii(from) && ii(to)) { if (to.int_bits() < from.int_bits()) emit(VM_CAST_I_I, (uint8_t)to.int_bits()); return 1; }
    if (from.id == T_BOOL && to.is_integer()) return 1;
    if (from.id == T_BOOL && to.is_float()) { emit(VM_CAST_I_F, to.id == T_FLOAT32); return 1; }
    if (ii(from) && to.is_float()) { emit(VM_CAST_I_F, to.id == T_FLOAT32); return 1; }
    if (from.is_float() && to.is_integer()) { emit(VM_CAST_F_I, (uint8_t)to.int_bits()); return 1; }
    if (from.is_float() && to.is_float()) { if (to.id == T_FLOAT32) emit(VM_CAST_F_F32); return 1; }
    if (from.is_integer() && to.id == T_BOOL) { emit(VM_CAST_I_BOOL); return 1; }
    if (from.is_float() && to.id == T_BOOL) { emit(VM_CAST_F_BOOL); return 1; }
    if (from.is_integer() && to.is_decimal()) {
      i128 m = pow10_i128(to.scale);
      emit(VM_CAST_I_DEC, 0, 0, pool({lo(m), hi(m), lo(lim), hi(lim)})); pop(1); push(2); return 2;
    }
    if (from.is_decimal() && to.is_decimal()) {
      int d = to.scale - from.scale; i128 f = pow10_i128(d < 0 ? -d : d);
      emit(VM_CAST_DEC_DEC, (uint8_t)(d == 0 ? 0 : d < 0 ? 1 : 2), 0, pool({lo(f), hi(f), lo(lim), hi(lim)})); return 2;
    }
    if (from.is_decimal() && to.is_integer()) {
      i128 f = pow10_i128(from.scale);
      emit(VM_CAST_DEC_I, (uint8_t)to.int_bits(), 0, pool({lo(f), hi(f)})); pop(2); push(1); return 1;
    }
    if (from.is_decimal() && to.is_float()) {
      emit(VM_CAST_DEC_F, to.id == T_FLOAT32, 0, pool({dbits(pow10_f64(from.scale))})); pop(2); push(1); return 1;
    }
    if (from.is_float() && to.is_decimal()) {
      emit(VM_CAST_F_DEC, 0, 0, pool({dbits(pow10_f64(to.scale)), lo(lim), hi(lim)})); pop(1); push(2); return 2;
    }
    throw PlanError(B200Q_ERR_UNSUPPORTED, "cast " + from.str() + " -> " + to.str() + " is not on the hot path");
  }

  int case_(const ExprP& e) {
    // children = [base?] w1 t1 ... [else]; evaluated branch-free:
    //   result = SELECT(c1, t1, SELECT(c2, t2, ... else))   -- build from the last WHEN backwards
    size_t i0 = e->case_has_base ? 1 : 0;
    size_t nwt = (e->children.size() - i0 - (e->case_has_else ? 1 : 0)) / 2;
    if (e->type.id == T_UTF8 || (e->case_has_base && e->children[0]->type.id == T_UTF8)) throw PlanError(B200Q_ERR_UNSUPPORTED, "CASE over strings is not on the hot path");
    int n = slots(e->type);
    // emit conditions and THENs in order, then ELSE, then fold with SELECTs (stack: c1 t1 c2 t2 ... else)
    for (size_t k = 0; k < nwt; k++) {
      const ExprP &w = e->children[i0 + 2 * k], &t = e->children[i0 + 2 * k + 1];
      if (e->case_has_base) {
        const ExprP& base = e->children[0];
        int bn = expr(base); expr(w, &base->type);
        if (base->type.is_decimal()) emit(VM_CMP_DEC, CMP_EQ); else if (base->type.is_float()) emit(VM_CMP_F, CMP_EQ); else emit(VM_CMP_I, CMP_EQ);
        pop(2 * bn); push(1);
      } else expr(w);
      expr(t, &e->type);
    }
    if (e->case_has_else) expr(e->children.back(), &e->type); else push_null(n);
    for (size_t k = 0; k < nwt; k++) { emit(VM_SELECT, (uint8_t)n); pop(1 + 2 * n); push(n); }
    return n;
  }

  int in_list(const ExprP& e) {
    const ExprP& x = e->children[0];
    if (x->type.id == T_UTF8) return in_list_str(e);
    int kind = x->type.is_decimal() ? 2 : x->type.is_float() ? 1 : 0;
    bool has_null = false; std::vector<uint64_t> items;
    for (size_t i = 1; i < e->children.size(); i++) {
      ExprP it = e->children[i];
      // literal items only (Spark In/InSet lists are literals); a TryCast-wrapped literal is folded here
      DType want = x->type;
      uint64_t vlo = 0, vhi = 0; bool null = false;
      if (!fold_literal(it, want, vlo, vhi, null)) throw PlanError(B200Q_ERR_UNSUPPORTED, "IN list items must be literals on the hot path");
      if (null) { has_null = true; continue; }
      items.push_back(vlo); if (kind == 2) items.push_back(vhi);
    }
    int n = expr(x);
    if (p().n_pool + items.size() > VM_MAX_POOL) throw PlanError(B200Q_ERR_UNSUPPORTED, "IN list too long for the device evaluator");
    uint32_t at = p().n_pool;
    for (auto v : items) p().pool[p().n_pool++] = v;
    uint16_t cnt = (uint16_t)(kind == 2 ? items.size() / 2 : items.size());
    emit(VM_IN_LIST, (uint8_t)(kind | (e->negated ? 4 : 0) | (has_null ? 8 : 0)), cnt, at); pop(n); push(1); return 1;
  }

  int in_list_str(const ExprP& e) {
    bool has_null = false; std::vector<const std::string*> items;
    for (size_t i = 1; i < e->children.size(); i++) {
      ExprP it = e->children[i];
      if ((it->kind == E_TRY_CAST || it->kind == E_CAST) && it->children[0]->kind == E_LITERAL && it->children[0]->type.id == T_NULL) it = it->children[0];   // TryCast(NULL)
      if (it->kind != E_LITERAL || !(it->type.id == T_UTF8 || it->type.id == T_NULL)) throw PlanError(B200Q_ERR_UNSUPPORTED, "IN list items must be literals on the hot path");
      if (it->lit_null || it->type.id == T_NULL) has_null = true; else items.push_back(&it->lit_str);
    }
    int n = expr(e->children[0]);
    uint32_t at = p().n_pool;
    for (auto* s : items) str_const(*s);                     // consecutive {ptr, len} pairs
    emit(VM_IN_LIST, (uint8_t)(3 | (e->negated ? 4 : 0) | (has_null ? 8 : 0)), (uint16_t)items.size(), at); pop(n); push(1); return 1;
  }

  // constant-fold Literal / TryCast(Literal) to `want` (only the conversions IN lists need)
  static bool fold_literal(const ExprP& e, const DType& want, uint64_t& vlo, uint64_t& vhi, bool& null) {
    if (e->kind == E_LITERAL) {
      null = e->lit_null || e->type.id == T_NULL; vlo = e->lit_lo; vhi = e->lit_hi;
      return e->type == want || null;
    }
    if ((e->kind == E_TRY_CAST || e->kind == E_CAST) && e->children[0]->kind == E_LITERAL) {
      const ExprP& l = e->children[0];
      null = l->lit_null || l->type.id == T_NULL; if (null) return true;
      if (l->type.is_integer() && want.is_integer()) {
        int64_t v = (int64_t)l->lit_lo; int b = want.int_bits();
        if (b < 64 && (v < -(1LL << (b - 1)) || v > (1LL << (b - 1)) - 1)) { null = true; return true; }
        vlo = (uint64_t)v; vhi = 0; return true;
      }
      if (l->type.is_integer() && want.id == T_FLOAT64) { double d = (double)(int64_t)l->lit_lo; memcpy(&vlo, &d, 8); return true; }
      if (l->type.is_integer() && want.is_decimal()) {
        i128 v = (i128)(int64_t)l->lit_lo * pow10_i128(want.scale); i128 lim = pow10_i128(want.precision);
        if (v <= -lim || v >= lim) { null = true; return true; }
        vlo = lo(v); vhi = hi(v); return true;
      }
    }
    return false;
  }

  // BloomFilterMightContain: a NULL filter is `false` for every row without evaluating the value (bloom_filter_might_contain.rs)
  int bloom(const ExprP& e) {
    if (!e->bloom) throw PlanError(B200Q_ERR_INVALID_PLAN, "BloomFilterMightContain: the scalar subquery was not resolved");
    out.vm_only = true;
    if (e->bloom->is_null) { emit(VM_LOAD_LIT, 0, 0, pool({0, 0})); push(1); return 1; }
    if (out.blooms.size() >= (size_t)VM_MAX_BLOOMS)
      throw PlanError(B200Q_ERR_UNSUPPORTED, "more than " + std::to_string(VM_MAX_BLOOMS) + " BloomFilterMightContain expressions in one fused pipeline");
    expr(e->children[0]);                                        // Int8..Int64: already an i64 on the stack
    const uint32_t at = pool({0, 64 * (uint64_t)e->bloom->words.size(), (uint64_t)e->bloom->num_hash_functions});
    out.blooms.push_back(CompiledProgram::BloomRef{at, e->bloom});
    emit(VM_BLOOM_PROBE, 0, 0, at);
    return 1;
  }

  int scalar_fn(const ExprP& e) {
    const std::string& nm = e->name;
    if (nm == "Placeholder") throw PlanError(B200Q_ERR_INVALID_PLAN, "placeholder() should never be called");
    if (nm == "UnscaledValue") { expr(e->children[0]); emit(VM_UNSCALED); pop(2); push(1); return 1; }
    if (nm == "MakeDecimal") { expr(e->children[0]); emit(VM_MAKE_DEC); pop(1); push(2); return 2; }
    if (nm == "CheckOverflow") {
      const DType from = e->children[0]->type, to = e->type;
      expr(e->children[0]);
      int d = to.scale - from.scale; i128 f = pow10_i128(d < 0 ? -d : d);
      i128 lim = pow10_i128(std::min<int>(to.precision, 38));
      bool identity = to.precision == from.precision && to.scale == from.scale;     // spark_check_overflow.rs:93-95
      emit(VM_CHECK_OVERFLOW, (uint8_t)(d == 0 ? 0 : d < 0 ? 1 : 2), identity ? 1 : 0, pool({lo(f), hi(f), lo(lim), hi(lim)})); return 2;
    }
    if (nm == "NullIfZero") {
      const DType& t = e->children[0]->type; int n = expr(e->children[0]);
      emit(t.is_decimal() ? VM_NULL_IF_ZERO_DEC : t.is_float() ? VM_NULL_IF_ZERO_F : VM_NULL_IF_ZERO_I); return n;
    }
    if (nm == "NullIf") {
      const DType& t = e->children[0]->type;
      int n = expr(e->children[0]); expr(e->children[0]); expr(e->children[1], &t);
      emit(t.is_decimal() ? VM_CMP_DEC : t.is_float() ? VM_CMP_F : VM_CMP_I, CMP_EQ); pop(2 * n); push(1);
      emit(VM_NULLIFY, (uint8_t)n); pop(1); return n;
    }
    if (nm == "NormalizeNanAndZero") { expr(e->children[0]); emit(VM_NORM_NAN_ZERO, e->type.id == T_FLOAT32); return 1; }
    if (nm == "XxHash64") {                 // h = 42; per argument h = xxhash64(value, h), a NULL argument leaves h
      out.vm_only = true;
      emit(VM_LOAD_LIT, 0, 0, pool({42, 0})); push(1);
      for (auto& a : e->children) {
        if (a->type.id == T_NULL) continue;                      // an untyped NULL hashes nothing
        const int n = expr(a);
        emit(VM_XXHASH64, (uint8_t)phys_of(a->type)); pop(n);
      }
      return 1;
    }
    throw PlanError(B200Q_ERR_UNSUPPORTED, "spark ext function '" + nm + "' is not on the hot path");
  }
};

}  // namespace

CompiledProgram compile_program(const std::vector<ExprP>& filters, const std::vector<ExprP>& outs, bool with_compact, int sel_out) {
  Compiler c;
  memset(&c.out.prog, 0, sizeof(VmProgram));
  for (auto& f : filters) {
    if (f->type.id != T_BOOL) throw PlanError(B200Q_ERR_INVALID_PLAN, "Filter predicate must return boolean values");
    c.expr(f); c.emit(VM_FILTER); c.pop(1);
  }
  c.out.prog.n_filters = (uint32_t)filters.size();
  if (with_compact) c.emit(VM_COMPACT);
  if (outs.size() + (sel_out >= 0 ? 1 : 0) > VM_MAX_OUT) throw PlanError(B200Q_ERR_UNSUPPORTED, "too many outputs for one fused pipeline");
  for (size_t i = 0; i < outs.size(); i++) {
    const ExprP& e = outs[i];
    int n = c.expr(e);
    c.emit(VM_OUT, (uint8_t)phys_of(e->type), (uint16_t)i); c.pop(n);
    c.out.outs.push_back(OutDesc{e->type, e->nullable, n});
  }
  if (sel_out >= 0) c.emit(VM_OUT_SEL, 0, (uint16_t)sel_out);
  c.emit(VM_END);
  return c.out;
}

VmProgram relocated_program(const CompiledProgram& cp, const void* device_copy) {
  VmProgram p = cp.prog;
  const uint64_t base = (uint64_t)(uintptr_t)device_copy + offsetof(VmProgram, str_pool);
  for (uint32_t i : cp.str_relocs) p.pool[i] += base;
  return p;
}

}  // namespace b200q
