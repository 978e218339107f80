// Plan decoding: protobuf bytes of the reference's `auron.proto` -> hot-path IR.
//
// Restates, for the {Filter, Projection, Agg, FFIReader, EmptyPartitions} subset, what
// `TryInto<Arc<dyn ExecutionPlan>> for &PhysicalPlanNode` and `try_parse_physical_expr` do
// (native-engine/auron-serde/src/from_proto.rs:107-152, 407-500, 839-1026), including the
// constructor-time rewrites of `create_agg` (datafusion-ext-plans/src/agg/agg.rs:171-205) and the
// validation of FilterExec::try_new (filter_exec.rs:58-66) / AggContext::try_new (agg_ctx.rs:110-141).
// No protoc in this image: the proto3 wire format is read by hand (field numbers cited inline).
#include <cstring>
#include <sstream>

#include "../../include/blaze_b200.h"
#include "ir.h"

namespace b200q {

std::string DType::str() const {
  switch (id) {
    case T_BOOL: return "bool"; case T_INT8: return "int8"; case T_INT16: return "int16"; case T_INT32: return "int32";
    case T_INT64: return "int64"; case T_FLOAT32: return "float32"; case T_FLOAT64: return "float64";
    case T_DATE32: return "date32"; case T_TIMESTAMP_US: return "timestamp[us]";
    case T_DECIMAL128: return "decimal128(" + std::to_string(precision) + "," + std::to_string(scale) + ")";
    case T_BINARY: return "binary"; case T_UTF8: return "utf8"; default: return "null";
  }
}

namespace {

[[noreturn]] void bad(const std::string& m) { throw PlanError(B200Q_ERR_INVALID_PLAN, m); }
[[noreturn]] void unsupported(const std::string& m) { throw PlanError(B200Q_ERR_UNSUPPORTED, m); }

// ---- proto3 wire reader ---------------------------------------------------------------------------
struct Reader {
  const uint8_t* p; const uint8_t* end;
  Reader(const uint8_t* b, size_t n) : p(b), end(b + n) {}
  bool done() const { return p >= end; }
  uint64_t varint() {
    uint64_t v = 0; int shift = 0;
    while (true) {
      if (p >= end) bad("protobuf: truncated varint");
      uint8_t b = *p++;
      v |= (uint64_t)(b & 0x7F) << shift;
      if (!(b & 0x80)) return v;
      shift += 7;
      if (shift > 63) bad("protobuf: varint too long");
    }
  }
  // reads a tag; returns field number, sets wire type
  uint32_t tag(int& wt) { uint64_t t = varint(); wt = (int)(t & 7); return (uint32_t)(t >> 3); }
  Reader bytes() {
    uint64_t n = varint();
    if ((uint64_t)(end - p) < n) bad("protobuf: truncated length-delimited field");
    Reader r(p, (size_t)n); p += n; return r;
  }
  std::string str() { Reader r = bytes(); return std::string((const char*)r.p, (size_t)(r.end - r.p)); }
  void skip(int wt) {
    switch (wt) {
      case 0: varint(); break;
      case 1: if (end - p < 8) bad("protobuf: truncated fixed64"); p += 8; break;
      case 2: bytes(); break;
      case 5: if (end - p < 4) bad("protobuf: truncated fixed32"); p += 4; break;
      default: bad("protobuf: unsupported wire type " + std::to_string(wt));
    }
  }
  // repeated enum/varint: accepts packed (wt 2) and unpacked (wt 0)
  void varints(int wt, std::vector<uint64_t>& out) {
    if (wt == 0) { out.push_back(varint()); return; }
    if (wt != 2) bad("protobuf: bad wire type for repeated varint");
    Reader r = bytes();
    while (!r.done()) out.push_back(r.varint());
  }
};

// ---- ArrowType (auron.proto:860-896) ----------------------------------------------------------------
DType parse_arrow_type(Reader r) {
  DType d; bool set = false;
  while (!r.done()) {
    int wt; uint32_t f = r.tag(wt);
    auto empty = [&](TypeId id) { r.skip(wt); d = DType(); d.id = id; set = true; };
    switch (f) {
      case 1: empty(T_NULL); break;        // NONE
      case 2: empty(T_BOOL); break;
      case 4: empty(T_INT8); break;
      case 6: empty(T_INT16); break;
      case 8: empty(T_INT32); break;
      case 10: empty(T_INT64); break;
      case 12: empty(T_FLOAT32); break;
      case 13: empty(T_FLOAT64); break;
      case 15: empty(T_BINARY); break;
      case 17: empty(T_DATE32); break;
      case 20: {                           // Timestamp{time_unit=1, timezone=2} (auron.proto:755-758)
        Reader t = r.bytes(); uint64_t unit = 0;
        while (!t.done()) { int w; uint32_t g = t.tag(w); if (g == 1) unit = t.varint(); else t.skip(w); }
        if (unit != 2) unsupported("only Timestamp(Microsecond) is on the hot path");
        d = DType(); d.id = T_TIMESTAMP_US; set = true; break;
      }
      case 24: {                           // Decimal{whole=1 (precision), fractional=2 (scale)} (auron.proto:786-789)
        Reader t = r.bytes(); uint64_t whole = 0; int64_t frac = 0;
        while (!t.done()) { int w; uint32_t g = t.tag(w); if (g == 1) whole = t.varint(); else if (g == 2) frac = (int64_t)t.varint(); else t.skip(w); }
        if (whole < 1 || whole > 38) bad("Decimal precision out of range");
        d = DType(); d.id = T_DECIMAL128; d.precision = (uint8_t)whole; d.scale = (int8_t)frac; set = true; break;
      }
      case 3: case 5: case 7: case 9: unsupported("unsigned integer columns are not on the hot path");
      case 14: empty(T_UTF8); break;
      case 32: unsupported("LargeUtf8 columns are not on the hot path");
      default: unsupported("ArrowType tag " + std::to_string(f) + " is not on the hot path");
    }
  }
  if (!set) bad("ArrowType: empty oneof");
  return d;
}

FieldDef parse_field(Reader c) {               // Field{name=1,arrow_type=2,nullable=3}
  FieldDef fd; fd.nullable = false; bool have_t = false;
  while (!c.done()) {
    int w; uint32_t g = c.tag(w);
    if (g == 1) fd.name = c.str();
    else if (g == 2) { fd.type = parse_arrow_type(c.bytes()); have_t = true; }
    else if (g == 3) fd.nullable = c.varint() != 0;
    else c.skip(w);
  }
  if (!have_t) bad("Field without arrow_type");
  return fd;
}

SchemaDef parse_schema(Reader r) {            // Schema{columns=1}
  SchemaDef s;
  while (!r.done()) {
    int wt; uint32_t f = r.tag(wt);
    if (f == 1) s.fields.push_back(parse_field(r.bytes()));
    else r.skip(wt);
  }
  return s;
}

// ---- expressions --------------------------------------------------------------------------------------
ExprP mk(ExprKind k) { auto e = std::make_shared<Expr>(); e->kind = k; return e; }
DType bool_t() { DType d; d.id = T_BOOL; return d; }
DType i64_t() { DType d; d.id = T_INT64; return d; }

BinOp parse_binop(const std::string& s) {      // auron-serde/src/lib.rs:70-102
  static const std::pair<const char*, BinOp> tbl[] = {
      {"And", OP_AND}, {"Or", OP_OR}, {"Eq", OP_EQ}, {"NotEq", OP_NE}, {"LtEq", OP_LE}, {"Lt", OP_LT}, {"Gt", OP_GT},
      {"GtEq", OP_GE}, {"Plus", OP_PLUS}, {"Minus", OP_MINUS}, {"Multiply", OP_MUL}, {"Divide", OP_DIV}, {"Modulo", OP_MOD},
      {"BitwiseAnd", OP_BIT_AND}, {"BitwiseOr", OP_BIT_OR}, {"BitwiseXor", OP_BIT_XOR}};
  for (auto& kv : tbl) if (s == kv.first) return kv.second;
  static const char* known[] = {"IsDistinctFrom", "IsNotDistinctFrom", "BitwiseShiftLeft", "BitwiseShiftRight", "RegexIMatch",
                                "RegexMatch", "RegexNotIMatch", "RegexNotMatch", "StringConcat"};
  for (auto k : known) if (s == k) unsupported("binary operator '" + s + "' is not on the hot path");
  bad("Unsupported binary operator '\"" + s + "\"'");
}

ExprP parse_expr(Reader r, const SchemaDef& schema);

ExprP parse_boxed(Reader r, uint32_t field, const SchemaDef& schema) {  // message{expr=field}
  ExprP e;
  while (!r.done()) { int wt; uint32_t f = r.tag(wt); if (f == field) e = parse_expr(r.bytes(), schema); else r.skip(wt); }
  if (!e) bad("Missing required field in protobuf");
  return e;
}

ExprP wrap_try_cast(ExprP e, DType to) {
  auto c = mk(E_TRY_CAST); c->children = {e}; c->type = to; c->nullable = true;   // TryCastExpr::nullable = true (cast.rs:65-67)
  return c;
}

void check_cast_supported(const DType& from, const DType& to, bool try_cast);

ExprP finish_binary(ExprP l, BinOp op, ExprP rr) {
  auto e = mk(E_BINARY); e->op = op; e->children = {l, rr};
  e->nullable = l->nullable || rr->nullable;
  const DType &lt = l->type, &rt = rr->type;
  if (op == OP_AND || op == OP_OR) {
    if (lt.id != T_BOOL || rt.id != T_BOOL) bad("And/Or over non-boolean operands");
    e->type = bool_t(); return e;
  }
  if (op >= OP_EQ && op <= OP_GE) {
    if (lt.id == T_NULL || rt.id == T_NULL) unsupported("comparison with an untyped NULL literal");
    if (lt.is_decimal() && rt.is_decimal()) { if (lt.scale != rt.scale) bad("comparison of decimals with different scale (arrow cmp requires equal types)"); }
    else if (lt != rt) bad("comparison of " + lt.str() + " with " + rt.str() + ": arrow cmp requires equal types");
    if (lt.id == T_BINARY) unsupported("binary comparison is not on the hot path");
    e->type = bool_t(); return e;
  }
  if (op >= OP_BIT_AND) {
    if (lt != rt || !lt.is_integer()) bad("bitwise operator over " + lt.str() + "," + rt.str());
    e->type = lt; return e;
  }
  // arithmetic
  if (lt.is_decimal() && rt.is_decimal()) {
    if (op != OP_PLUS && op != OP_MINUS) unsupported("decimal Multiply/Divide/Modulo is not on the hot path (round 1)");
    int s = std::max<int>(lt.scale, rt.scale);
    int p = std::min(38, std::max(lt.precision - lt.scale, rt.precision - rt.scale) + s + 1);
    e->type.id = T_DECIMAL128; e->type.precision = (uint8_t)p; e->type.scale = (int8_t)s; return e;
  }
  if (lt != rt) bad("arithmetic over " + lt.str() + " and " + rt.str() + ": arrow kernels require equal types");
  if (!(lt.is_integer() || lt.is_float())) unsupported("arithmetic over " + lt.str());
  e->type = lt; return e;
}

ExprP parse_scalar_function(Reader r, const SchemaDef& schema) {   // PhysicalScalarFunctionNode{name=1,fun=2,args=3,return_type=4}
  std::string name; uint64_t fun = 0; std::vector<ExprP> args; DType rt; bool have_rt = false;
  while (!r.done()) {
    int wt; uint32_t f = r.tag(wt);
    if (f == 1) name = r.str(); else if (f == 2) fun = r.varint();
    else if (f == 3) args.push_back(parse_expr(r.bytes(), schema));
    else if (f == 4) { rt = parse_arrow_type(r.bytes()); have_rt = true; }
    else r.skip(wt);
  }
  if (fun != 10000) unsupported("DataFusion built-in scalar function #" + std::to_string(fun) + " is not on the hot path");
  if (!have_rt) bad("Missing required field in protobuf");
  auto e = mk(E_SCALAR_FN); e->name = name; e->children = args; e->type = rt; e->nullable = true;   // from_proto.rs:965-972
  auto lit_i32 = [&](size_t i) { return args.size() > i && args[i]->kind == E_LITERAL && !args[i]->lit_null && args[i]->type.id == T_INT32; };
  if (name == "Placeholder") return e;
  if (name == "UnscaledValue") { if (args.size() != 1 || !args[0]->type.is_decimal()) bad("UnscaledValue expects one decimal argument"); e->type = i64_t(); return e; }
  if (name == "MakeDecimal" || name == "CheckOverflow") {
    if (args.size() != 3 || !lit_i32(1) || !lit_i32(2)) bad(name + ": precision/scale must be int32 literals");
    if (name == "MakeDecimal" && args[0]->type.id != T_INT64) bad("MakeDecimal expects an int64 argument");
    if (name == "CheckOverflow" && !args[0]->type.is_decimal()) bad("CheckOverflow expects a decimal argument");
    int64_t p = (int64_t)args[1]->lit_lo, s = (int64_t)args[2]->lit_lo;
    if (p < 1 || p > 38) bad(name + ": illegal precision");
    e->type.id = T_DECIMAL128; e->type.precision = (uint8_t)p; e->type.scale = (int8_t)s; return e;
  }
  // NullIf / NullIfZero return their argument's value: over a string that is a string-valued expression, which stays off the device
  if ((name == "NullIfZero" || name == "NullIf") && !args.empty() && args[0]->type.is_varlen())
    unsupported(name + " over a " + args[0]->type.str() + " argument is not on the hot path");
  if (name == "NullIfZero") { if (args.size() != 1) bad("NullIfZero expects one argument"); e->type = args[0]->type; return e; }
  if (name == "NullIf") {
    if (args.size() != 2) bad("NullIf expects two arguments");
    if (args[0]->type != args[1]->type) bad("NullIf over different types");
    e->type = args[0]->type; return e;
  }
  if (name == "NormalizeNanAndZero") { if (args.size() != 1 || !args[0]->type.is_float()) bad("NormalizeNanAndZero expects a float"); e->type = args[0]->type; return e; }
  unsupported("spark ext function '" + name + "' is not on the hot path");
}

ExprP parse_expr(Reader r, const SchemaDef& schema) {
  // PhysicalExprNode oneof ExprType (auron.proto:58-125)
  while (!r.done()) {
    int wt; uint32_t f = r.tag(wt);
    switch (f) {
      case 1: {                              // PhysicalColumn{name=1,index=2}: resolved BY NAME (from_proto.rs:850)
        Reader c = r.bytes(); std::string name;
        while (!c.done()) { int w; uint32_t g = c.tag(w); if (g == 1) name = c.str(); else c.skip(w); }
        int idx = schema.index_of(name);
        if (idx < 0) bad("Unable to get field named \"" + name + "\"");
        auto e = mk(E_COLUMN); e->col_index = idx; e->name = name; e->type = schema.fields[idx].type; e->nullable = schema.fields[idx].nullable;
        return e;
      }
      case 2: {                              // ScalarValue{ipc_bytes=1}
        Reader c = r.bytes(); ExprP e;
        while (!c.done()) { int w; uint32_t g = c.tag(w); if (g == 1) { Reader b = c.bytes(); e = decode_ipc_literal(b.p, (size_t)(b.end - b.p)); } else c.skip(w); }
        if (!e) bad("literal without ipc_bytes");
        return e;
      }
      case 3: {                              // BoundReference{index=1,data_type=2,nullable=3}: positional (from_proto.rs:852-855)
        Reader c = r.bytes(); uint64_t idx = 0;
        while (!c.done()) { int w; uint32_t g = c.tag(w); if (g == 1) idx = c.varint(); else c.skip(w); }
        if (idx >= schema.fields.size()) bad("BoundReference index out of range");
        auto e = mk(E_COLUMN); e->col_index = (int)idx; e->name = schema.fields[idx].name; e->type = schema.fields[idx].type; e->nullable = schema.fields[idx].nullable;
        return e;
      }
      case 4: {                              // PhysicalBinaryExprNode{l=1,r=2,op=3}
        Reader c = r.bytes(); ExprP l, rr; std::string op;
        while (!c.done()) { int w; uint32_t g = c.tag(w); if (g == 1) l = parse_expr(c.bytes(), schema); else if (g == 2) rr = parse_expr(c.bytes(), schema); else if (g == 3) op = c.str(); else c.skip(w); }
        if (!l || !rr) bad("Missing required field in protobuf");
        return finish_binary(l, parse_binop(op), rr);
      }
      case 5: bad("Cannot convert aggregate expr node to physical expression");
      case 11: bad("Cannot convert sort expr node to physical expression");
      case 6: { auto e = mk(E_IS_NULL); e->children = {parse_boxed(r.bytes(), 1, schema)}; e->type = bool_t(); e->nullable = false; return e; }
      case 7: { auto e = mk(E_IS_NOT_NULL); e->children = {parse_boxed(r.bytes(), 1, schema)}; e->type = bool_t(); e->nullable = false; return e; }
      case 8: {
        auto e = mk(E_NOT); e->children = {parse_boxed(r.bytes(), 1, schema)};
        if (e->children[0]->type.id != T_BOOL) bad("Not over a non-boolean operand");
        e->type = bool_t(); e->nullable = e->children[0]->nullable; return e;
      }
      case 12: {
        auto e = mk(E_NEGATIVE); e->children = {parse_boxed(r.bytes(), 1, schema)};
        const DType& t = e->children[0]->type;
        if (!(t.is_integer() || t.is_float() || t.is_decimal())) bad("Negative over " + t.str());
        e->type = t; e->nullable = e->children[0]->nullable; return e;
      }
      case 9: {                              // PhysicalCaseNode{expr=1, when_then_expr=2{when=1,then=2}, else_expr=3}
        Reader c = r.bytes(); ExprP base, els; std::vector<std::pair<ExprP, ExprP>> wts;
        while (!c.done()) {
          int w; uint32_t g = c.tag(w);
          if (g == 1) base = parse_expr(c.bytes(), schema);
          else if (g == 2) {
            Reader wt2 = c.bytes(); ExprP we, te;
            while (!wt2.done()) { int w2; uint32_t h = wt2.tag(w2); if (h == 1) we = parse_expr(wt2.bytes(), schema); else if (h == 2) te = parse_expr(wt2.bytes(), schema); else wt2.skip(w2); }
            if (!we || !te) bad("Missing required field in protobuf");
            wts.push_back({we, te});
          } else if (g == 3) els = parse_expr(c.bytes(), schema);
          else c.skip(w);
        }
        if (wts.empty()) bad("There must be at least one WHEN clause");
        auto e = mk(E_CASE); e->case_has_base = (bool)base; e->case_has_else = (bool)els;
        if (base) e->children.push_back(base);
        DType out; bool have = false, nullable = !els;
        for (auto& wt2 : wts) {
          if (base) { if (wt2.first->type != base->type && wt2.first->type.id != T_NULL) bad("CASE: WHEN type differs from the base expression type"); }
          else if (wt2.first->type.id != T_BOOL) bad("CASE: WHEN expression must be boolean");
          if (!have && wt2.second->type.id != T_NULL) { out = wt2.second->type; have = true; }
          nullable = nullable || wt2.second->nullable;
          e->children.push_back(wt2.first); e->children.push_back(wt2.second);
        }
        if (els) { if (!have && els->type.id != T_NULL) { out = els->type; have = true; } nullable = nullable || els->nullable; e->children.push_back(els); }
        for (auto& wt2 : wts) if (wt2.second->type.id != T_NULL && wt2.second->type != out) bad("CASE: THEN expressions have different types");
        if (els && els->type.id != T_NULL && els->type != out) bad("CASE: ELSE type differs from THEN type");
        e->type = out; e->nullable = nullable; return e;
      }
      case 10: case 15: {                    // PhysicalCastNode / PhysicalTryCastNode {expr=1, arrow_type=2}
        Reader c = r.bytes(); ExprP ch; DType to; bool have_t = false;
        while (!c.done()) { int w; uint32_t g = c.tag(w); if (g == 1) ch = parse_expr(c.bytes(), schema); else if (g == 2) { to = parse_arrow_type(c.bytes()); have_t = true; } else c.skip(w); }
        if (!ch || !have_t) bad("Missing required field in protobuf");
        check_cast_supported(ch->type, to, f == 15);
        auto e = mk(f == 10 ? E_CAST : E_TRY_CAST); e->children = {ch}; e->type = to;
        e->nullable = f == 10 ? ch->nullable : true;
        return e;
      }
      case 13: {                             // PhysicalInListNode{expr=1,list=2,negated=3}
        Reader c = r.bytes(); ExprP x; std::vector<ExprP> items; bool neg = false;
        while (!c.done()) { int w; uint32_t g = c.tag(w); if (g == 1) x = parse_expr(c.bytes(), schema); else if (g == 2) items.push_back(parse_expr(c.bytes(), schema)); else if (g == 3) neg = c.varint() != 0; else c.skip(w); }
        if (!x) bad("Missing required field in protobuf");
        auto e = mk(E_IN_LIST); e->negated = neg; e->children.push_back(x); e->type = bool_t(); e->nullable = x->nullable;
        for (auto& it : items) {
          ExprP item = it;
          if (item->type != x->type) { check_cast_supported(item->type, x->type, true); item = wrap_try_cast(item, x->type); }   // from_proto.rs:888-895
          e->nullable = e->nullable || item->nullable;
          e->children.push_back(item);
        }
        return e;
      }
      case 14: return parse_scalar_function(r.bytes(), schema);
      case 3000: case 3001: {                // PhysicalSCAndExprNode / PhysicalSCOrExprNode {left=1,right=2}
        Reader c = r.bytes(); ExprP l, rr;
        while (!c.done()) { int w; uint32_t g = c.tag(w); if (g == 1) l = parse_expr(c.bytes(), schema); else if (g == 2) rr = parse_expr(c.bytes(), schema); else c.skip(w); }
        if (!l || !rr) bad("Missing required field in protobuf");
        auto e = finish_binary(l, f == 3000 ? OP_AND : OP_OR, rr);
        e->kind = f == 3000 ? E_SC_AND : E_SC_OR; return e;
      }
      case 20: unsupported("LIKE is not on the hot path");
      case 10000: case 10001: unsupported("JVM-callback expressions (Spark UDF / scalar subquery wrappers) are not on the hot path");
      case 10002: case 10003: case 11000: unsupported("nested-type expressions are not on the hot path");
      case 20000: case 20001: case 20002: {   // StringStartsWith/EndsWith/ContainsExprNode{expr=1, prefix|suffix|infix=2} (auron.proto:339-352)
        Reader c = r.bytes(); ExprP x; std::string pat;
        while (!c.done()) { int w; uint32_t g = c.tag(w); if (g == 1) x = parse_expr(c.bytes(), schema); else if (g == 2) pat = c.str(); else c.skip(w); }
        if (!x) bad("Missing required field in protobuf");
        if (x->type.id != T_UTF8) bad("string match over a " + x->type.str() + " operand");
        auto e = mk(E_STR_MATCH); e->children = {x}; e->lit_str = pat; e->str_match = (StrMatch)(f - 20000);
        e->type = bool_t(); e->nullable = true;           // string_starts_with.rs:73-79
        return e;
      }
      case 20100: unsupported("RowNum is not on the hot path");
      case 20200: unsupported("BloomFilterMightContain is not on the hot path");
      default: r.skip(wt);
    }
  }
  bad("Unexpected empty physical expression");
}

// TryCast (the reference's TryCastExpr) from Utf8 to a signed integer is Spark's UTF8String.toLong; Cast (DataFusion CastExpr) from
// Utf8 is arrow's parser with other semantics and stays off the device
void check_cast_supported(const DType& from, const DType& to, bool try_cast) {
  if (from == to) return;
  if (from.id == T_NULL || to.id == T_NULL) return;
  if (from.id == T_UTF8 && to.is_integer() && try_cast) return;
  auto num = [](const DType& t) { return t.is_integer() || t.is_float(); };
  bool ok = (num(from) && num(to)) || (from.id == T_BOOL && num(to)) || (num(from) && to.id == T_BOOL) ||
            (from.id == T_DATE32 && to.id == T_INT32) || (from.id == T_INT32 && to.id == T_DATE32) ||
            (from.id == T_TIMESTAMP_US && (to.id == T_INT64 || to.id == T_FLOAT64)) || (from.id == T_INT64 && to.id == T_TIMESTAMP_US) ||
            (from.is_integer() && to.is_decimal()) || (from.is_decimal() && to.is_decimal()) ||
            (from.is_decimal() && (to.is_integer() || to.is_float())) || (from.is_float() && to.is_decimal());
  if (!ok) unsupported("cast " + from.str() + " -> " + to.str() + " is not on the hot path");
  if (to.is_decimal() && to.scale < 0) unsupported("negative decimal scale");
}

// ---- plan nodes ------------------------------------------------------------------------------------------
PlanP parse_plan(Reader r);

PlanP parse_leaf(Reader r, bool ffi) {
  auto n = std::make_shared<PlanNode>(); n->kind = N_LEAF; n->leaf_kind = ffi ? "FFIReader" : "EmptyPartitions";
  bool have = false;
  while (!r.done()) {
    int wt; uint32_t f = r.tag(wt);
    if (ffi) {                               // FFIReaderExecNode{num_partitions=1, schema=2, export_iter_provider_resource_id=3}
      if (f == 2) { n->schema = parse_schema(r.bytes()); have = true; } else if (f == 3) n->resource_id = r.str(); else r.skip(wt);
    } else {                                 // EmptyPartitionsExecNode{schema=1, num_partitions=2}
      if (f == 1) { n->schema = parse_schema(r.bytes()); have = true; } else r.skip(wt);
    }
  }
  if (!have) bad("leaf node without schema");
  return n;
}

// ParquetScanExecNode{base_conf=1, pruning_predicates=2, fsResourceId=3}; FileScanExecConf{num_partitions=1, partition_index=2, file_group=3,
// schema=4, projection=6, limit=7, statistics=8, partition_schema=9} (auron.proto:404-419; from_proto.rs ParquetScan arm)
PlanP parse_parquet_scan(Reader r) {
  auto n = std::make_shared<PlanNode>(); n->kind = N_LEAF; n->leaf_kind = "ParquetScan";
  std::vector<Reader> preds; bool have_conf = false;
  while (!r.done()) {
    int wt; uint32_t f = r.tag(wt);
    if (f == 1) {
      Reader c = r.bytes(); have_conf = true;
      while (!c.done()) {
        int w2; uint32_t g = c.tag(w2);
        if (g == 3) {                                                            // FileGroup{files=1}
          Reader fg = c.bytes();
          while (!fg.done()) {
            int w3; uint32_t h = fg.tag(w3);
            if (h != 1) { fg.skip(w3); continue; }
            Reader pf = fg.bytes(); PlanNode::ScanFile sf;                       // PartitionedFile{path=1,size=2,last_modified_ns=3,partition_values=4,range=5}
            while (!pf.done()) {
              int w4; uint32_t k = pf.tag(w4);
              if (k == 1) sf.path = pf.str(); else if (k == 2) sf.size = pf.varint();
              else if (k == 4) { pf.bytes(); unsupported("parquet scan with partition values (partition columns are appended by the host)"); }
              else if (k == 5) { Reader fr = pf.bytes(); sf.has_range = true; while (!fr.done()) { int w5; uint32_t q = fr.tag(w5); if (q == 1) sf.range_start = (int64_t)fr.varint(); else if (q == 2) sf.range_end = (int64_t)fr.varint(); else fr.skip(w5); } }
              else pf.skip(w4);
            }
            n->scan_files.push_back(sf);
          }
        } else if (g == 4) n->scan_file_schema = parse_schema(c.bytes());
        else if (g == 6) { std::vector<uint64_t> v; c.varints(w2, v); for (uint64_t x : v) n->scan_projection.push_back((int)x); }
        else if (g == 7) { Reader l = c.bytes(); n->scan_has_limit = true; while (!l.done()) { int w3; uint32_t h = l.tag(w3); if (h == 1) n->scan_limit = l.varint(); else l.skip(w3); } }
        else if (g == 9) { SchemaDef ps = parse_schema(c.bytes()); if (!ps.fields.empty()) unsupported("parquet scan with a partition schema"); }
        else c.skip(w2);
      }
    } else if (f == 2) preds.push_back(r.bytes());
    else r.skip(wt);
  }
  if (!have_conf) bad("Missing required field in protobuf");
  if (n->scan_projection.empty()) for (size_t i = 0; i < n->scan_file_schema.fields.size(); i++) n->scan_projection.push_back((int)i);
  for (int i : n->scan_projection) {
    if (i < 0 || (size_t)i >= n->scan_file_schema.fields.size()) bad("parquet scan projection index out of range");
    n->schema.fields.push_back(n->scan_file_schema.fields[(size_t)i]);
  }
  for (auto& p : preds) {
    try { n->scan_pruning.push_back(parse_expr(p, n->scan_file_schema)); } catch (const PlanError&) {}      // pruning is an optimisation: predicates outside the expression subset are dropped
  }
  return n;
}

PlanP parse_filter(Reader r) {               // FilterExecNode{input=1, expr=2}
  auto n = std::make_shared<PlanNode>(); n->kind = N_FILTER;
  std::vector<Reader> exprs;
  while (!r.done()) { int wt; uint32_t f = r.tag(wt); if (f == 1) n->input = parse_plan(r.bytes()); else if (f == 2) exprs.push_back(r.bytes()); else r.skip(wt); }
  if (!n->input) bad("Missing required field in protobuf");
  n->schema = n->input->schema;
  for (auto& e : exprs) n->predicates.push_back(parse_expr(e, n->schema));
  if (n->predicates.empty()) bad("Filter requires at least one predicate");                 // filter_exec.rs:58-60
  for (auto& p : n->predicates) if (p->type.id != T_BOOL) bad("Filter predicate must return boolean values");   // :61-66
  return n;
}

PlanP parse_projection(Reader r) {           // ProjectionExecNode{input=1, expr=2, expr_name=3, data_type=4}
  auto n = std::make_shared<PlanNode>(); n->kind = N_PROJECT;
  std::vector<Reader> exprs; std::vector<std::string> names; std::vector<DType> types;
  while (!r.done()) {
    int wt; uint32_t f = r.tag(wt);
    if (f == 1) n->input = parse_plan(r.bytes()); else if (f == 2) exprs.push_back(r.bytes()); else if (f == 3) names.push_back(r.str());
    else if (f == 4) types.push_back(parse_arrow_type(r.bytes())); else r.skip(wt);
  }
  if (!n->input) bad("Missing required field in protobuf");
  size_t cnt = std::min(exprs.size(), std::min(names.size(), types.size()));   // zip semantics (from_proto.rs:126-129)
  for (size_t i = 0; i < cnt; i++) {
    ExprP e = parse_expr(exprs[i], n->input->schema);
    if (e->type != types[i]) { check_cast_supported(e->type, types[i], true); e = wrap_try_cast(e, types[i]); }   // from_proto.rs:133-137
    n->proj_exprs.push_back(e);
    n->schema.fields.push_back(FieldDef{names[i], e->type, e->nullable});     // project_exec.rs:62-72
  }
  return n;
}

PlanP parse_agg(Reader r) {                  // AggExecNode (auron.proto:675-685)
  auto n = std::make_shared<PlanNode>(); n->kind = N_AGG;
  std::vector<Reader> gexprs, aexprs; std::vector<uint64_t> modes; std::vector<std::string> gnames, anames;
  while (!r.done()) {
    int wt; uint32_t f = r.tag(wt);
    switch (f) {
      case 1: n->input = parse_plan(r.bytes()); break;
      case 2: n->exec_mode = (int)r.varint(); break;
      case 3: gexprs.push_back(r.bytes()); break;
      case 4: aexprs.push_back(r.bytes()); break;
      case 5: r.varints(wt, modes); break;
      case 6: gnames.push_back(r.str()); break;
      case 7: anames.push_back(r.str()); break;
      case 9: n->supports_partial_skipping = r.varint() != 0; break;
      default: r.skip(wt);                   // 8 = initial_input_buffer_offset: sent but ignored natively (agg_ctx.rs:280)
    }
  }
  if (!n->input) bad("Missing required field in protobuf");
  if (n->exec_mode != 0 && n->exec_mode != 1) bad("invalid AggExecMode");
  const SchemaDef& in = n->input->schema;
  size_t ng = std::min(gexprs.size(), gnames.size());
  for (size_t i = 0; i < ng; i++) {
    ExprP e = parse_expr(gexprs[i], in);
    if (e->type.is_varlen() || e->type.id == T_NULL) unsupported("grouping by " + e->type.str() + " is not on the hot path");
    n->group_exprs.push_back(e); n->group_names.push_back(gnames[i]);
    n->schema.fields.push_back(FieldDef{gnames[i], e->type, e->nullable});    // agg_ctx.rs:91-101
  }
  size_t na = std::min(aexprs.size(), std::min(anames.size(), modes.size()));
  for (size_t i = 0; i < na; i++) {
    Reader er = aexprs[i];
    bool found = false; AggDef a; std::vector<ExprP> children; DType rt; bool have_rt = false; uint64_t fn = 0;
    while (!er.done()) {
      int wt; uint32_t f = er.tag(wt);
      if (f == 5) {                          // PhysicalAggExprNode{agg_function=1, udaf=2, children=3, return_type=4}
        found = true; Reader ar = er.bytes();
        while (!ar.done()) {
          int w; uint32_t g = ar.tag(w);
          if (g == 1) fn = ar.varint(); else if (g == 3) children.push_back(parse_expr(ar.bytes(), in));
          else if (g == 4) { rt = parse_arrow_type(ar.bytes()); have_rt = true; } else ar.skip(w);
        }
      } else er.skip(wt);
    }
    if (!found) bad("Invalid aggregate expression for AggExec");
    if (!have_rt) bad("Missing required field in protobuf");
    if (modes[i] > 2) bad("invalid AggMode");
    a.mode = (AggMode)modes[i]; a.field_name = anames[i];
    if (fn > 4) unsupported("aggregate function #" + std::to_string(fn) + " is out of the hot-path scope (variable-length / JVM-callback state)");
    a.fn = (AggFn)fn;
    // create_agg (agg/agg.rs:171-205)
    if (a.fn == AGG_COUNT) {
      a.data_type = i64_t();
      for (auto& c : children) if (c->nullable) a.args.push_back(c);
    } else {
      if (children.empty()) bad("aggregate without children");
      if (a.fn == AGG_SUM || a.fn == AGG_AVG) {
        a.data_type = rt;
        if (a.mode == MODE_PARTIAL) {
          if (!(rt.is_integer() || rt.id == T_FLOAT64 || rt.is_decimal())) unsupported("sum/avg accumulating at " + rt.str() + " is not on the hot path");
          if (children[0]->type.is_varlen()) unsupported(std::string(a.fn == AGG_SUM ? "sum" : "avg") + " over a " + children[0]->type.str() + " column is not on the hot path (cast it to a number first)");
          check_cast_supported(children[0]->type, rt, true);
        }
        a.args.push_back(wrap_try_cast(children[0], rt));
      } else {
        a.data_type = a.mode == MODE_PARTIAL ? children[0]->type : children[0]->type;
        a.args.push_back(children[0]);
      }
      if (a.data_type.is_varlen() || a.data_type.id == T_FLOAT32 && (a.fn == AGG_SUM || a.fn == AGG_AVG))
        unsupported("aggregate over " + a.data_type.str() + " is not on the hot path");
    }
    n->aggs.push_back(a);
  }
  for (auto& a : n->aggs) {
    n->need_partial_update |= a.mode == MODE_PARTIAL;
    n->need_partial_merge |= a.mode != MODE_PARTIAL;
    n->need_final_merge |= a.mode == MODE_FINAL;
  }
  if (n->need_final_merge) for (auto& a : n->aggs) if (a.mode != MODE_FINAL) bad("final aggregates may not exist along with partial/partial-merge");   // agg_ctx.rs:115
  if (n->need_partial_merge) {
    // Min/Max of a merge-mode agg take their type from the (placeholder) child; a placeholder has the
    // Null type, so the merge side needs the real type: it is the type of the partial state, which the
    // reference carries implicitly in the Binary column.  We recover it from the declared return_type.
    if (in.fields.empty()) bad("merge-mode aggregate over an empty input schema");
  }
  if (n->need_final_merge) for (auto& a : n->aggs) n->schema.fields.push_back(FieldDef{a.field_name, a.final_type(), a.nullable()});
  else { DType b; b.id = T_BINARY; n->schema.fields.push_back(FieldDef{AGG_BUF_COLUMN_NAME, b, false}); }   // agg_ctx.rs:130-141
  return n;
}

// PhysicalRepartition (auron.proto:629-655) -> parse_protobuf_partitioning (auron-serde/src/from_proto.rs:1107-1187)
void parse_repartition(Reader r, PlanNode& n, const SchemaDef& schema) {
  bool have = false;
  while (!r.done()) {
    int wt; uint32_t f = r.tag(wt);
    if (f < 1 || f > 4 || wt != 2) { r.skip(wt); continue; }
    Reader b = r.bytes(); have = true;
    n.shuffle_kind = (ShuffleKind)(f - 1); n.num_partitions = 0; n.hash_exprs.clear();
    while (!b.done()) {
      int w2; uint32_t g = b.tag(w2);
      if (f == 1 || f == 3) { if (g == 1) n.num_partitions = b.varint(); else b.skip(w2); }                    // single / round robin: partition_count = 1
      else if (f == 2) { if (g == 1) n.hash_exprs.push_back(parse_expr(b.bytes(), schema)); else if (g == 2) n.num_partitions = b.varint(); else b.skip(w2); }
      else { if (g == 2) n.num_partitions = b.varint(); else b.skip(w2); }                                         // range: sort_expr = 1, partition_count = 2, list_value = 3
    }
    if (f == 1) n.num_partitions = 1;                                                                            // SinglePartitioning()
    if (f == 4 && n.num_partitions == 1) n.shuffle_kind = SHUFFLE_SINGLE;                                        // from_proto.rs:1140-1141
  }
  if (!have) bad("partition::from_proto() Unsupported partition");
}

PlanP parse_shuffle_writer(Reader r) {       // ShuffleWriterExecNode{input=1, output_partitioning=2, output_data_file=3, output_index_file=4}
  auto n = std::make_shared<PlanNode>(); n->kind = N_SHUFFLE_WRITER;
  bool have_part = false; Reader part(nullptr, 0);
  while (!r.done()) {
    int wt; uint32_t f = r.tag(wt);
    if (f == 1) n->input = parse_plan(r.bytes()); else if (f == 2) { part = r.bytes(); have_part = true; }
    else if (f == 3) n->data_file = r.str(); else if (f == 4) n->index_file = r.str(); else r.skip(wt);
  }
  if (!n->input) bad("Missing required field in protobuf");
  if (!have_part) bad("shuffle writer without output_partitioning");        // from_proto.rs:266-270 unwraps it
  n->schema = n->input->schema;                                               // shuffle_writer_exec.rs:76-78
  parse_repartition(part, *n, n->schema);
  return n;
}

PlanP parse_sort(Reader r) {                 // SortExecNode{input=1, expr=2 (PhysicalExprNode.sort = 11), fetch_limit=3{limit=1}}; try_parse_physical_sort_expr
  auto n = std::make_shared<PlanNode>(); n->kind = N_SORT;
  std::vector<Reader> exprs;
  while (!r.done()) {
    int wt; uint32_t f = r.tag(wt);
    if (f == 1) n->input = parse_plan(r.bytes()); else if (f == 2) exprs.push_back(r.bytes());
    else if (f == 3) { Reader fl = r.bytes(); n->sort_has_fetch = true; while (!fl.done()) { int w2; uint32_t g = fl.tag(w2); if (g == 1) n->sort_fetch = fl.varint(); else fl.skip(w2); } }
    else r.skip(wt);
  }
  if (!n->input) bad("Missing required field in protobuf");
  n->schema = n->input->schema;                                             // sort_exec.rs:164-166
  for (auto& e : exprs) {
    Reader er = e; bool found = false;
    while (!er.done()) {
      int wt; uint32_t f = er.tag(wt);
      if (f != 11) { er.skip(wt); continue; }
      Reader sr = er.bytes(); PlanNode::SortExprDef d; d.asc = false; d.nulls_first = false;      // proto3 defaults
      while (!sr.done()) { int w2; uint32_t g = sr.tag(w2); if (g == 1) d.expr = parse_expr(sr.bytes(), n->schema); else if (g == 2) d.asc = sr.varint() != 0; else if (g == 3) d.nulls_first = sr.varint() != 0; else sr.skip(w2); }
      if (!d.expr) bad("physical_plan::from_proto() Unexpected expr: sort expression without an expression");
      n->sort_exprs.push_back(d); found = true;
    }
    if (!found) bad("physical_plan::from_proto() Unexpected expr: expected a sort expression");
  }
  return n;
}

// ExpandExecNode{input=1, schema=2, projections=3}, ExpandProjection{expr=1} (from_proto.rs:518-534) validated like
// ExpandExec::try_new (expand_exec.rs:49-77)
PlanP parse_expand(Reader r) {
  auto n = std::make_shared<PlanNode>(); n->kind = N_EXPAND;
  bool have_schema = false; std::vector<Reader> projs;
  while (!r.done()) {
    int wt; uint32_t f = r.tag(wt);
    if (f == 1) n->input = parse_plan(r.bytes()); else if (f == 2) { n->schema = parse_schema(r.bytes()); have_schema = true; }
    else if (f == 3) projs.push_back(r.bytes()); else r.skip(wt);
  }
  if (!n->input || !have_schema) bad("Missing required field in protobuf");
  const SchemaDef& in = n->input->schema;
  for (auto& pr : projs) {
    std::vector<ExprP> exprs;
    Reader pp = pr;
    while (!pp.done()) { int wt; uint32_t f = pp.tag(wt); if (f == 1) exprs.push_back(parse_expr(pp.bytes(), in)); else pp.skip(wt); }
    for (size_t i = 0; i < n->schema.fields.size(); i++) {
      const DType& want = n->schema.fields[i].type;
      if (i >= exprs.size() || exprs[i]->type != want)
        bad("ExpandExec data type not matches: " + (i < exprs.size() ? "Some(" + exprs[i]->type.str() + ")" : std::string("None")) + " vs " + want.str());
    }
    exprs.resize(n->schema.fields.size());              // execute_expand zips the expressions with the schema fields
    n->expand_projections.push_back(std::move(exprs));
  }
  return n;
}

// WindowExecNode{input=1, window_expr=2, partition_spec=3, order_spec=4, group_limit=5{k=1}, output_window_cols=6},
// WindowExprNode{field=1, return_type=1000, func_type=2, window_func=3, agg_func=4, children=5} (from_proto.rs:535-668),
// validated like WindowContext::try_new and create_agg (agg/agg.rs:171-205)
PlanP parse_window(Reader r) {
  auto n = std::make_shared<PlanNode>(); n->kind = N_WINDOW;
  std::vector<Reader> wexprs, parts, orders;
  while (!r.done()) {
    int wt; uint32_t f = r.tag(wt);
    switch (f) {
      case 1: n->input = parse_plan(r.bytes()); break;
      case 2: wexprs.push_back(r.bytes()); break;
      case 3: parts.push_back(r.bytes()); break;
      case 4: orders.push_back(r.bytes()); break;
      case 5: { Reader gl = r.bytes(); n->window_has_limit = true; while (!gl.done()) { int w2; uint32_t g = gl.tag(w2); if (g == 1) n->window_limit = (uint32_t)gl.varint(); else gl.skip(w2); } break; }
      case 6: n->output_window_cols = r.varint() != 0; break;
      default: r.skip(wt);
    }
  }
  if (!n->input) bad("Missing required field in protobuf");
  const SchemaDef& in = n->input->schema;
  auto check_key = [](const ExprP& e, const char* what) {
    if (e->type.is_varlen() || e->type.id == T_NULL) unsupported(std::string("WindowExec: ") + what + " key of type " + e->type.str() + " is not on the GPU path");
  };
  for (auto& p : parts) { n->window_partition.push_back(parse_expr(p, in)); check_key(n->window_partition.back(), "partition"); }
  for (auto& o : orders) {
    Reader er = o; bool found = false; PlanNode::SortExprDef d; d.asc = false; d.nulls_first = false;
    while (!er.done()) {
      int wt; uint32_t f = er.tag(wt);
      if (f != 11) { er.skip(wt); continue; }
      Reader sr = er.bytes(); found = true;
      while (!sr.done()) { int w2; uint32_t g = sr.tag(w2); if (g == 1) d.expr = parse_expr(sr.bytes(), in); else if (g == 2) d.asc = sr.varint() != 0; else if (g == 3) d.nulls_first = sr.varint() != 0; else sr.skip(w2); }
    }
    if (!found) bad("physical_plan::from_proto() Unexpected expr: a window order_spec entry is not a PhysicalSortExprNode");
    if (!d.expr) bad("physical_plan::from_proto() Unexpected sort expr: sort expression without an expression");
    check_key(d.expr, "order");
    n->window_order.push_back(d);
  }
  if (n->window_partition.size() + n->window_order.size() > (size_t)WINDOW_MAX_KEYS)
    unsupported("WindowExec with more than " + std::to_string(WINDOW_MAX_KEYS) + " partition + order keys is not on the GPU path");
  for (auto& wr : wexprs) {
    Reader er = wr; PlanNode::WindowExprDef w; bool have_field = false, have_rt = false; DType rt; uint64_t func_type = 0, wfn = 0, afn = 0;
    std::vector<ExprP> children;
    while (!er.done()) {
      int wt; uint32_t f = er.tag(wt);
      if (f == 1) { w.field = parse_field(er.bytes()); have_field = true; }
      else if (f == 1000) { rt = parse_arrow_type(er.bytes()); have_rt = true; }
      else if (f == 2) func_type = er.varint(); else if (f == 3) wfn = er.varint(); else if (f == 4) afn = er.varint();
      else if (f == 5) children.push_back(parse_expr(er.bytes(), in));
      else er.skip(wt);
    }
    if (!have_field) bad("physical_plan::from_proto() Unexpected sort expr: window expression without a field");
    if (!have_rt) bad("Missing required field in protobuf");
    DType out;
    if (func_type == 0) {
      if (wfn > 2) bad("invalid WindowFunction");
      w.is_rank = true; w.rank_fn = (int)wfn; out.id = T_INT32;
    } else if (func_type == 1) {
      static const char* names[] = {"MIN", "MAX", "SUM", "AVG", "COUNT", "COLLECT_LIST", "COLLECT_SET", "FIRST", "FIRST_IGNORES_NULL", "BLOOM_FILTER"};
      if (afn > 4) {
        if (afn <= 9 || (afn >= 1000 && afn <= 1002)) unsupported(std::string("window aggregate ") + (afn <= 9 ? names[afn] : afn == 1002 ? "UDAF" : "BRICKHOUSE") + " is not on the GPU path (MIN / MAX / SUM / AVG / COUNT are)");
        bad("invalid AggFunction");
      }
      w.is_rank = false;
      AggDef& a = w.agg; a.fn = (AggFn)afn; a.mode = MODE_PARTIAL; a.field_name = w.field.name;
      if (a.fn == AGG_COUNT) {
        a.data_type = i64_t();
        for (auto& c : children) if (c->nullable) a.args.push_back(c);
        if (a.args.size() > (size_t)WINDOW_MAX_COUNT_ARGS) unsupported("window COUNT of more than " + std::to_string(WINDOW_MAX_COUNT_ARGS) + " nullable arguments is not on the GPU path");
      } else {
        if (children.empty()) bad("aggregate without children");
        const DType ct = children[0]->type;
        if (a.fn == AGG_SUM || a.fn == AGG_AVG) {
          if (ct.is_varlen()) unsupported(std::string("window ") + (a.fn == AGG_SUM ? "SUM" : "AVG") + " over a " + ct.str() + " column is not on the GPU path");
          if (a.fn == AGG_SUM && !(rt.is_integer() || rt.id == T_FLOAT64 || rt.is_decimal())) unsupported("window SUM accumulating at " + rt.str() + " is not on the GPU path");
          if (a.fn == AGG_AVG && !(rt.id == T_FLOAT64 || rt.is_decimal())) unsupported("window AVG returning " + rt.str() + " is not on the GPU path");
          check_cast_supported(ct, rt, true);
          a.data_type = rt;
          a.args.push_back(wrap_try_cast(children[0], rt));
        } else {
          if (ct.id == T_BOOL || ct.is_varlen() || ct.id == T_NULL) unsupported(std::string("window ") + (a.fn == AGG_MIN ? "MIN" : "MAX") + " over " + ct.str() + " is not on the GPU path");
          a.data_type = ct;
          a.args.push_back(children[0]);
        }
      }
      out = a.data_type;
    } else bad("invalid WindowFunctionType");
    if (out != w.field.type) unsupported("WindowExec: window column " + w.field.name + " is computed as " + out.str() + " but its field is " + w.field.type.str() + " (the cast is not on the GPU path)");
    n->window_exprs.push_back(w);
  }
  if (n->window_exprs.size() > (size_t)WINDOW_MAX_EXPRS) unsupported("WindowExec with more than " + std::to_string(WINDOW_MAX_EXPRS) + " window expressions is not on the GPU path");
  if (n->window_has_limit) {
    if (n->window_exprs.size() != 1) bad("WindowExec: a group limit needs exactly one window expression, got " + std::to_string(n->window_exprs.size()));   // window_exec.rs:228
    if (!n->window_exprs[0].is_rank) unsupported("WindowExec: a group limit over an aggregate window column is not on the GPU path (rank-like functions are)");
  }
  n->schema = in;                                                             // WindowContext::try_new: input ++ window fields
  if (n->output_window_cols) for (auto& w : n->window_exprs) n->schema.fields.push_back(w.field);
  return n;
}

// the `~TABLE` column the reference appends to the build side's batches (joins/join_hash_map.rs:409-431, 459-465)
SchemaDef join_hash_map_schema(const SchemaDef& data) {
  SchemaDef s = data;
  for (auto& f : s.fields) f.nullable = true;
  DType b; b.id = T_BINARY; s.fields.push_back(FieldDef{"~TABLE", b, true});
  return s;
}

PlanP parse_join_build(Reader r) {           // BroadcastJoinBuildHashMapExecNode{input=1, keys=2}
  auto n = std::make_shared<PlanNode>(); n->kind = N_JOIN_BUILD;
  std::vector<Reader> keys;
  while (!r.done()) { int wt; uint32_t f = r.tag(wt); if (f == 1) n->input = parse_plan(r.bytes()); else if (f == 2) keys.push_back(r.bytes()); else r.skip(wt); }
  if (!n->input) bad("Missing required field in protobuf");
  for (auto& k : keys) n->join_build_keys.push_back(parse_expr(k, n->input->schema));
  n->schema = join_hash_map_schema(n->input->schema);
  return n;
}

// HashJoinExecNode{schema=1,left=2,right=3,on=4,join_type=5,build_side=6} (from_proto.rs:187-223) and
// BroadcastJoinExecNode{...,broadcast_side=6,cached_build_hash_map_id=7} (from_proto.rs:334-372): both become BroadcastJoinExec
PlanP parse_join(Reader r, bool broadcast) {
  auto n = std::make_shared<PlanNode>(); n->kind = N_JOIN;
  PlanP left, right; std::vector<Reader> on; bool have_schema = false; uint64_t side = 0;
  while (!r.done()) {
    int wt; uint32_t f = r.tag(wt);
    switch (f) {
      case 1: n->schema = parse_schema(r.bytes()); have_schema = true; break;
      case 2: left = parse_plan(r.bytes()); break;
      case 3: right = parse_plan(r.bytes()); break;
      case 4: on.push_back(r.bytes()); break;
      case 5: n->join_type = (int)r.varint(); break;
      case 6: side = r.varint(); break;
      case 7: if (broadcast) n->cached_build_hash_map_id = r.str(); else r.skip(wt); break;
      default: r.skip(wt);
    }
  }
  if (!have_schema || !left || !right) bad("Missing required field in protobuf");
  if (n->join_type < 0 || n->join_type > 6) bad("invalid JoinType");
  if (side > 1) bad(broadcast ? "invalid BroadcastSide" : "invalid BuildSide");
  // a broadcast side arrives wrapped in BroadcastJoinBuildHashMapExec: its data schema is what the join sees
  auto data_schema = [](const PlanP& p) { return p->kind == N_JOIN_BUILD ? p->input->schema : p->schema; };
  n->join_left_schema = data_schema(left); n->join_right_schema = data_schema(right);
  for (auto& o : on) {                         // JoinOn{left=1, right=2}
    Reader jr = o; ExprP l, rr;
    while (!jr.done()) { int wt; uint32_t f = jr.tag(wt); if (f == 1) l = parse_expr(jr.bytes(), n->join_left_schema); else if (f == 2) rr = parse_expr(jr.bytes(), n->join_right_schema); else jr.skip(wt); }
    if (!l || !rr) bad("JoinOn without both sides");
    n->join_on.push_back({l, rr});
  }
  n->join_build_is_left = side == 0;           // JoinSide::LEFT_SIDE = 0 (auron.proto:670-673)
  n->join_build = n->join_build_is_left ? left : right;
  n->input = n->join_build_is_left ? right : left;
  return n;
}

PlanP parse_plan(Reader r) {                  // PhysicalPlanNode oneof (auron.proto:27-55)
  while (!r.done()) {
    int wt; uint32_t f = r.tag(wt);
    switch (f) {
      case 2: return parse_shuffle_writer(r.bytes());
      case 5: return parse_parquet_scan(r.bytes());
      case 6: return parse_projection(r.bytes());
      case 7: return parse_sort(r.bytes());
      case 8: return parse_filter(r.bytes());
      case 11: return parse_join(r.bytes(), false);
      case 12: return parse_join_build(r.bytes());
      case 13: return parse_join(r.bytes(), true);
      case 15: return parse_leaf(r.bytes(), false);
      case 16: return parse_agg(r.bytes());
      case 18: return parse_leaf(r.bytes(), true);
      case 20: return parse_expand(r.bytes());
      case 22: return parse_window(r.bytes());
      case 1: case 3: case 4: case 9: case 10: case 14: case 17: case 19:
      case 21: case 23: case 24: case 25:
        unsupported("plan node #" + std::to_string(f) + " is outside the Filter/Project/Agg hot path (SURVEY.md §8)");
      default: r.skip(wt);
    }
  }
  bad("physical_plan::from_proto() Unsupported physical plan (empty PhysicalPlanType)");
}

const char* binop_name(BinOp op) {
  static const char* n[] = {"And", "Or", "Eq", "NotEq", "Lt", "LtEq", "Gt", "GtEq", "Plus", "Minus", "Multiply", "Divide", "Modulo", "BitwiseAnd", "BitwiseOr", "BitwiseXor"};
  return n[op];
}

}  // namespace

std::string explain_expr(const ExprP& e) {
  std::ostringstream o;
  switch (e->kind) {
    case E_COLUMN: o << e->name << "@" << e->col_index; break;
    case E_LITERAL:
      if (e->lit_null) o << "NULL";
      else if (e->type.is_float()) { double d; memcpy(&d, &e->lit_lo, 8); o << d; }
      else if (e->type.is_decimal()) { o << "dec(" << (int64_t)e->lit_hi << ":" << e->lit_lo << ")"; }
      else if (e->type.id == T_UTF8) o << "'" << e->lit_str << "'";
      else o << (int64_t)e->lit_lo;
      o << ":" << e->type.str(); break;
    case E_BINARY: case E_SC_AND: case E_SC_OR:
      o << "(" << explain_expr(e->children[0]) << " " << (e->kind == E_SC_AND ? "SCAnd" : e->kind == E_SC_OR ? "SCOr" : binop_name(e->op)) << " " << explain_expr(e->children[1]) << ")"; break;
    case E_IS_NULL: o << "IsNull(" << explain_expr(e->children[0]) << ")"; break;
    case E_IS_NOT_NULL: o << "IsNotNull(" << explain_expr(e->children[0]) << ")"; break;
    case E_NOT: o << "Not(" << explain_expr(e->children[0]) << ")"; break;
    case E_NEGATIVE: o << "Negative(" << explain_expr(e->children[0]) << ")"; break;
    case E_CAST: o << "Cast(" << explain_expr(e->children[0]) << " AS " << e->type.str() << ")"; break;
    case E_TRY_CAST: o << "TryCast(" << explain_expr(e->children[0]) << " AS " << e->type.str() << ")"; break;
    case E_CASE: { o << "Case("; for (size_t i = 0; i < e->children.size(); i++) o << (i ? ", " : "") << explain_expr(e->children[i]); o << ")"; break; }
    case E_IN_LIST: { o << explain_expr(e->children[0]) << (e->negated ? " NOT IN (" : " IN ("); for (size_t i = 1; i < e->children.size(); i++) o << (i > 1 ? ", " : "") << explain_expr(e->children[i]); o << ")"; break; }
    case E_STR_MATCH: { static const char* nm[] = {"StartsWith", "EndsWith", "Contains"}; o << nm[e->str_match] << "(" << explain_expr(e->children[0]) << ", '" << e->lit_str << "')"; break; }
    case E_SCALAR_FN: { o << e->name << "("; for (size_t i = 0; i < e->children.size(); i++) o << (i ? ", " : "") << explain_expr(e->children[i]); o << ")"; break; }
  }
  return o.str();
}

static void explain_rec(const PlanP& p, int depth, std::ostringstream& o) {
  std::string ind(depth * 2, ' ');
  auto schema_str = [&](const SchemaDef& s) {
    std::string r = "[";
    for (size_t i = 0; i < s.fields.size(); i++) r += (i ? ", " : "") + s.fields[i].name + ":" + s.fields[i].type.str() + (s.fields[i].nullable ? "?" : "");
    return r + "]";
  };
  switch (p->kind) {
    case N_LEAF:
      o << ind << p->leaf_kind;
      if (p->leaf_kind == "ParquetScan") {
        o << " files=[";
        for (size_t i = 0; i < p->scan_files.size(); i++) { o << (i ? ", " : "") << p->scan_files[i].path; if (p->scan_files[i].has_range) o << "[" << p->scan_files[i].range_start << "," << p->scan_files[i].range_end << ")"; }
        o << "] pruning=[";
        for (size_t i = 0; i < p->scan_pruning.size(); i++) o << (i ? ", " : "") << explain_expr(p->scan_pruning[i]);
        o << "]"; if (p->scan_has_limit) o << " limit=" << p->scan_limit;
      }
      o << " schema=" << schema_str(p->schema) << "\n"; break;
    case N_FILTER:
      o << ind << "FilterExec [";
      for (size_t i = 0; i < p->predicates.size(); i++) o << (i ? ", " : "") << explain_expr(p->predicates[i]);
      o << "] schema=" << schema_str(p->schema) << "\n"; break;
    case N_PROJECT:
      o << ind << "ProjectExec [";
      for (size_t i = 0; i < p->proj_exprs.size(); i++) o << (i ? ", " : "") << explain_expr(p->proj_exprs[i]) << " AS " << p->schema.fields[i].name;
      o << "] schema=" << schema_str(p->schema) << "\n"; break;
    case N_AGG: {
      static const char* fn[] = {"Min", "Max", "Sum", "Avg", "Count"}; static const char* md[] = {"Partial", "PartialMerge", "Final"};
      o << ind << "AggExec " << (p->exec_mode == 0 ? "HashAgg" : "SortAgg") << " groupings=[";
      for (size_t i = 0; i < p->group_exprs.size(); i++) o << (i ? ", " : "") << explain_expr(p->group_exprs[i]) << " AS " << p->group_names[i];
      o << "] aggs=[";
      for (size_t i = 0; i < p->aggs.size(); i++) {
        auto& a = p->aggs[i]; o << (i ? ", " : "") << fn[a.fn] << "(";
        for (size_t j = 0; j < a.args.size(); j++) o << (j ? ", " : "") << explain_expr(a.args[j]);
        o << "):" << a.data_type.str() << "/" << md[a.mode] << " AS " << a.field_name;
      }
      o << "] partial_skipping=" << (p->supports_partial_skipping ? "true" : "false") << " schema=" << schema_str(p->schema) << "\n"; break;
    }
    case N_EXPAND: {
      o << ind << "ExpandExec projections=[";
      for (size_t j = 0; j < p->expand_projections.size(); j++) {
        o << (j ? ", " : "") << "[";
        for (size_t i = 0; i < p->expand_projections[j].size(); i++) o << (i ? ", " : "") << explain_expr(p->expand_projections[j][i]) << " AS " << p->schema.fields[i].name;
        o << "]";
      }
      o << "] schema=" << schema_str(p->schema) << "\n"; break;
    }
    case N_WINDOW: {
      static const char* rank_names[] = {"row_number", "rank", "dense_rank"};
      static const char* agg_names[] = {"MIN", "MAX", "SUM", "AVG", "COUNT"};
      o << ind << "WindowExec: [";
      for (size_t i = 0; i < p->window_exprs.size(); i++) {
        const auto& w = p->window_exprs[i];
        o << (i ? ", " : "");
        if (w.is_rank) o << rank_names[w.rank_fn] << "()";
        else { o << agg_names[w.agg.fn] << "("; for (size_t j = 0; j < w.agg.args.size(); j++) o << (j ? ", " : "") << explain_expr(w.agg.args[j]); o << ")"; }
        o << " AS " << w.field.name << ":" << w.field.type.str();
      }
      o << "] partition_by=[";
      for (size_t i = 0; i < p->window_partition.size(); i++) o << (i ? ", " : "") << explain_expr(p->window_partition[i]);
      o << "] order_by=[";
      for (size_t i = 0; i < p->window_order.size(); i++) o << (i ? ", " : "") << explain_expr(p->window_order[i].expr) << (p->window_order[i].asc ? " ASC" : " DESC") << (p->window_order[i].nulls_first ? " NULLS FIRST" : " NULLS LAST");
      o << "]";
      if (p->window_has_limit) o << " group_limit=" << p->window_limit;
      o << " output_window_cols=" << (p->output_window_cols ? "true" : "false") << "\n";
      break;
    }
    case N_SORT: {
      o << ind << "SortExec [";
      for (size_t i = 0; i < p->sort_exprs.size(); i++) o << (i ? ", " : "") << explain_expr(p->sort_exprs[i].expr) << (p->sort_exprs[i].asc ? " ASC" : " DESC") << (p->sort_exprs[i].nulls_first ? " NULLS FIRST" : " NULLS LAST");
      o << "]"; if (p->sort_has_fetch) o << " fetch=" << p->sort_fetch;
      o << " schema=" << schema_str(p->schema) << "\n"; break;
    }
    case N_JOIN_BUILD: {
      o << ind << "BroadcastJoinBuildHashMapExec keys=[";
      for (size_t i = 0; i < p->join_build_keys.size(); i++) o << (i ? ", " : "") << explain_expr(p->join_build_keys[i]);
      o << "] schema=" << schema_str(p->schema) << "\n"; break;
    }
    case N_JOIN: {
      static const char* jt[] = {"Inner", "Left", "Right", "Full", "LeftSemi", "LeftAnti", "Existence"};
      o << ind << "BroadcastJoinExec " << jt[p->join_type] << " on=[";
      for (size_t i = 0; i < p->join_on.size(); i++) o << (i ? ", " : "") << "(" << explain_expr(p->join_on[i].first) << ", " << explain_expr(p->join_on[i].second) << ")";
      o << "] map_side=" << (p->join_build_is_left ? "Left" : "Right") << " schema=" << schema_str(p->schema) << "\n";
      o << ind << "  [map side]\n"; explain_rec(p->join_build, depth + 2, o);
      o << ind << "  [probed side]\n"; explain_rec(p->input, depth + 2, o);
      return;
    }
    case N_SHUFFLE_WRITER: {
      static const char* kd[] = {"Single", "Hash", "RoundRobin", "Range"};
      o << ind << "ShuffleWriterExec partitioning=" << kd[p->shuffle_kind] << "([";
      for (size_t i = 0; i < p->hash_exprs.size(); i++) o << (i ? ", " : "") << explain_expr(p->hash_exprs[i]);
      o << "], " << p->num_partitions << ") data=" << p->data_file << " index=" << p->index_file << " schema=" << schema_str(p->schema) << "\n"; break;
    }
  }
  if (p->input) explain_rec(p->input, depth + 1, o);
}

std::string explain_plan(const PlanP& p) { std::ostringstream o; explain_rec(p, 0, o); return o.str(); }

PlanP decode_plan(const uint8_t* bytes, size_t n, int plan_kind) {
  if (!bytes && n) bad("null plan bytes");
  Reader r(bytes, n);
  if (plan_kind == B200Q_TASK_DEFINITION) {   // TaskDefinition{task_id=1, plan=2, output_partitioning=3}
    PlanP p;
    while (!r.done()) { int wt; uint32_t f = r.tag(wt); if (f == 2) p = parse_plan(r.bytes()); else r.skip(wt); }
    if (!p) bad("TaskDefinition without plan");
    return p;
  }
  if (plan_kind != B200Q_PLAN_NODE) throw PlanError(B200Q_ERR_INVALID_ARG, "unknown plan_kind");
  return parse_plan(r);
}

}  // namespace b200q
