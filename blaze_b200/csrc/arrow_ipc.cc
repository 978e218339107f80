// Minimal Arrow IPC *stream* reader for plan literals.
//
// The reference ships every literal as `ScalarValue{ipc_bytes}` = a complete IPC stream written by
// arrow-java's ArrowStreamWriter holding one schema message and one 1-row record batch whose single
// field is named "" (spark-extension/.../NativeConverters.scala:382-403); the native side reads
// column 0, row 0 (auron-serde/src/lib.rs:447-457).  We decode exactly that shape by hand: the
// encapsulated-message framing and the three flatbuffer tables involved (Message, Schema/Field/Type,
// RecordBatch) as laid out by Arrow's format/Message.fbs + Schema.fbs.
#include <cstring>

#include "../../include/blaze_b200.h"
#include "ir.h"

namespace b200q {
namespace {

struct Buf {
  const uint8_t* p; size_t n;
  void need(size_t off, size_t len) const { if (off + len > n || off + len < off) throw PlanError(B200Q_ERR_INVALID_PLAN, "literal ipc_bytes: truncated flatbuffer"); }
  template <class T> T rd(size_t off) const { need(off, sizeof(T)); T v; memcpy(&v, p + off, sizeof(T)); return v; }
};

// flatbuffer table accessor
struct Table {
  Buf b; size_t pos; size_t vt; uint16_t vtsize;
  Table(Buf buf, size_t table_pos) : b(buf), pos(table_pos) {
    int32_t soff = b.rd<int32_t>(pos);
    vt = (size_t)((int64_t)pos - soff);
    vtsize = b.rd<uint16_t>(vt);
  }
  size_t field_off(int idx) const {   // 0 if absent
    size_t slot = 4 + 2 * (size_t)idx;
    if (slot + 2 > vtsize) return 0;
    uint16_t o = b.rd<uint16_t>(vt + slot);
    return o ? pos + o : 0;
  }
  template <class T> T scalar(int idx, T dflt) const { size_t o = field_off(idx); return o ? b.rd<T>(o) : dflt; }
  bool has(int idx) const { return field_off(idx) != 0; }
  size_t indirect(int idx) const { size_t o = field_off(idx); if (!o) return 0; return o + b.rd<uint32_t>(o); }   // table/vector/string position
};

struct Vec { Buf b; size_t pos; uint32_t len; Vec(Buf buf, size_t p) : b(buf), pos(p + 4), len(buf.rd<uint32_t>(p)) {} };

// Arrow `Type` union tags (Schema.fbs)
enum { TY_Null = 1, TY_Int = 2, TY_FloatingPoint = 3, TY_Binary = 4, TY_Utf8 = 5, TY_Bool = 6, TY_Decimal = 7, TY_Date = 8,
       TY_Time = 9, TY_Timestamp = 10 };
enum { HDR_Schema = 1, HDR_DictionaryBatch = 2, HDR_RecordBatch = 3 };

struct Msg { uint8_t header_type; size_t header_pos; int64_t body_len; Buf meta; size_t body_off; };

// returns false at end-of-stream
bool next_message(const uint8_t* bytes, size_t n, size_t& cur, Msg& m) {
  if (cur + 4 > n) return false;
  uint32_t w; memcpy(&w, bytes + cur, 4); cur += 4;
  if (w == 0xFFFFFFFFu) {                       // continuation marker (format >= 0.15)
    if (cur + 4 > n) return false;
    memcpy(&w, bytes + cur, 4); cur += 4;
  }
  if (w == 0) return false;                     // EOS
  if (cur + w > n) throw PlanError(B200Q_ERR_INVALID_PLAN, "literal ipc_bytes: truncated message");
  m.meta = Buf{bytes + cur, w};
  uint32_t root = m.meta.rd<uint32_t>(0);
  Table t(m.meta, root);
  m.header_type = t.scalar<uint8_t>(1, 0);
  m.header_pos = t.indirect(2);
  m.body_len = t.scalar<int64_t>(3, 0);
  cur += w;
  m.body_off = cur;
  if (m.body_len < 0 || cur + (size_t)m.body_len > n) throw PlanError(B200Q_ERR_INVALID_PLAN, "literal ipc_bytes: truncated body");
  cur += (size_t)m.body_len;
  return true;
}

DType parse_field_type(const Table& field, bool allow_binary) {
  uint8_t tt = field.scalar<uint8_t>(2, 0);
  size_t tp = field.indirect(3);
  DType d;
  switch (tt) {
    case TY_Null: d.id = T_NULL; return d;
    case TY_Bool: d.id = T_BOOL; return d;
    case TY_Int: {
      Table t(field.b, tp);
      int32_t bw = t.scalar<int32_t>(0, 0); bool sg = t.scalar<uint8_t>(1, 0) != 0;
      if (!sg) throw PlanError(B200Q_ERR_UNSUPPORTED, "literal: unsigned integers are not on the hot path");
      d.id = bw == 8 ? T_INT8 : bw == 16 ? T_INT16 : bw == 32 ? T_INT32 : T_INT64;
      if (bw != 8 && bw != 16 && bw != 32 && bw != 64) throw PlanError(B200Q_ERR_INVALID_PLAN, "literal: bad int bit width");
      return d;
    }
    case TY_FloatingPoint: {
      Table t(field.b, tp);
      int16_t prec = t.scalar<int16_t>(0, 0);
      if (prec == 1) d.id = T_FLOAT32; else if (prec == 2) d.id = T_FLOAT64;
      else throw PlanError(B200Q_ERR_UNSUPPORTED, "literal: float16 is not on the hot path");
      return d;
    }
    case TY_Decimal: {
      Table t(field.b, tp);
      int32_t p = t.scalar<int32_t>(0, 0), s = t.scalar<int32_t>(1, 0), bw = t.scalar<int32_t>(2, 128);
      if (bw != 128) throw PlanError(B200Q_ERR_UNSUPPORTED, "literal: only decimal128");
      d.id = T_DECIMAL128; d.precision = (uint8_t)p; d.scale = (int8_t)s; return d;
    }
    case TY_Date: {
      Table t(field.b, tp);
      int16_t unit = t.scalar<int16_t>(0, 1);
      if (unit != 0) throw PlanError(B200Q_ERR_UNSUPPORTED, "literal: only date32[day]");
      d.id = T_DATE32; return d;
    }
    case TY_Timestamp: {
      Table t(field.b, tp);
      int16_t unit = t.scalar<int16_t>(0, 0);
      if (unit != 2) throw PlanError(B200Q_ERR_UNSUPPORTED, "literal: only timestamp[us]");
      d.id = T_TIMESTAMP_US; return d;
    }
    case TY_Utf8: d.id = T_UTF8; return d;
    case TY_Binary:
      if (allow_binary) { d.id = T_BINARY; return d; }
      throw PlanError(B200Q_ERR_UNSUPPORTED, "literal: binary literals are not on the hot path");
    default:
      throw PlanError(B200Q_ERR_UNSUPPORTED, "literal: unsupported arrow type tag " + std::to_string(tt));
  }
}

}  // namespace

ExprP decode_ipc_literal(const uint8_t* bytes, size_t n, bool allow_binary) {
  size_t cur = 0;
  Msg m;
  bool have_schema = false, have_batch = false;
  auto e = std::make_shared<Expr>();
  e->kind = E_LITERAL;
  while (next_message(bytes, n, cur, m)) {
    if (m.header_type == HDR_Schema) {
      Table schema(m.meta, m.header_pos);
      if (schema.scalar<int16_t>(0, 0) != 0) throw PlanError(B200Q_ERR_UNSUPPORTED, "literal: big-endian IPC");
      size_t fv = schema.indirect(1);
      if (!fv) throw PlanError(B200Q_ERR_INVALID_PLAN, "literal: schema without fields");
      Vec fields(m.meta, fv);
      if (fields.len < 1) throw PlanError(B200Q_ERR_INVALID_PLAN, "literal: schema without fields");
      size_t f0 = fields.pos + m.meta.rd<uint32_t>(fields.pos);
      e->type = parse_field_type(Table(m.meta, f0), allow_binary);
      have_schema = true;
    } else if (m.header_type == HDR_RecordBatch) {
      if (!have_schema) throw PlanError(B200Q_ERR_INVALID_PLAN, "literal: record batch before schema");
      Table rb(m.meta, m.header_pos);
      int64_t length = rb.scalar<int64_t>(0, 0);
      if (length < 1) throw PlanError(B200Q_ERR_INVALID_PLAN, "literal: empty record batch");
      if (rb.has(3)) throw PlanError(B200Q_ERR_UNSUPPORTED, "literal: compressed IPC body");
      Vec nodes(m.meta, rb.indirect(1));      // struct FieldNode{int64 length; int64 null_count}
      Vec bufs(m.meta, rb.indirect(2));       // struct Buffer{int64 offset; int64 length}
      if (nodes.len < 1) throw PlanError(B200Q_ERR_INVALID_PLAN, "literal: no field node");
      int64_t null_count = m.meta.rd<int64_t>(nodes.pos + 8);
      auto buf_at = [&](uint32_t i, int64_t& off, int64_t& len) {
        if (i >= bufs.len) throw PlanError(B200Q_ERR_INVALID_PLAN, "literal: missing buffer");
        off = m.meta.rd<int64_t>(bufs.pos + 16 * (size_t)i); len = m.meta.rd<int64_t>(bufs.pos + 16 * (size_t)i + 8);
        if (off < 0 || len < 0 || len > (int64_t)m.body_len || off > (int64_t)m.body_len - len) throw PlanError(B200Q_ERR_INVALID_PLAN, "literal: buffer out of body");
      };
      const uint8_t* body = bytes + m.body_off;
      if (e->type.id == T_NULL) { e->lit_null = true; have_batch = true; break; }
      int64_t voff, vlen, doff, dlen;
      buf_at(0, voff, vlen); buf_at(1, doff, dlen);
      bool valid = true;
      if (null_count > 0) valid = vlen > 0 ? (body[voff] & 1) != 0 : false;
      e->lit_null = !valid;
      if (valid && e->type.is_varlen()) {          // Utf8 / Binary buffers: validity, int32 offsets (row 0: [o0, o1)), data
        int64_t xoff, xlen; buf_at(2, xoff, xlen);
        if (dlen < 8) throw PlanError(B200Q_ERR_INVALID_PLAN, "literal: " + e->type.str() + " offsets buffer too short");
        int32_t o0, o1; memcpy(&o0, body + doff, 4); memcpy(&o1, body + doff + 4, 4);
        if (o0 < 0 || o1 < o0 || (int64_t)o1 > xlen) throw PlanError(B200Q_ERR_INVALID_PLAN, "literal: " + e->type.str() + " offsets out of the data buffer");
        e->lit_str.assign((const char*)body + xoff + o0, (size_t)(o1 - o0));
      } else if (valid) {
        const uint8_t* d = body + doff;
        auto need = [&](int64_t w) { if (dlen < w) throw PlanError(B200Q_ERR_INVALID_PLAN, "literal: value buffer too short"); };
        switch (e->type.id) {
          case T_BOOL: need(1); e->lit_lo = d[0] & 1; break;
          case T_INT8: { need(1); int8_t v; memcpy(&v, d, 1); e->lit_lo = (uint64_t)(int64_t)v; break; }
          case T_INT16: { need(2); int16_t v; memcpy(&v, d, 2); e->lit_lo = (uint64_t)(int64_t)v; break; }
          case T_INT32: case T_DATE32: { need(4); int32_t v; memcpy(&v, d, 4); e->lit_lo = (uint64_t)(int64_t)v; break; }
          case T_INT64: case T_TIMESTAMP_US: { need(8); memcpy(&e->lit_lo, d, 8); break; }
          case T_FLOAT32: { need(4); float f; memcpy(&f, d, 4); double dd = (double)f; memcpy(&e->lit_lo, &dd, 8); break; }
          case T_FLOAT64: { need(8); memcpy(&e->lit_lo, d, 8); break; }
          case T_DECIMAL128: { need(16); memcpy(&e->lit_lo, d, 8); memcpy(&e->lit_hi, d + 8, 8); break; }
          default: throw PlanError(B200Q_ERR_UNSUPPORTED, "literal: unsupported type");
        }
      }
      have_batch = true;
      break;   // the reference reads only the first batch
    }
  }
  if (!have_schema || !have_batch) throw PlanError(B200Q_ERR_INVALID_PLAN, "literal ipc_bytes: missing record batch");
  e->nullable = e->lit_null;
  return e;
}

}  // namespace b200q
