// Parquet metadata and page framing on the host (SURVEY.md §8(f) rank 3: ParquetScanExec decode).
//
// The reference delegates all of this to the un-vendored `parquet` 55.2 crate (datafusion-ext-plans/src/parquet_exec.rs:150-203
// builds DataFusion's ParquetOpener; :316-396 only supplies byte ranges).  What is restated here is the published Apache
// Parquet format (parquet-format 2.x: parquet.thrift, Encodings.md) and Thrift's compact protocol:
//   file   = "PAR1" column chunks ... FileMetaData(thrift) u32 length "PAR1"
//   chunk  = [dictionary page] data pages; page = PageHeader(thrift) + body (compressed as a whole for v1; levels outside for v2)
//   v1 body = [def levels: u32 length + RLE hybrid] values;   dictionary-encoded values = u8 bit width + RLE hybrid indices
// Parity is pinned against a second engine (pyarrow's libparquet reads the same files in tests/test_gpu_parquet.py), as
// SURVEY.md §8(f)-3 prescribes: the reference holds no native golden for this path ("parity unpinned").
#include "parquet_meta.h"

#include <algorithm>
#include <cstring>

#include "../../include/blaze_b200.h"

namespace b200q {

namespace {

[[noreturn]] void bad(const std::string& m) { throw PlanError(B200Q_ERR_EXECUTION, "parquet: " + m); }
[[noreturn]] void unsupported(const std::string& m) { throw PlanError(B200Q_ERR_UNSUPPORTED, "parquet: " + m); }

// ---- Thrift compact protocol --------------------------------------------------------------------------------------
struct TReader {
  const uint8_t* p; const uint8_t* end;
  TReader(const uint8_t* b, size_t n) : p(b), end(b + n) {}
  uint8_t byte() { if (p >= end) bad("truncated thrift data"); return *p++; }
  uint64_t varint() { uint64_t v = 0; int s = 0; while (true) { const uint8_t b = byte(); v |= (uint64_t)(b & 0x7F) << s; if (!(b & 0x80)) return v; s += 7; if (s > 63) bad("thrift varint too long"); } }
  int64_t zigzag() { const uint64_t v = varint(); return (int64_t)(v >> 1) ^ -(int64_t)(v & 1); }
  std::string binary() { const uint64_t n = varint(); if ((uint64_t)(end - p) < n) bad("truncated thrift binary"); std::string s((const char*)p, (size_t)n); p += n; return s; }
  // field header: returns false at STOP; type in `t`, id in `id` (running)
  bool field(int& t, int& id) {
    const uint8_t h = byte();
    if (h == 0) return false;
    t = h & 0x0F;
    const int delta = h >> 4;
    id = delta ? id + delta : (int)zigzag();
    return true;
  }
  void list(int& elem_type, uint64_t& size) { const uint8_t h = byte(); elem_type = h & 0x0F; size = h >> 4; if (size == 15) size = varint(); }
  void skip(int t) {
    switch (t) {
      case 1: case 2: break;                                   // boolean carried by the field header
      case 3: byte(); break;
      case 4: case 5: case 6: varint(); break;
      case 7: if (end - p < 8) bad("truncated double"); p += 8; break;
      case 8: binary(); break;
      case 9: case 10: { int et; uint64_t n; list(et, n); for (uint64_t i = 0; i < n; i++) skip_elem(et); break; }
      case 11: { const uint64_t n = varint(); if (n) { const uint8_t kv = byte(); for (uint64_t i = 0; i < n; i++) { skip_elem(kv >> 4); skip_elem(kv & 0x0F); } } break; }
      case 12: { int ft, id = 0; while (field(ft, id)) skip(ft); break; }
      default: bad("unknown thrift type " + std::to_string(t));
    }
  }
  void skip_elem(int t) { if (t == 1 || t == 2) byte(); else skip(t); }      // booleans inside containers take a byte
};

struct SchemaElement { int type = -1, type_length = 0, repetition = 0, num_children = 0, converted = -1, scale = 0, precision = 0; std::string name;
                       bool l_date = false, l_ts_micros = false, l_ts_other = false, l_decimal = false, l_string = false; int l_int_bits = 0; bool l_int_signed = true; };

void parse_logical_type(TReader& r, SchemaElement& e) {          // union LogicalType
  int t, id = 0;
  while (r.field(t, id)) {
    if (t != 12) { r.skip(t); continue; }
    int ft, fid = 0;
    switch (id) {
      case 1: e.l_string = true; while (r.field(ft, fid)) r.skip(ft); break;
      case 5: e.l_decimal = true; while (r.field(ft, fid)) { if (fid == 1) e.scale = (int)r.zigzag(); else if (fid == 2) e.precision = (int)r.zigzag(); else r.skip(ft); } break;
      case 6: e.l_date = true; while (r.field(ft, fid)) r.skip(ft); break;
      case 8: {                                                  // TIMESTAMP{1: isAdjustedToUTC, 2: unit{1 MILLIS, 2 MICROS, 3 NANOS}}
        bool micros = false;
        while (r.field(ft, fid)) {
          if (fid == 2 && ft == 12) { int ut, uid = 0; while (r.field(ut, uid)) { if (uid == 2) micros = true; r.skip(ut); } }
          else r.skip(ft);
        }
        if (micros) e.l_ts_micros = true; else e.l_ts_other = true;
        break;
      }
      case 10: while (r.field(ft, fid)) { if (fid == 1) e.l_int_bits = (int8_t)r.byte(); else if (fid == 2) e.l_int_signed = ft == 1; else r.skip(ft); } break;
      default: while (r.field(ft, fid)) r.skip(ft);
    }
  }
}

SchemaElement parse_schema_element(TReader& r) {
  SchemaElement e; int t, id = 0;
  while (r.field(t, id)) {
    switch (id) {
      case 1: e.type = (int)r.zigzag(); break;
      case 2: e.type_length = (int)r.zigzag(); break;
      case 3: e.repetition = (int)r.zigzag(); break;
      case 4: e.name = r.binary(); break;
      case 5: e.num_children = (int)r.zigzag(); break;
      case 6: e.converted = (int)r.zigzag(); break;
      case 7: e.scale = (int)r.zigzag(); break;
      case 8: e.precision = (int)r.zigzag(); break;
      case 10: if (t == 12) parse_logical_type(r, e); else r.skip(t); break;
      default: r.skip(t);
    }
  }
  return e;
}

PqStats parse_stats(TReader& r) {
  PqStats s; int t, id = 0;
  while (r.field(t, id)) {
    switch (id) {
      case 1: r.binary(); break;                                   // the deprecated max / min have an undefined sort order: not used for pruning
      case 2: r.binary(); break;
      case 3: s.null_count = r.zigzag(); break;
      case 5: s.max = r.binary(); s.has_max = true; break;
      case 6: s.min = r.binary(); s.has_min = true; break;
      default: r.skip(t);
    }
  }
  return s;
}

PqColumnChunk parse_column_meta(TReader& r) {
  PqColumnChunk c; int t, id = 0;
  while (r.field(t, id)) {
    switch (id) {
      case 1: c.type = (int)r.zigzag(); break;
      case 4: c.codec = (int)r.zigzag(); break;
      case 5: c.num_values = r.zigzag(); break;
      case 6: c.total_uncompressed_size = r.zigzag(); break;
      case 7: c.total_compressed_size = r.zigzag(); break;
      case 9: c.data_page_offset = r.zigzag(); break;
      case 11: c.dictionary_page_offset = r.zigzag(); break;
      case 12: if (t == 12) c.stats = parse_stats(r); else r.skip(t); break;
      default: r.skip(t);
    }
  }
  return c;
}

PqColumnChunk parse_column_chunk(TReader& r) {
  PqColumnChunk c; int t, id = 0; bool have = false;
  while (r.field(t, id)) {
    if (id == 3 && t == 12) { c = parse_column_meta(r); have = true; } else r.skip(t);
  }
  if (!have) bad("column chunk without meta_data");
  return c;
}

PqRowGroup parse_row_group(TReader& r) {
  PqRowGroup g; int t, id = 0;
  while (r.field(t, id)) {
    if (id == 1 && t == 9) { int et; uint64_t n; r.list(et, n); for (uint64_t i = 0; i < n; i++) g.columns.push_back(parse_column_chunk(r)); }
    else if (id == 3) g.num_rows = r.zigzag();
    else r.skip(t);
  }
  return g;
}

DType arrow_type_of(const PqColumnSchema& c) {
  DType d; d.id = T_NULL;
  // unsigned integers (UINT_8..UINT_64) are outside this repo's type subset.  Decided before the width: a uint8 / uint16 column must
  // not pass for int8 / int16 (tests/test_gpu_parquet_edges.py::test_unsupported_shapes_are_refused[uint8])
  const bool is_unsigned = (c.int_bits && !c.int_signed) || (c.converted_type >= 11 && c.converted_type <= 14);
  switch (c.type) {
    case PQ_BOOLEAN: d.id = T_BOOL; break;
    case PQ_INT32:
      if (c.logical_date || c.converted_type == 6) d.id = T_DATE32;
      else if (c.logical_decimal || c.converted_type == 5) { d.id = T_DECIMAL128; d.precision = (uint8_t)c.precision; d.scale = (int8_t)c.scale; }
      else if (is_unsigned) d.id = T_NULL;
      else if (c.int_bits == 8 || c.converted_type == 15) d.id = T_INT8;
      else if (c.int_bits == 16 || c.converted_type == 16) d.id = T_INT16;
      else d.id = T_INT32;
      break;
    case PQ_INT64:
      if (c.logical_ts_micros || c.converted_type == 10) d.id = T_TIMESTAMP_US;
      else if (c.logical_decimal || c.converted_type == 5) { d.id = T_DECIMAL128; d.precision = (uint8_t)c.precision; d.scale = (int8_t)c.scale; }
      else if (c.converted_type == 9 || is_unsigned) d.id = T_NULL;                                                   // millisecond timestamps / unsigned
      else d.id = T_INT64;
      break;
    case PQ_FLOAT: d.id = T_FLOAT32; break;
    case PQ_DOUBLE: d.id = T_FLOAT64; break;
    case PQ_FIXED_LEN_BYTE_ARRAY:
      if ((c.logical_decimal || c.converted_type == 5) && c.type_length >= 1 && c.type_length <= 16) { d.id = T_DECIMAL128; d.precision = (uint8_t)c.precision; d.scale = (int8_t)c.scale; }
      break;
    default: break;                                                                                                    // BYTE_ARRAY (strings), INT96
  }
  return d;
}

}  // namespace

PqFileMeta parquet_parse_footer(const uint8_t* footer, size_t n) {
  TReader r(footer, n);
  PqFileMeta m; std::vector<SchemaElement> schema; int t, id = 0;
  while (r.field(t, id)) {
    switch (id) {
      case 2: { int et; uint64_t cnt; r.list(et, cnt); for (uint64_t i = 0; i < cnt; i++) schema.push_back(parse_schema_element(r)); break; }
      case 3: m.num_rows = r.zigzag(); break;
      case 4: { int et; uint64_t cnt; r.list(et, cnt); for (uint64_t i = 0; i < cnt; i++) m.row_groups.push_back(parse_row_group(r)); break; }
      default: r.skip(t);
    }
  }
  if (schema.empty()) bad("file metadata without a schema");
  // element 0 is the root; a flat schema has only primitive children
  for (size_t i = 1; i < schema.size(); i++) {
    const SchemaElement& e = schema[i];
    if (e.num_children > 0 || e.repetition == 2) { m.flat = false; continue; }
    PqColumnSchema c; c.name = e.name; c.type = e.type; c.type_length = e.type_length; c.optional = e.repetition == 1;
    c.converted_type = e.converted; c.scale = e.scale; c.precision = e.precision;
    c.logical_date = e.l_date; c.logical_ts_micros = e.l_ts_micros; c.logical_decimal = e.l_decimal; c.int_bits = e.l_int_bits; c.int_signed = e.l_int_signed;
    c.arrow = (e.l_ts_other || e.l_string) ? DType{} : arrow_type_of(c);
    if (e.l_ts_other || e.l_string) c.arrow.id = T_NULL;
    m.columns.push_back(c);
  }
  for (auto& g : m.row_groups) if (m.flat && g.columns.size() != m.columns.size()) bad("row group with " + std::to_string(g.columns.size()) + " column chunks, the schema has " + std::to_string(m.columns.size()) + " leaves");
  return m;
}

// ---- Snappy raw format ------------------------------------------------------------------------------------------------
void ByteBuf::reserve(size_t want) {
  if (want <= cap) return;
  size_t nc = (size_t)1 << 16; while (nc < want) nc <<= 1;                       // power-of-two capacities: blocks are interchangeable in the scan's pinned pool
  uint8_t* np = (uint8_t*)(alloc_fn ? alloc_fn(nc) : malloc(nc));
  if (!np) throw PlanError(B200Q_ERR_EXECUTION, "parquet: out of host memory for " + std::to_string(nc) + " bytes of page data");
  if (n) memcpy(np, p, n);
  if (p) { if (free_fn) free_fn(p); else free(p); }
  p = np; cap = nc;
}

size_t snappy_uncompress(const uint8_t* src, size_t n, ByteBuf& out) {
  size_t ip = 0; uint64_t ulen = 0; int shift = 0;
  while (true) { if (ip >= n) bad("snappy: truncated preamble"); const uint8_t b = src[ip++]; ulen |= (uint64_t)(b & 0x7F) << shift; if (!(b & 0x80)) break; shift += 7; if (shift > 35) bad("snappy: bad preamble"); }
  if (ulen > (uint64_t)1 << 31) bad("snappy: block above 2 GiB");
  uint8_t* const dst = out.grow((size_t)ulen);
  const size_t olen = (size_t)ulen;
  size_t op = 0;
  // one element with every bound checked (the tail of the block, long literals, overlapping copies)
  auto careful = [&]() {
    const uint8_t tag = src[ip++];
    size_t len, offset;
    switch (tag & 3) {
      case 0: {
        len = (size_t)(tag >> 2) + 1;
        if (len > 60) { const size_t nb = len - 60; if (ip + nb > n) bad("snappy: truncated literal length"); len = 0; for (size_t i = 0; i < nb; i++) len |= (size_t)src[ip + i] << (8 * i); len += 1; ip += nb; }
        if (ip + len > n || op + len > olen) bad("snappy: literal overruns the buffer");
        memcpy(dst + op, src + ip, len); ip += len; op += len;
        return;
      }
      case 1: if (ip + 1 > n) bad("snappy: truncated copy"); len = (size_t)((tag >> 2) & 7) + 4; offset = ((size_t)(tag >> 5) << 8) | src[ip]; ip += 1; break;
      case 2: if (ip + 2 > n) bad("snappy: truncated copy"); len = (size_t)(tag >> 2) + 1; offset = (size_t)src[ip] | ((size_t)src[ip + 1] << 8); ip += 2; break;
      default: if (ip + 4 > n) bad("snappy: truncated copy"); len = (size_t)(tag >> 2) + 1; offset = (size_t)src[ip] | ((size_t)src[ip + 1] << 8) | ((size_t)src[ip + 2] << 16) | ((size_t)src[ip + 3] << 24); ip += 4; break;
    }
    if (offset == 0 || offset > op || op + len > olen) bad("snappy: copy outside the buffer");
    uint8_t* d = dst + op; const uint8_t* s = d - offset;
    if (offset >= len) memcpy(d, s, len);
    else for (size_t i = 0; i < len; i++) d[i] = s[i];              // overlapping copy: byte-wise (run-length patterns)
    op += len;
  };
  // Fast loop (the usual Snappy decoder tricks): while at least 21 input bytes and 80 output bytes remain, short literals move one 16-byte block
  // and copies with offset >= 8 move 8-byte blocks (they never read what they are about to write).  The blocks may write up to 15 bytes past
  // the element: that slop lies inside this block's output and is overwritten by the elements that follow.
  while (ip + 21 <= n && op + 80 <= olen) {
    const uint8_t tag = src[ip];
    const unsigned kind = tag & 3;
    if (kind == 0) {
      const size_t len = (size_t)(tag >> 2) + 1;
      if (len > 16) { careful(); continue; }
      memcpy(dst + op, src + ip + 1, 16); ip += 1 + len; op += len;
      continue;
    }
    size_t len, offset, adv;
    if (kind == 1) { len = (size_t)((tag >> 2) & 7) + 4; offset = ((size_t)(tag >> 5) << 8) | src[ip + 1]; adv = 2; }
    else if (kind == 2) { len = (size_t)(tag >> 2) + 1; offset = (size_t)src[ip + 1] | ((size_t)src[ip + 2] << 8); adv = 3; }
    else { len = (size_t)(tag >> 2) + 1; offset = (size_t)src[ip + 1] | ((size_t)src[ip + 2] << 8) | ((size_t)src[ip + 3] << 16) | ((size_t)src[ip + 4] << 24); adv = 5; }
    if (offset < 8 || offset > op) { careful(); continue; }         // overlapping pattern or a bad offset: the checked path decides
    uint8_t* d = dst + op; const uint8_t* s = d - offset;           // len <= 64, op + 80 <= olen: the 8-byte blocks stay inside the output
    memcpy(d, s, 8); memcpy(d + 8, s + 8, 8);
    for (size_t i = 16; i < len; i += 8) memcpy(d + i, s + i, 8);
    ip += adv; op += len;
  }
  while (ip < n) careful();
  if (op != olen) bad("snappy: decompressed size mismatch");
  return op;
}

namespace {

struct PageHeader { int type = -1; int32_t uncompressed = 0, compressed = 0; int32_t num_values = 0; int encoding = 0, def_encoding = PQ_RLE;
                    int32_t v2_def_len = 0, v2_rep_len = 0, v2_num_nulls = 0; bool v2_compressed = true; size_t header_len = 0; };

PageHeader parse_page_header(const uint8_t* p, size_t n) {
  TReader r(p, n); PageHeader h; int t, id = 0;
  while (r.field(t, id)) {
    if (id == 1) h.type = (int)r.zigzag();
    else if (id == 2) h.uncompressed = (int32_t)r.zigzag();
    else if (id == 3) h.compressed = (int32_t)r.zigzag();
    else if ((id == 5 || id == 7 || id == 8) && t == 12) {
      int ft, fid = 0;
      while (r.field(ft, fid)) {
        if (id == 5) { if (fid == 1) h.num_values = (int32_t)r.zigzag(); else if (fid == 2) h.encoding = (int)r.zigzag(); else if (fid == 3) h.def_encoding = (int)r.zigzag(); else r.skip(ft); }
        else if (id == 7) { if (fid == 1) h.num_values = (int32_t)r.zigzag(); else if (fid == 2) h.encoding = (int)r.zigzag(); else r.skip(ft); }
        else {
          if (fid == 1) h.num_values = (int32_t)r.zigzag(); else if (fid == 2) h.v2_num_nulls = (int32_t)r.zigzag(); else if (fid == 4) h.encoding = (int)r.zigzag();
          else if (fid == 5) h.v2_def_len = (int32_t)r.zigzag(); else if (fid == 6) h.v2_rep_len = (int32_t)r.zigzag(); else if (fid == 7) h.v2_compressed = ft == 1; else r.skip(ft);
        }
      }
    } else r.skip(t);
  }
  h.header_len = (size_t)(r.p - p);
  return h;
}

// RLE / bit-packed hybrid (Encodings.md): header varint; odd: (header >> 1) groups of 8 bit-packed values; even: a run of (header >> 1)
// copies of one value stored in ceil(bit_width / 8) bytes.  -> runs; bit offsets are relative to `base_bit` (position of data[0])
int64_t hybrid_runs(const uint8_t* data, size_t n, int bit_width, int64_t max_values, std::vector<PqRun>& runs, int64_t* ones /* RLE level runs: values == 1 */) {
  size_t ip = 0; int64_t got = 0; int64_t nonzero = 0;
  const int vbytes = (bit_width + 7) / 8;
  while (got < max_values && ip < n) {
    uint64_t h = 0; int s = 0;
    while (true) { if (ip >= n) bad("truncated RLE header"); const uint8_t b = data[ip++]; h |= (uint64_t)(b & 0x7F) << s; if (!(b & 0x80)) break; s += 7; }
    if (h & 1) {
      const uint64_t groups = h >> 1; uint64_t cnt = groups * 8;
      const size_t bytes = (size_t)groups * bit_width;
      if (ip + bytes > n) { if (bit_width == 0) {} else if (ip + (size_t)(((uint64_t)(max_values - got) * bit_width + 7) / 8) > n) bad("truncated bit-packed run"); }
      if ((int64_t)cnt > max_values - got) cnt = (uint64_t)(max_values - got);
      runs.push_back(PqRun{(uint32_t)cnt, 0u, (uint64_t)ip * 8});
      if (ones) for (uint64_t i = 0; i < cnt; i++) { const uint64_t bit = (uint64_t)ip * 8 + i * bit_width; nonzero += (data[bit >> 3] >> (bit & 7)) & 1; }    // levels: bit_width == 1
      ip += bytes; got += (int64_t)cnt;
    } else {
      uint64_t cnt = h >> 1;
      if (ip + vbytes > n) bad("truncated RLE run");
      uint64_t v = 0; for (int i = 0; i < vbytes; i++) v |= (uint64_t)data[ip + i] << (8 * i);
      ip += vbytes;
      if ((int64_t)cnt > max_values - got) cnt = (uint64_t)(max_values - got);
      if (cnt) runs.push_back(PqRun{(uint32_t)cnt, 1u, v});
      if (ones && v) nonzero += (int64_t)cnt;
      got += (int64_t)cnt;
    }
  }
  if (got < max_values) bad("RLE data ends after " + std::to_string(got) + " of " + std::to_string(max_values) + " values");
  if (ones) *ones = nonzero;
  return (int64_t)ip;
}

}  // namespace

std::vector<PqPage> parquet_read_pages(const uint8_t* chunk, size_t n, const PqColumnChunk& cc, const PqColumnSchema& cs, ByteBuf& out, ByteBuf& dict_out) {
  out.clear(); dict_out.clear();
  if (cc.codec != PQ_UNCOMPRESSED && cc.codec != PQ_SNAPPY) unsupported("compression codec " + std::to_string(cc.codec) + " (only UNCOMPRESSED and SNAPPY are decoded)");
  std::vector<PqPage> pages;
  size_t pos = 0; int64_t seen = 0;
  while (pos < n && seen < cc.num_values) {
    const PageHeader h = parse_page_header(chunk + pos, n - pos);
    pos += h.header_len;
    if (h.compressed < 0 || pos + (size_t)h.compressed > n) bad("page body overruns its column chunk");
    const uint8_t* body = chunk + pos; const size_t blen = (size_t)h.compressed;
    pos += blen;
    if (h.type == PQ_INDEX_PAGE) continue;
    PqPage pg; pg.type = h.type; pg.num_values = h.num_values; pg.encoding = h.encoding;
    ByteBuf& dst = h.type == PQ_DICTIONARY_PAGE ? dict_out : out;
    pg.base = dst.size();
    size_t levels = 0;
    if (h.type == PQ_DATA_PAGE_V2) {                               // levels are stored uncompressed in front of the (optionally compressed) values
      levels = (size_t)h.v2_rep_len + (size_t)h.v2_def_len;
      if (levels > blen) bad("v2 level bytes overrun the page");
      if (h.v2_rep_len) unsupported("repetition levels (nested columns)");
      dst.append(body, levels);
      if (cc.codec == PQ_SNAPPY && h.v2_compressed && blen > levels) snappy_uncompress(body + levels, blen - levels, dst);
      else dst.append(body + levels, blen - levels);
    } else if (cc.codec == PQ_SNAPPY) snappy_uncompress(body, blen, dst);
    else dst.append(body, blen);
    pg.size = dst.size() - pg.base;
    if (h.type == PQ_DICTIONARY_PAGE) {
      if (h.encoding != PQ_PLAIN && h.encoding != PQ_PLAIN_DICTIONARY) unsupported("dictionary page encoding " + std::to_string(h.encoding));
      pg.values_offset = 0; pg.non_null = h.num_values;
      pages.push_back(std::move(pg));
      continue;
    }
    const uint8_t* pb = dst.data() + pg.base;                        // valid until the next append (offsets are kept, not pointers)
    if (h.type != PQ_DATA_PAGE && h.type != PQ_DATA_PAGE_V2) unsupported("page type " + std::to_string(h.type));
    seen += h.num_values;
    size_t at = 0;
    pg.non_null = h.num_values;
    if (cs.optional) {                                             // definition levels, max level 1 (flat schema)
      int64_t ones = 0;
      if (h.type == PQ_DATA_PAGE) {
        if (h.def_encoding != PQ_RLE) unsupported("definition level encoding " + std::to_string(h.def_encoding));
        if (pg.size < 4) bad("page without definition levels");
        uint32_t len; memcpy(&len, pb, 4);
        if (4 + (size_t)len > pg.size) bad("definition levels overrun the page");
        hybrid_runs(pb + 4, len, 1, h.num_values, pg.def_runs, &ones);
        for (auto& r : pg.def_runs) if (!r.is_rle) r.value_or_bit_offset += 32;          // bit offsets relative to bytes[0]
        at = 4 + len;
      } else {
        hybrid_runs(pb, (size_t)h.v2_def_len, 1, h.num_values, pg.def_runs, &ones);
        at = levels;
      }
      pg.non_null = ones;
      if (ones == h.num_values) pg.def_runs.clear();               // every value present
    } else if (h.type == PQ_DATA_PAGE_V2) at = levels;
    pg.values_offset = at;
    if (h.encoding == PQ_PLAIN_DICTIONARY || h.encoding == PQ_RLE_DICTIONARY) {
      if (pg.non_null > 0) {
        if (at >= pg.size) bad("dictionary-encoded page without a bit width");
        pg.dict_bit_width = pb[at];
        if (pg.dict_bit_width > 32) bad("dictionary index width " + std::to_string(pg.dict_bit_width));
        hybrid_runs(pb + at + 1, pg.size - at - 1, pg.dict_bit_width, pg.non_null, pg.idx_runs, nullptr);
        for (auto& r : pg.idx_runs) if (!r.is_rle) r.value_or_bit_offset += (uint64_t)(at + 1) * 8;
      }
    } else if (h.encoding == PQ_PLAIN) {
    } else if (h.encoding == PQ_RLE && cs.type == PQ_BOOLEAN) {     // v2 Boolean values: u32 length + RLE hybrid of width 1
      if (at + 4 > pg.size) bad("RLE Boolean page without a length");
      uint32_t len; memcpy(&len, pb + at, 4);
      pg.dict_bit_width = 1;
      hybrid_runs(pb + at + 4, len, 1, pg.non_null, pg.idx_runs, nullptr);
      for (auto& r : pg.idx_runs) if (!r.is_rle) r.value_or_bit_offset += (uint64_t)(at + 4) * 8;
    } else unsupported("value encoding " + std::to_string(h.encoding) + " (PLAIN and RLE_DICTIONARY are decoded)");
    pages.push_back(std::move(pg));
  }
  return pages;
}

}  // namespace b200q
