// Record table of IpcReaderExec: the host walks the batch_serde records (batch_serde.rs:79-99) of one push's decoded stream.
// It reads only what it needs to find the next record: the row count, each column's null flag, and for Binary / Utf8 the 4
// length planes (the data that follows is their sum).  The device later reads exactly the extents recorded here.
#include "ipc_records.h"

#include <algorithm>
#include <cstring>

namespace b200q {

namespace {

class Stream {
  const std::vector<IpcSegment>& segs_;
  std::vector<size_t> start_;
  size_t seg_ = 0;
 public:
  size_t total = 0;
  explicit Stream(const std::vector<IpcSegment>& s) : segs_(s) {
    for (auto& g : s) { start_.push_back(total); total += g.n; }
  }
  size_t seg_of(size_t pos) {
    if (seg_ < segs_.size() && pos >= start_[seg_] && pos - start_[seg_] < segs_[seg_].n) return seg_;
    seg_ = (size_t)(std::upper_bound(start_.begin(), start_.end(), pos) - start_.begin()) - 1;
    while (segs_[seg_].n == 0) seg_++;                              // empty segments share their start with the next one
    return seg_;
  }
  uint8_t at(size_t pos) { const size_t s = seg_of(pos); return segs_[s].p[pos - start_[s]]; }
  // bytes [pos, pos + n) (in bounds): in place when they lie in one segment, else gathered into `tmp`
  const uint8_t* span(size_t pos, size_t n, std::vector<uint8_t>& tmp) {
    if (n == 0) return nullptr;
    const size_t s = seg_of(pos);
    if (pos - start_[s] + n <= segs_[s].n) return segs_[s].p + (pos - start_[s]);
    tmp.resize(n);
    for (size_t i = 0; i < n;) {
      const size_t k = seg_of(pos + i), off = pos + i - start_[k], m = std::min(n - i, segs_[k].n - off);
      memcpy(tmp.data() + i, segs_[k].p + off, m); i += m;
    }
    return tmp.data();
  }
};

}  // namespace

void ipc_walk_records(const std::vector<IpcSegment>& segs, const std::vector<DType>& types, IpcRecordTable& out) {
  Stream st(segs);
  const size_t total = st.total, C = types.size();
  std::vector<uint8_t> tmp[4];
  size_t pos = 0;
  auto varint = [&](const char* what) -> uint64_t {                 // io/mod.rs:70-83: 7 bits per byte, low group first
    uint64_t v = 0;
    for (int shift = 0;; shift += 7) {
      if (pos >= total) throw IpcRecordError(std::string("truncated ") + what, pos);
      const uint8_t b = st.at(pos++);
      if (shift == 63 && (b & 0x7E)) throw IpcRecordError(std::string(what) + " above 2^64", pos - 1);
      v |= (uint64_t)(b & 0x7F) << shift;
      if (b < 128) return v;
      if (shift == 63) throw IpcRecordError(std::string(what) + " above 2^64", pos - 1);
    }
  };
  auto need = [&](uint64_t n, const std::string& what) {
    if (n > total - pos) throw IpcRecordError(what + " of " + std::to_string(n) + " bytes runs past the end of the stream (" + std::to_string(total - pos) + " left)", pos);
  };
  while (pos < total) {
    const size_t rec_start = pos;
    const uint64_t n = varint("record row count");
    if (n > 0x7FFFFFFFull) throw IpcRecordError("record row count " + std::to_string(n) + " above 2^31 - 1", rec_start);
    const uint64_t nb = (n + 7) / 8;
    IpcColExtent* ext = nullptr;
    out.rows.push_back((int64_t)n); out.start.push_back((int64_t)rec_start);
    out.ext.resize(out.ext.size() + C);
    ext = out.ext.data() + out.ext.size() - C;
    for (size_t c = 0; c < C; c++) {
      IpcColExtent& e = ext[c];
      const std::string col = "column " + std::to_string(c);
      const uint64_t has_nulls = varint("null flag");
      if (has_nulls > 1) throw IpcRecordError(col + ": null flag " + std::to_string(has_nulls) + " (0 or 1)", pos - 1);
      if (has_nulls) { need(nb, col + ": validity bitmap"); e.valid = (int64_t)pos; pos += nb; }
      e.values = (int64_t)pos;
      const DType& t = types[c];
      if (t.id == T_BOOL) { need(nb, col + ": Boolean values"); pos += nb; }
      else if (t.is_varlen()) {
        need(4 * n, col + ": length planes");
        const uint8_t* p[4];
        for (int k = 0; k < 4; k++) p[k] = st.span(pos + (size_t)k * n, n, tmp[k]);
        uint64_t sum = 0;
        for (uint64_t i = 0; i < n; i++) {
          if (p[3][i] & 0x80) throw IpcRecordError(col + ": negative length at row " + std::to_string(i), pos + 3 * n + i);
          sum += (uint64_t)p[0][i] | ((uint64_t)p[1][i] << 8) | ((uint64_t)p[2][i] << 16) | ((uint64_t)p[3][i] << 24);
        }
        pos += 4 * n;
        need(sum, col + ": row data");
        e.data = (int64_t)pos; e.data_len = (int64_t)sum; pos += sum;
      } else {
        const int w = t.byte_width();
        if (w <= 0) throw IpcRecordError(col + ": type without a batch_serde layout", pos);
        need((uint64_t)w * n, col + ": value planes");
        pos += (size_t)w * n;
      }
    }
  }
}

}  // namespace b200q
