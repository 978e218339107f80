// The record table of IpcReaderExec (ipc_records.cc): where every column of every batch_serde record lies in the decoded
// byte stream of one push.  Host only, no CUDA: tools/fuzz builds it on its own.
#pragma once
#include <cstddef>
#include <cstdint>
#include <stdexcept>
#include <string>
#include <vector>

#include "ir.h"

namespace b200q {

struct IpcSegment { const uint8_t* p; size_t n; };              // the decompressed payload of one compression block

// stream offsets of one column of one record
struct IpcColExtent {
  int64_t valid = -1;        // validity bitmap ((rows + 7) / 8 bytes), or -1 when the record carries no NULLs for the column
  int64_t values = 0;        // Boolean: value bits; Binary / Utf8: the 4 length planes; else `width` byte planes of `rows` bytes
  int64_t data = 0;          // Binary / Utf8: the row bytes, back to back
  int64_t data_len = 0;
};

struct IpcRecordTable {
  size_t ncols = 0;
  std::vector<int64_t> rows;               // per record
  std::vector<int64_t> start;              // stream offset of each record
  std::vector<IpcColExtent> ext;           // record-major: ext[r * ncols + c]
  size_t count() const { return rows.size(); }
};

// a stream that breaks the format; `offset` is the stream byte where the walk stopped
struct IpcRecordError : std::runtime_error {
  size_t offset;
  IpcRecordError(const std::string& m, size_t off) : std::runtime_error(m), offset(off) {}
};

// Walks every record of the concatenated segments (batch_serde.rs:79-99, restated by oracle/shuffle_oracle.py::read_batch):
// varint row count, then per column a varint null flag (0 or 1) and the bitmap, then the values.  Every extent is checked
// against the stream; Binary / Utf8 lengths are summed from their planes (negative lengths and sums past the stream are
// errors).  The stream must end exactly after a record.  Appends to `out` (whose ncols must equal types.size()).
void ipc_walk_records(const std::vector<IpcSegment>& segs, const std::vector<DType>& types, IpcRecordTable& out);

}  // namespace b200q
