// Host runtime of the operator pipeline behind the C ABI (include/blaze_b200.h).
//
// An op = a chain of stages compiled from the plan subtree:
//   FilterProjectStage  FilterExec / ProjectExec chain fused into one kernel   (filter_exec.rs, project_exec.rs)
//   AggStage            AggExec with everything below it (Filter/Project) fused into its update kernel (agg_exec.rs)
// Batches between stages stay in HBM.
#pragma once
#include <cuda_runtime.h>

#include <algorithm>
#include <deque>
#include <functional>
#include <memory>
#include <string>
#include <vector>

#include "../../include/blaze_b200.h"
#include "compile.h"
#include "ir.h"
#include "kernels.cuh"

namespace b200q {

struct CudaError : std::runtime_error {
  CudaError(const std::string& m) : std::runtime_error(m) {}
};
struct ExecError : std::runtime_error {
  int code;
  ExecError(int c, const std::string& m) : std::runtime_error(m), code(c) {}
};

#define B200Q_CUDA(expr)                                                                                      \
  do {                                                                                                        \
    cudaError_t _e = (expr);                                                                                  \
    if (_e != cudaSuccess) throw ::b200q::CudaError(std::string(#expr) + ": " + cudaGetErrorString(_e));      \
  } while (0)

// The op's CUDA stream outlives the op while exported device arrays still reference allocations made on it
// (their release frees stream-ordered memory): the stream returns to the device's pool when the last reference goes away.
struct StreamRef {
  cudaStream_t s = nullptr; int device = 0;
  ~StreamRef();
};
std::shared_ptr<StreamRef> stream_ref_create(int device);      // a recycled stream of `device` when one is free
std::shared_ptr<StreamRef> stream_ref_lookup(cudaStream_t s);
// per-device pool of events (`timing`: created without cudaEventDisableTiming); get with `device` current.  An event may be
// put back while a record of it is still pending: its next user records it again before waiting on it
cudaEvent_t event_get(int device, bool timing);
void event_put(int device, cudaEvent_t e, bool timing);

// a device allocation (stream-ordered) or a borrowed device pointer kept alive by `owner`
struct DevMem {
  void* ptr = nullptr;
  size_t bytes = 0;
  cudaStream_t stream = nullptr;
  bool owned = false;
  std::shared_ptr<void> owner;
  std::shared_ptr<StreamRef> stream_keep;
  ~DevMem();
  static std::shared_ptr<DevMem> alloc(size_t bytes, cudaStream_t s, bool zero = false);
  static std::shared_ptr<DevMem> borrow(const void* p, size_t bytes, std::shared_ptr<void> owner);
};
using DevMemP = std::shared_ptr<DevMem>;

struct DevColumn {
  DType type;
  DevMemP values;        // fixed-width values / bit-packed bools / binary data
  DevMemP validity;      // bitmap or null
  DevMemP offsets;       // binary only (int32)
  int64_t offset = 0;    // Arrow element offset (applies to values, validity and offsets)
};

struct DevBatch {
  std::vector<DevColumn> cols;
  int64_t num_rows = 0;
};

struct Metrics {
  int64_t input_rows = 0, input_batches = 0, output_rows = 0, output_batches = 0;
  int64_t launches = 0, fast_launches = 0, h2d_bytes = 0, d2h_bytes = 0;
  int64_t num_groups = 0, table_capacity = 0, grow_count = 0;
  double gpu_ms = 0;
  double hot_ms = 0; int64_t hot_rows = 0, hot_launches = 0;
};

struct OpContext {
  int device = 0;
  cudaStream_t stream = nullptr;
  b200q_conf conf;
  Metrics m;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;   // timing of the dominant kernel on `stream`
  int cur_stage = 0;                          // hot_kernel_* metrics describe stage 0 (the stage that sees the input rows)
};

class Stage {
 public:
  virtual ~Stage() {}
  SchemaDef in_schema, out_schema;
  std::vector<int> used_input_cols;      // which input columns the stage reads (column pruning, column_pruning.rs:68-90)
  virtual void push(OpContext& cx, DevBatch& in, std::vector<DevBatch>& outs) = 0;
  virtual void finish(OpContext& cx, std::vector<DevBatch>& outs) = 0;
};

std::unique_ptr<Stage> make_filter_project_stage(OpContext& cx, const SchemaDef& in_schema, const std::vector<ExprP>& filters,
                                                 const std::vector<ExprP>& outs, const SchemaDef& out_schema);
// ExpandExec not fused into an aggregate: every pushed batch yields one batch per projection, in order (expand_exec.rs:147-187)
std::unique_ptr<Stage> make_expand_stage(OpContext& cx, const SchemaDef& in_schema, const std::vector<ExprP>& filters,
                                         const std::vector<std::vector<ExprP>>& projections, const SchemaDef& out_schema);
// one projection of an ExpandExec fused below AggExec(Partial): its grouping keys and aggregate arguments over the stage input
struct AggSetExprs { std::vector<ExprP> group_exprs; std::vector<std::vector<ExprP>> agg_args; };
// `sets` (two or more): every input row is inserted once per set; empty: group_exprs / agg_args are the one set
std::unique_ptr<Stage> make_agg_stage(OpContext& cx, const SchemaDef& in_schema, const std::vector<ExprP>& filters, const PlanNode& agg,
                                      const std::vector<ExprP>& group_exprs, const std::vector<std::vector<ExprP>>& agg_args,
                                      const std::vector<AggSetExprs>& sets = {});

// AggExec whose aggregates are all BLOOM_FILTER, without grouping keys (bloom_stage.cu).  Partial: value_cols[i] is the input
// column of aggregate i's value; merge modes read the Binary state column(s) of the input
std::unique_ptr<Stage> make_bloom_agg_stage(OpContext& cx, const SchemaDef& in_schema, const PlanNode& agg, const std::vector<int>& value_cols);

// ShuffleWriterExec (shuffle_stage.cu): terminal stage; its result is the two shuffle files and/or the encoded chunks
std::unique_ptr<Stage> make_shuffle_write_stage(OpContext& cx, const SchemaDef& in_schema, const PlanNode& node);
struct ShuffleResult {
  virtual ~ShuffleResult() {}
  virtual int64_t chunk_count() const = 0;
  virtual void chunk(int64_t i, b200q_shuffle_chunk* out) const = 0;
};

// ParquetScanExec (parquet_source.cu): the source of an op whose leaf is a ParquetScanExecNode; `emit` receives one device batch per row group
void run_parquet_scan(OpContext& cx, const PlanNode& leaf, const std::function<void(DevBatch&)>& emit);
void set_file_reader(b200q_file_reader_fn fn, void* ctx);
// the process-wide pool of pinned host blocks (parquet_source.cu) the scan and the IpcReaderExec source stage their bytes in;
// pinned_alloc returns null when the driver refuses the allocation
void* pinned_alloc(size_t n);
void pinned_free(void* p);

// IpcReaderExec (ipc_source.cu): the source of an op whose leaf is an IpcReaderExecNode.  push() takes the bytes of one BlockObject
// (`u32 LE length ‖ LZ4 frame` blocks), decompresses them on host threads into pinned blocks, walks their batch_serde records and
// uploads them; the records accumulate into one device batch of up to conf.staging_rows rows, decoded on the device and handed to
// `emit` (at push when full, at flush otherwise).  Malformed input -> ExecError(INVALID_ARG) before anything of the push is kept.
class IpcSource {
 public:
  virtual ~IpcSource() {}
  virtual void push(OpContext& cx, const uint8_t* data, size_t len, const std::function<void(DevBatch&)>& emit) = 0;
  virtual void flush(OpContext& cx, const std::function<void(DevBatch&)>& emit) = 0;
};
std::unique_ptr<IpcSource> make_ipc_source(OpContext& cx, const SchemaDef& schema, const std::vector<int>& used_cols);

// SortExec (sort_stage.cu): collects its input, emits the sorted (and `fetch`-limited) rows at finish
std::unique_ptr<Stage> make_sort_stage(OpContext& cx, const SchemaDef& in_schema, const PlanNode& node);

// WindowExec (window_stage.cu): partition / order keys and aggregate arguments are input columns, by index; the output is the
// first `n_fwd` input columns ++ one column per window expression (the trailing input columns are dropped)
struct WindowCols { std::vector<int> partition_cols, order_cols; std::vector<std::vector<int>> agg_args; size_t n_fwd = 0; };
std::unique_ptr<Stage> make_window_stage(OpContext& cx, const SchemaDef& in_schema, const PlanNode& node, const WindowCols& cols);

// Hash join (join_stage.cu): the build side is its own op; probe ops attach to its result
struct JoinBuilt;
std::unique_ptr<Stage> make_join_build_stage(OpContext& cx, const SchemaDef& in_schema, const PlanNode& node);
std::unique_ptr<Stage> make_join_probe_stage(OpContext& cx, const SchemaDef& in_schema, const PlanNode& node);
// all `srcs` through one index vector (JOIN_NIL: a NULL row): one gather kernel per 16 columns (join_stage.cu).  A source's
// validity is vbytes (one byte per row), else vbits at bit_offset, else none; may_be_null: the output gets a validity bitmap
struct GatherSrc { DType type; const void* values; const uint8_t* vbits; uint32_t bit_offset; const uint8_t* vbytes; bool may_be_null; };
std::vector<DevColumn> gather_columns(OpContext& cx, const std::vector<GatherSrc>& srcs, const uint32_t* idx, int64_t n);
struct JoinBuildResult { virtual ~JoinBuildResult() {} virtual std::shared_ptr<JoinBuilt> built() const = 0; };
struct JoinProbeAttach { virtual ~JoinProbeAttach() {} virtual void attach(std::shared_ptr<JoinBuilt> b) = 0; };

// SortMergeJoinExec (smj_stage.cu): the op's pushed input is the LEFT side; the right side is the queued output of another,
// finished op (b200q_op_attach_right), taken over by reference at attach
std::unique_ptr<Stage> make_smj_stage(OpContext& cx, const SchemaDef& in_schema, const PlanNode& node);
struct SmjRightAttach {
  virtual ~SmjRightAttach() {}
  virtual bool right_attached() const = 0;
  // `schema`: the right op's output schema; throws ExecError (INVALID_ARG: schema, unsorted; UNSUPPORTED: 2^31 rows or more)
  virtual void attach_right(OpContext& cx, const std::vector<DevBatch>& batches, const SchemaDef& schema) = 0;
};

// a column as the kernels see it (stages.cu)
DevCol dev_col_of(const DevColumn& c);

// ---- batch plumbing shared by the stages (stages.cu) ----------------------------------------------------------------------
// a validity / Boolean bitmap of n rows: whole 32-bit words, as pack_valid_kernel writes them
inline size_t bitmap_bytes(int64_t n) { return (size_t)((n + 31) / 32) * 4; }
// n bytes (one per row, nonzero = set) packed into a new bitmap; every word is written, so the allocation is not zeroed
DevMemP pack_bits(OpContext& cx, const void* bytes, int64_t n);
// contiguous columns with validity as one byte per row: values rows*w + 16 bytes, valid rows + 16 (the 16-byte tail serves the
// kernels' 128-bit loads); valid[c] is null when no row of column c can be NULL
struct ByteCols { int64_t rows = 0; std::vector<DevMemP> values, valid; };
// Arrow-form batches (any offset, bit validity), or ByteCols, copied one after another into one ByteCols; the rows of a part
// without validity read as valid.  concat releases its parts.
ByteCols to_byte_cols(OpContext& cx, const SchemaDef& schema, const std::vector<const DevBatch*>& parts);
ByteCols concat(OpContext& cx, const SchemaDef& schema, std::vector<ByteCols>&& parts);
// n rows of NULL in every column of `schema` (zeroed values and bitmaps)
std::vector<DevColumn> null_columns(OpContext& cx, const SchemaDef& schema, int64_t n);
// after the stream sync: cx.ev0 -> cx.ev1 into gpu_ms, and when `hot` also into the hot_kernel_* metrics over `rows` rows
void add_kernel_time(OpContext& cx, int64_t rows, bool hot);
// whether a column may be passed on without a copy: offset 0 and every buffer owned by the op or kept alive by an owner
// (borrowed caller memory, push_device, is only valid until the batch is released)
inline bool kept_alive(const DevMemP& m) { return !m || m->owned || m->owner; }
inline bool forwardable(const DevColumn& c) { return c.offset == 0 && kept_alive(c.values) && kept_alive(c.validity) && kept_alive(c.offsets); }
// f(window) for consecutive windows of at most `rows` rows of `in` (the same buffers at moved offsets)
template <class F> void for_each_window(const DevBatch& in, int64_t rows, F&& f) {
  for (int64_t r0 = 0; r0 < in.num_rows; r0 += rows) {
    DevBatch part; part.num_rows = std::min(rows, in.num_rows - r0);
    for (auto& c : in.cols) { DevColumn p = c; p.offset = c.offset + r0; part.cols.push_back(p); }
    f(part);
  }
}
// an Arrow-form column (bit validity at its offset) as a gather source
inline GatherSrc gather_src_of(const DevColumn& c, bool nil_possible) {
  return GatherSrc{c.type, (const uint8_t*)c.values->ptr + (size_t)c.offset * c.type.byte_width(), c.validity ? (const uint8_t*)c.validity->ptr : nullptr,
                   (uint32_t)c.offset, nullptr, nil_possible || (bool)c.validity};
}

// helpers of the C ABI layer (capi.cu) shared with exchange.cu
DType type_of_format(const char* arrow_format);
void export_device(DevBatch& db, int device, ArrowDeviceArray* out);
b200q_status fail(int code, const std::string& msg);
b200q_status guarded_call(const std::function<void()>& f);        // exceptions -> status + b200q_last_error()

// state columns of one aggregate in the columnar partial-state layout
struct StateCols { std::vector<FieldDef> fields; std::vector<uint8_t> frozen; };   // frozen: FrozenKind of each field in the Binary agg-buffer column
StateCols state_columns_of(const AggDef& a);

}  // namespace b200q
