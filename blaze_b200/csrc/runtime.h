// Host runtime of the operator pipeline behind the C ABI (include/blaze_b200.h).
//
// An op = a chain of stages compiled from the plan subtree:
//   FilterProjectStage  FilterExec / ProjectExec chain fused into one kernel   (filter_exec.rs, project_exec.rs)
//   AggStage            AggExec with everything below it (Filter/Project) fused into its update kernel (agg_exec.rs)
// Batches between stages stay in HBM.
#pragma once
#include <cuda_runtime.h>

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
// (their release frees stream-ordered memory): the stream is destroyed when the last reference goes away.
struct StreamRef {
  cudaStream_t s = nullptr; int device = 0;
  ~StreamRef();
};
std::shared_ptr<StreamRef> stream_ref_create(int device);
std::shared_ptr<StreamRef> stream_ref_lookup(cudaStream_t s);

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
struct JoinBuildResult { virtual ~JoinBuildResult() {} virtual std::shared_ptr<JoinBuilt> built() const = 0; };
struct JoinProbeAttach { virtual ~JoinProbeAttach() {} virtual void attach(std::shared_ptr<JoinBuilt> b) = 0; };

// a column as the kernels see it (stages.cu)
DevCol dev_col_of(const DevColumn& c);

// helpers of the C ABI layer (capi.cu) shared with exchange.cu
DType type_of_format(const char* arrow_format);
void export_device(DevBatch& db, int device, ArrowDeviceArray* out);
b200q_status fail(int code, const std::string& msg);
b200q_status guarded_call(const std::function<void()>& f);        // exceptions -> status + b200q_last_error()

// state columns of one aggregate in the columnar partial-state layout
struct StateCols { std::vector<FieldDef> fields; };
StateCols state_columns_of(const AggDef& a);

}  // namespace b200q
