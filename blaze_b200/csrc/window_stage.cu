// WindowStage: WindowExecNode (datafusion-ext-plans/src/window_exec.rs, window/*).
//
// The input arrives sorted by (partition spec, order spec).  Partition and order keys and aggregate arguments are columns of
// the stage input, by index: computed ones were appended as trailing columns by the FilterProjectStage below (build_pipeline),
// and the stage drops them from its output.  Output = the first `n_fwd` input columns ++ one column per window expression.
// Every push runs window_flags_kernel once, then one reduce-then-scan per function (kernels_window.cu); the state after the last
// row (key words and every function's scan state) stays on the device for the next push.
#include "kernels_window.cuh"
#include "runtime.h"

namespace b200q {

namespace {

inline size_t bitmap_bytes(int64_t n) { return (size_t)((n + 31) / 32) * 4; }

class WindowStage : public Stage {
  WinKeys keys_{};
  std::vector<WinFn> fns_;
  std::vector<int> fn_out_;                        // aggregates: the window expression each function writes (rank pass: -1)
  int rank_out_[3] = {-1, -1, -1};                 // window expression of row_number / rank / dense_rank (the first one of each kind)
  std::vector<std::vector<int>> rank_dup_;         // later expressions of the same rank-like kind: copies of the first one's column
  std::vector<int> key_cols_;                      // input column of each key of keys_
  std::vector<std::vector<int>> fn_args_;
  size_t n_fwd_;
  std::vector<FieldDef> win_fields_;
  DevMemP carry_;                                  // WinKeyCarry, then one WinState per function
  std::unique_ptr<Stage> fwd_;                     // copies the forwarded columns when they cannot be shared

 public:
  WindowStage(OpContext& cx, const SchemaDef& in, const PlanNode& node, const WindowCols& wc) : n_fwd_(wc.n_fwd) {
    in_schema = in;
    for (size_t i = 0; i < n_fwd_; i++) out_schema.fields.push_back(in.fields[i]);
    for (auto& w : node.window_exprs) { out_schema.fields.push_back(w.field); win_fields_.push_back(w.field); }
    for (size_t i = 0; i < in.fields.size(); i++) used_input_cols.push_back((int)i);
    auto add_key = [&](int col, bool is_order) {
      WinKey& k = keys_.k[keys_.nkeys++];
      k.phys = phys_of(in.fields[(size_t)col].type); k.is_order = is_order;
      key_cols_.push_back(col);
    };
    for (int c : wc.partition_cols) add_key(c, false);
    for (int c : wc.order_cols) add_key(c, true);
    keys_.has_partition = !wc.partition_cols.empty(); keys_.has_order = !wc.order_cols.empty();
    rank_dup_.resize(3);
    bool any_rank = false;
    for (size_t e = 0; e < node.window_exprs.size(); e++) {
      const PlanNode::WindowExprDef& w = node.window_exprs[e];
      if (w.is_rank) {
        if (rank_out_[w.rank_fn] >= 0) rank_dup_[w.rank_fn].push_back((int)e); else rank_out_[w.rank_fn] = (int)e;
        any_rank = true;
        continue;
      }
      WinFn f{};
      const DType& dt = w.agg.data_type;
      const DType at = wc.agg_args[e].empty() ? dt : in.fields[(size_t)wc.agg_args[e][0]].type;      // COUNT without nullable arguments: no argument
      f.out_phys = phys_of(dt); f.nargs = (uint8_t)wc.agg_args[e].size();
      if (w.agg.fn != AGG_COUNT) f.arg_phys = phys_of(at);
      switch (w.agg.fn) {
        case AGG_SUM: f.op = dt.is_decimal() ? WOP_SUM_I128 : dt.id == T_FLOAT64 ? WOP_SUM_F64 : WOP_SUM_I64; break;
        case AGG_AVG: f.op = dt.is_decimal() ? WOP_AVG_DEC : WOP_AVG_F64; break;
        case AGG_COUNT: f.op = WOP_COUNT; break;
        default: {
          const bool mn = w.agg.fn == AGG_MIN;
          f.op = at.is_decimal() ? (mn ? WOP_MIN_I128 : WOP_MAX_I128) : at.is_float() ? (mn ? WOP_MIN_F : WOP_MAX_F) : (mn ? WOP_MIN_I64 : WOP_MAX_I64);
        }
      }
      fns_.push_back(f); fn_out_.push_back((int)e); fn_args_.push_back(wc.agg_args[e]);
    }
    if (any_rank) { WinFn f{}; f.op = WOP_RANK; fns_.push_back(f); fn_out_.push_back(-1); fn_args_.push_back({}); }
    carry_ = DevMem::alloc(sizeof(WinKeyCarry) + fns_.size() * sizeof(WinState), cx.stream, true);
    std::vector<ExprP> fwd_cols;
    for (size_t i = 0; i < n_fwd_; i++) {
      auto e = std::make_shared<Expr>(); e->kind = E_COLUMN; e->col_index = (int)i; e->name = in.fields[i].name; e->type = in.fields[i].type; e->nullable = in.fields[i].nullable;
      fwd_cols.push_back(e);
    }
    SchemaDef fwd_schema; fwd_schema.fields.assign(in.fields.begin(), in.fields.begin() + (long)n_fwd_);
    fwd_ = make_filter_project_stage(cx, in, {}, fwd_cols, fwd_schema);
  }

  void push(OpContext& cx, DevBatch& in, std::vector<DevBatch>& outs) override {
    const int64_t n = in.num_rows;
    if (n == 0) return;
    if (n > 0x7FFFFFFFLL) throw ExecError(B200Q_ERR_UNSUPPORTED, "batches above 2^31-1 rows must be split by the caller");
    WinKeys keys = keys_;
    for (int k = 0; k < keys.nkeys; k++) keys.k[k].col = dev_col_of(in.cols[(size_t)key_cols_[(size_t)k]]);
    DevBatch ob; ob.num_rows = n;
    // forwarded columns: shared when the op owns them at offset 0 (the identity-path rule), copied otherwise
    bool plain = true;
    auto ours = [](const DevMemP& m) { return !m || m->owned || m->owner; };
    for (size_t i = 0; i < n_fwd_; i++) { const DevColumn& c = in.cols[i]; plain = plain && c.offset == 0 && ours(c.values) && ours(c.validity) && ours(c.offsets); }
    if (plain) ob.cols.assign(in.cols.begin(), in.cols.begin() + (long)n_fwd_);
    else {
      // the copy is timed into gpu_ms by the nested stage, but kept out of the hot_kernel_* metrics: those describe this stage's
      // window kernels (and count each input row once)
      std::vector<DevBatch> f;
      const int stage = cx.cur_stage; cx.cur_stage = -1;
      fwd_->push(cx, in, f);
      cx.cur_stage = stage;
      ob.cols = f.at(0).cols;
    }
    std::vector<DevColumn> wcols(win_fields_.size());
    std::vector<DevMemP> valid_bytes(win_fields_.size());
    for (size_t e = 0; e < win_fields_.size(); e++) {
      const DType& t = win_fields_[e].type;
      wcols[e].type = t;
      wcols[e].values = DevMem::alloc((size_t)n * (size_t)t.byte_width() + 16, cx.stream);
    }
    const int64_t ntiles = window_num_tiles(n);
    DevMemP flags = DevMem::alloc((size_t)n + 16, cx.stream);
    DevMemP tsum = DevMem::alloc((size_t)ntiles * sizeof(WinState), cx.stream), tpre = DevMem::alloc((size_t)ntiles * sizeof(WinState), cx.stream);
    WinKeyCarry* kc = (WinKeyCarry*)carry_->ptr;
    WinState* sc = (WinState*)((uint8_t*)carry_->ptr + sizeof(WinKeyCarry));
    B200Q_CUDA(cudaEventRecord(cx.ev0, cx.stream));
    cx.m.launches += launch_window_flags(keys, n, kc, (uint8_t*)flags->ptr, cx.stream);
    for (size_t j = 0; j < fns_.size(); j++) {
      WinFn f = fns_[j];
      for (size_t a = 0; a < fn_args_[j].size(); a++) f.arg[a] = dev_col_of(in.cols[(size_t)fn_args_[j][a]]);
      if (f.op == WOP_RANK) { for (int r = 0; r < 3; r++) f.out[r] = rank_out_[r] >= 0 ? wcols[(size_t)rank_out_[r]].values->ptr : nullptr; }
      else {
        const int e = fn_out_[j];
        f.out[0] = wcols[(size_t)e].values->ptr;
        if (f.op != WOP_COUNT) { valid_bytes[(size_t)e] = DevMem::alloc((size_t)n + 16, cx.stream); f.out_valid = (uint8_t*)valid_bytes[(size_t)e]->ptr; }
      }
      cx.m.launches += launch_window_scan(f, (const uint8_t*)flags->ptr, n, sc + j, (WinState*)tsum->ptr, (WinState*)tpre->ptr, cx.stream);
    }
    B200Q_CUDA(cudaEventRecord(cx.ev1, cx.stream));
    B200Q_CUDA(cudaGetLastError());
    for (int r = 0; r < 3; r++)
      for (int e : rank_dup_[r]) B200Q_CUDA(cudaMemcpyAsync(wcols[(size_t)e].values->ptr, wcols[(size_t)rank_out_[r]].values->ptr, (size_t)n * 4, cudaMemcpyDeviceToDevice, cx.stream));
    for (size_t e = 0; e < win_fields_.size(); e++) {
      if (!valid_bytes[e]) continue;
      wcols[e].validity = DevMem::alloc(bitmap_bytes(n), cx.stream, true);
      cx.m.launches += launch_pack_valid((const uint8_t*)valid_bytes[e]->ptr, (uint32_t*)wcols[e].validity->ptr, n, cx.stream);
    }
    for (auto& c : wcols) ob.cols.push_back(c);
    B200Q_CUDA(cudaStreamSynchronize(cx.stream));
    { float ms = 0; B200Q_CUDA(cudaEventElapsedTime(&ms, cx.ev0, cx.ev1)); cx.m.gpu_ms += ms; if (cx.cur_stage == 0) { cx.m.hot_ms += ms; cx.m.hot_rows += n; cx.m.hot_launches++; } }
    outs.push_back(std::move(ob));
  }

  void finish(OpContext&, std::vector<DevBatch>&) override {}
};

}  // namespace

std::unique_ptr<Stage> make_window_stage(OpContext& cx, const SchemaDef& in_schema, const PlanNode& node, const WindowCols& cols) {
  return std::unique_ptr<Stage>(new WindowStage(cx, in_schema, node, cols));
}

}  // namespace b200q
