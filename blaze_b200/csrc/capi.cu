// C ABI (include/blaze_b200.h): plan -> stage pipeline, Arrow C Data / Device Data import + export,
// host staging (pinned ring) and the error convention.  See the header for the reference interfaces
// each entry point replaces.
#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <mutex>

#include "lz4_frame.h"
#include "parquet_meta.h"
#include "runtime.h"

namespace b200q {

static thread_local std::string g_last_error;

// ---------------------------------------------------------------------------------------------------
// Arrow schema import / export
// ---------------------------------------------------------------------------------------------------
static std::string format_of(const DType& t) {
  switch (t.id) {
    case T_BOOL: return "b"; case T_INT8: return "c"; case T_INT16: return "s"; case T_INT32: return "i"; case T_INT64: return "l";
    case T_FLOAT32: return "f"; case T_FLOAT64: return "g"; case T_DATE32: return "tdD"; case T_TIMESTAMP_US: return "tsu:";
    case T_DECIMAL128: return "d:" + std::to_string(t.precision) + "," + std::to_string(t.scale);
    case T_BINARY: return "z"; case T_UTF8: return "u"; default: return "n";
  }
}
DType type_of_format(const char* f) {
  DType d; std::string s(f ? f : "");
  if (s == "b") d.id = T_BOOL; else if (s == "c") d.id = T_INT8; else if (s == "s") d.id = T_INT16; else if (s == "i") d.id = T_INT32;
  else if (s == "l") d.id = T_INT64; else if (s == "f") d.id = T_FLOAT32; else if (s == "g") d.id = T_FLOAT64; else if (s == "tdD") d.id = T_DATE32;
  else if (s.rfind("tsu:", 0) == 0) d.id = T_TIMESTAMP_US; else if (s == "z") d.id = T_BINARY; else if (s == "u") d.id = T_UTF8; else if (s == "n") d.id = T_NULL;
  else if (s.rfind("d:", 0) == 0) {
    int p = 0, sc = 0, bw = 128; if (sscanf(s.c_str(), "d:%d,%d,%d", &p, &sc, &bw) < 2 || bw != 128) throw PlanError(B200Q_ERR_UNSUPPORTED, "unsupported decimal format " + s);
    d.id = T_DECIMAL128; d.precision = (uint8_t)p; d.scale = (int8_t)sc;
  } else throw PlanError(B200Q_ERR_UNSUPPORTED, "arrow format '" + s + "' is not on the hot path");
  return d;
}

struct SchemaPriv { std::string format, name; std::vector<ArrowSchema> children; std::vector<ArrowSchema*> child_ptrs; };
static void release_schema(ArrowSchema* s) {
  if (!s || !s->release) return;
  auto* p = (SchemaPriv*)s->private_data;
  for (auto& c : p->children) if (c.release) c.release(&c);
  delete p; s->release = nullptr;
}
static void export_field(const std::string& name, const std::string& format, bool nullable, ArrowSchema* out) {
  auto* p = new SchemaPriv(); p->format = format; p->name = name;
  memset(out, 0, sizeof(*out));
  out->format = p->format.c_str(); out->name = p->name.c_str(); out->flags = nullable ? ARROW_FLAG_NULLABLE : 0;
  out->release = release_schema; out->private_data = p;
}
static void export_schema(const SchemaDef& s, ArrowSchema* out) {
  export_field("", "+s", false, out);
  auto* p = (SchemaPriv*)out->private_data;
  p->children.resize(s.fields.size()); p->child_ptrs.resize(s.fields.size());
  for (size_t i = 0; i < s.fields.size(); i++) { export_field(s.fields[i].name, format_of(s.fields[i].type), s.fields[i].nullable, &p->children[i]); p->child_ptrs[i] = &p->children[i]; }
  out->n_children = (int64_t)s.fields.size(); out->children = p->child_ptrs.data();
}

// ---------------------------------------------------------------------------------------------------
// the operator handle
// ---------------------------------------------------------------------------------------------------
struct HostBlock {      // one host allocation holding a whole output batch; shared by its slices
  std::vector<void*> ptrs;
  ~HostBlock() { for (void* p : ptrs) free(p); }
  void* alloc(size_t n) { void* p = malloc(n ? n : 8); if (!p) throw std::bad_alloc(); ptrs.push_back(p); return p; }
};
struct HostColumn { DType type; void* values = nullptr; void* validity = nullptr; void* offsets = nullptr; int64_t null_count = -1; };
struct HostBatch { std::shared_ptr<HostBlock> block; std::vector<HostColumn> cols; int64_t num_rows = 0; int64_t cursor = 0; };

struct PendingRelease { ArrowArray arr; cudaEvent_t ev; };

struct StagingSet {
  struct Col { bool any_null = false; void* values = nullptr; size_t values_cap = 0; uint8_t* validity = nullptr; int32_t* offsets = nullptr; uint8_t* data = nullptr; size_t data_cap = 0, data_len = 0; };
  std::vector<Col> cols;
  int64_t rows = 0;
  cudaEvent_t ev = nullptr;
  bool in_flight = false;
};

}  // namespace b200q

using namespace b200q;

struct b200q_op {
  OpContext cx;
  PlanP plan;
  std::vector<std::unique_ptr<Stage>> stages;
  SchemaDef in_schema, out_schema;
  std::deque<DevBatch> out_queue;
  HostBatch cur_host;           // output batch currently being sliced to the host
  bool has_cur_host = false;
  bool finished = false;
  std::string sticky_error; int sticky_code = 0;
  std::vector<PendingRelease> pending;
  StagingSet staging[2]; int cur_stage_set = 0; bool staging_ready = false;
  cudaEvent_t ev_a = nullptr, ev_b = nullptr;
  std::shared_ptr<StreamRef> stream_ref;
};

namespace b200q {

b200q_status fail(int code, const std::string& msg) { g_last_error = msg; return code; }

template <class F>
static b200q_status guarded(b200q_op* op, F&& f) {
  try {
    if (op && op->sticky_code) return fail(op->sticky_code, op->sticky_error);
    cudaGetLastError();      // drop stale (non-sticky) error state left by other CUDA users of this thread (torch, NCCL): our
                             // launch checks must only see our own launches
    f();
    return B200Q_OK;
  } catch (const PlanError& e) { return fail(e.code, e.what());
  } catch (const ExecError& e) { return fail(e.code, e.what());
  } catch (const CudaError& e) {
    if (op) { op->sticky_code = B200Q_ERR_CUDA; op->sticky_error = e.what(); }
    return fail(B200Q_ERR_CUDA, e.what());
  } catch (const std::exception& e) { return fail(B200Q_ERR_EXECUTION, e.what()); }
}
b200q_status guarded_call(const std::function<void()>& f) { return guarded(nullptr, f); }

// ---- pipeline construction ----------------------------------------------------------------------------
static std::vector<ExprP> identity_cols(const SchemaDef& s) {
  std::vector<ExprP> v;
  for (size_t i = 0; i < s.fields.size(); i++) {
    auto e = std::make_shared<Expr>(); e->kind = E_COLUMN; e->col_index = (int)i; e->name = s.fields[i].name; e->type = s.fields[i].type; e->nullable = s.fields[i].nullable;
    v.push_back(e);
  }
  return v;
}
static bool is_identity(const std::vector<ExprP>& cols, const SchemaDef& s) {
  if (cols.size() != s.fields.size()) return false;
  for (size_t i = 0; i < cols.size(); i++) if (cols[i]->kind != E_COLUMN || cols[i]->col_index != (int)i) return false;
  return true;
}

static bool fusable_partial_final(const PlanNode& p, const PlanNode& f) {
  static const bool off = getenv("B200Q_NO_AGG_FUSION") != nullptr;             // keeps the two-stage form reachable for tests
  if (off || p.kind != N_AGG || f.kind != N_AGG) return false;
  if (p.need_partial_merge || p.need_final_merge || !f.need_final_merge) return false;
  if (p.aggs.size() != f.aggs.size() || p.group_exprs.size() != f.group_exprs.size()) return false;
  for (size_t k = 0; k < f.group_exprs.size(); k++) {                            // the Final groups by the Partial's key columns, in order
    const ExprP& g = f.group_exprs[k];
    if (g->kind != E_COLUMN || g->col_index != (int)k || !(g->type == p.group_exprs[k]->type)) return false;
  }
  for (size_t a = 0; a < f.aggs.size(); a++) {
    if (p.aggs[a].mode != MODE_PARTIAL || f.aggs[a].mode != MODE_FINAL) return false;
    if (p.aggs[a].fn != f.aggs[a].fn || !(p.aggs[a].data_type == f.aggs[a].data_type)) return false;
  }
  return true;
}

static void build_pipeline(b200q_op* op) {
  std::vector<PlanNode*> chain;
  for (PlanNode* n = op->plan.get(); n; n = n->input.get()) chain.push_back(n);
  std::reverse(chain.begin(), chain.end());
  if (chain.empty() || chain[0]->kind != N_LEAF) throw PlanError(B200Q_ERR_INVALID_PLAN, "plan has no leaf");
  if (chain[0]->leaf_kind == "ParquetScan")
    for (auto& f : chain[0]->schema.fields)
      if (f.type.is_varlen()) throw PlanError(B200Q_ERR_UNSUPPORTED, "ParquetScanExec: column " + f.name + " is " + f.type.str() + "; BYTE_ARRAY decode is not on the GPU path");
  op->in_schema = chain[0]->schema;
  SchemaDef stage_in = chain[0]->schema;
  std::vector<ExprP> cur_cols = identity_cols(stage_in), filters;
  const PlanNode* last = chain[0];
  bool pending_tail = chain.size() == 1;
  // the aggregate chain[i] over the columns of each set (one set: `cur_cols`); on return chain[i] is the last node the stage consumed
  auto push_agg = [&](size_t& i, const std::vector<std::vector<ExprP>>& set_cols) {
    PlanNode* n = chain[i];
    std::vector<AggSetExprs> sets;
    for (auto& cols : set_cols) {
      AggSetExprs sx;
      for (auto& g : n->group_exprs) sx.group_exprs.push_back(substitute(g, cols));
      for (auto& a : n->aggs) { std::vector<ExprP> v; if (a.mode == MODE_PARTIAL) for (auto& e : a.args) v.push_back(substitute(e, cols)); sx.agg_args.push_back(v); }
      sets.push_back(std::move(sx));
    }
    // AggExec(Final) directly above AggExec(Partial) in the same op (Spark plans this when the child is already partitioned on the grouping keys):
    // the Partial stage's table holds one entry per group, so a Final stage would only re-insert unique keys into a second table.  One stage
    // accumulates from the raw inputs and emits the Final columns (AVG division, result types) straight from its table.
    PlanNode fused;
    const PlanNode* agg_node = n;
    last = n;
    if (i + 1 < chain.size() && fusable_partial_final(*n, *chain[i + 1])) {
      fused = *n; fused.need_final_merge = true; fused.schema = chain[i + 1]->schema;
      agg_node = &fused; last = chain[i + 1]; i++;
    }
    if (sets.size() > 1) op->stages.push_back(make_agg_stage(op->cx, stage_in, filters, *agg_node, sets[0].group_exprs, sets[0].agg_args, sets));
    else op->stages.push_back(make_agg_stage(op->cx, stage_in, filters, *agg_node, sets[0].group_exprs, sets[0].agg_args));
    stage_in = op->stages.back()->out_schema;
    cur_cols = identity_cols(stage_in); filters.clear(); pending_tail = false;
  };
  for (size_t i = 1; i < chain.size(); i++) {
    PlanNode* n = chain[i];
    last = n;
    if (n->kind == N_FILTER) { for (auto& p : n->predicates) filters.push_back(substitute(p, cur_cols)); pending_tail = true; }
    else if (n->kind == N_PROJECT) { std::vector<ExprP> nc; for (auto& e : n->proj_exprs) nc.push_back(substitute(e, cur_cols)); cur_cols = nc; pending_tail = true; }
    else if (n->kind == N_AGG) {
      if (n->need_partial_merge && !is_identity(cur_cols, stage_in)) throw PlanError(B200Q_ERR_UNSUPPORTED, "Projection fused below a merge-mode aggregate");
      push_agg(i, {cur_cols});
    } else if (n->kind == N_EXPAND) {
      std::vector<std::vector<ExprP>> sets;
      for (auto& proj : n->expand_projections) { std::vector<ExprP> v; for (auto& e : proj) v.push_back(substitute(e, cur_cols)); sets.push_back(v); }
      if (sets.size() == 1) { cur_cols = sets[0]; pending_tail = true; continue; }       // one projection: a ProjectExec
      // Expand -> [Project]* -> AggExec(Partial): the sets are fused into the aggregate (each input row is read once and inserted once per
      // set; filters below the Expand are shared by all sets).  Anything else above the Expand sees it materialised.
      std::vector<std::vector<ExprP>> composed = sets;
      size_t j = i + 1;
      for (; j < chain.size() && chain[j]->kind == N_PROJECT; j++)
        for (auto& cols : composed) { std::vector<ExprP> nc; for (auto& e : chain[j]->proj_exprs) nc.push_back(substitute(e, cols)); cols = nc; }
      bool fuse = sets.size() > 1 && j < chain.size() && chain[j]->kind == N_AGG && !chain[j]->need_partial_merge;
      if (fuse) for (auto& a : chain[j]->aggs) fuse = fuse && a.mode == MODE_PARTIAL;
      if (fuse) { i = j; push_agg(i, composed); continue; }
      op->stages.push_back(make_expand_stage(op->cx, stage_in, filters, sets, n->schema));
      stage_in = op->stages.back()->out_schema; cur_cols = identity_cols(stage_in); filters.clear(); pending_tail = false;
    } else if (n->kind == N_SORT) {
      if (pending_tail) {
        op->stages.push_back(make_filter_project_stage(op->cx, stage_in, filters, cur_cols, n->input->schema));
        stage_in = op->stages.back()->out_schema; cur_cols = identity_cols(stage_in); filters.clear(); pending_tail = false;
      }
      op->stages.push_back(make_sort_stage(op->cx, stage_in, *n));
      stage_in = op->stages.back()->out_schema; cur_cols = identity_cols(stage_in);
    } else if (n->kind == N_WINDOW) {
      // a WindowExec without a limit directly on one with a limit runs as ONE window: the parent's expressions, the child's
      // limit, output_window_cols = true, over the child's input (window_exec.rs:166-185)
      PlanNode combined;
      const PlanNode* w = n;
      if (n->window_has_limit && i + 1 < chain.size() && chain[i + 1]->kind == N_WINDOW && !chain[i + 1]->window_has_limit) {
        if (n->output_window_cols) throw PlanError(B200Q_ERR_UNSUPPORTED, "WindowExec over a group-limited WindowExec that outputs its window column");
        // the combined window outputs its window columns whatever the parent declares: a parent without them would disagree with it
        if (!chain[i + 1]->output_window_cols) throw PlanError(B200Q_ERR_UNSUPPORTED, "WindowExec with output_window_cols = false over a group-limited WindowExec");
        combined = *chain[i + 1]; combined.window_has_limit = true; combined.window_limit = n->window_limit; combined.output_window_cols = true;
        if (combined.window_exprs.size() != 1) throw PlanError(B200Q_ERR_INVALID_PLAN, "WindowExec: a group limit needs exactly one window expression, got " + std::to_string(combined.window_exprs.size()));
        if (!combined.window_exprs[0].is_rank) throw PlanError(B200Q_ERR_UNSUPPORTED, "WindowExec: a group limit over an aggregate window column is not on the GPU path (rank-like functions are)");
        w = &combined; i++; last = chain[i];
      }
      // keys and arguments that are not input columns are computed by a FilterProjectStage below, as trailing columns
      const size_t n_fwd = w->input->schema.fields.size();
      std::vector<ExprP> extra;
      SchemaDef win_in = w->input->schema;
      auto col_of = [&](ExprP e) {
        while ((e->kind == E_TRY_CAST || e->kind == E_CAST) && e->children[0]->type == e->type) e = e->children[0];   // create_agg's TryCast to the type it has
        if (e->kind == E_COLUMN) return e->col_index;
        extra.push_back(e);
        win_in.fields.push_back(FieldDef{"#window_arg" + std::to_string(extra.size() - 1), e->type, e->nullable});
        return (int)(n_fwd + extra.size() - 1);
      };
      WindowCols wc; wc.n_fwd = n_fwd;
      for (auto& e : w->window_partition) wc.partition_cols.push_back(col_of(e));
      for (auto& se : w->window_order) wc.order_cols.push_back(col_of(se.expr));
      for (auto& we : w->window_exprs) { std::vector<int> v; if (!we.is_rank) for (auto& a : we.agg.args) v.push_back(col_of(a)); wc.agg_args.push_back(v); }
      if (pending_tail || !extra.empty()) {
        std::vector<ExprP> outs = cur_cols;
        for (auto& e : extra) outs.push_back(substitute(e, cur_cols));
        op->stages.push_back(make_filter_project_stage(op->cx, stage_in, filters, outs, win_in));
        filters.clear(); pending_tail = false;
      }
      op->stages.push_back(make_window_stage(op->cx, win_in, *w, wc));
      stage_in = op->stages.back()->out_schema; cur_cols = identity_cols(stage_in);
      if (w->window_has_limit) {
        // WindowGroupLimit: keep the rows whose window column is <= (int32)k (window_exec.rs:227-235); the window column is dropped
        // unless output_window_cols.  A pending filter, fused into whatever runs next.
        auto col = cur_cols[n_fwd];
        auto lit = std::make_shared<Expr>(); lit->kind = E_LITERAL; lit->type.id = T_INT32; lit->nullable = false;
        lit->lit_lo = (uint64_t)(int64_t)(int32_t)w->window_limit;
        auto le = std::make_shared<Expr>(); le->kind = E_BINARY; le->op = OP_LE; le->type.id = T_BOOL; le->nullable = col->nullable; le->children = {col, lit};
        filters.push_back(le);
        if (!w->output_window_cols) cur_cols.resize(n_fwd);
        pending_tail = true;
      }
    } else if (n->kind == N_JOIN_BUILD || n->kind == N_JOIN) {
      if (pending_tail) {                               // Filter / Project chain below the join side: its own fused stage
        op->stages.push_back(make_filter_project_stage(op->cx, stage_in, filters, cur_cols, n->input->schema));
        stage_in = op->stages.back()->out_schema; cur_cols = identity_cols(stage_in); filters.clear(); pending_tail = false;
      }
      if (n->kind == N_JOIN_BUILD) {
        if (i + 1 != chain.size()) throw PlanError(B200Q_ERR_UNSUPPORTED, "BroadcastJoinBuildHashMapExec below another operator: build the map side with its own op and attach it (b200q_op_attach_build)");
        op->stages.push_back(make_join_build_stage(op->cx, stage_in, *n));
      } else {
        op->stages.push_back(make_join_probe_stage(op->cx, stage_in, *n));
        stage_in = op->stages.back()->out_schema; cur_cols = identity_cols(stage_in);
      }
    } else if (n->kind == N_SHUFFLE_WRITER) {
      if (i + 1 != chain.size()) throw PlanError(B200Q_ERR_UNSUPPORTED, "ShuffleWriterExec below another operator");
      if (pending_tail) {                               // Filter / Project chain below the writer: its own fused stage
        op->stages.push_back(make_filter_project_stage(op->cx, stage_in, filters, cur_cols, n->input->schema));
        stage_in = op->stages.back()->out_schema; cur_cols = identity_cols(stage_in); filters.clear(); pending_tail = false;
      }
      op->stages.push_back(make_shuffle_write_stage(op->cx, stage_in, *n));
    } else throw PlanError(B200Q_ERR_INVALID_PLAN, "leaf in the middle of the plan");
  }
  if (pending_tail) {
    SchemaDef out = last->schema;
    op->stages.push_back(make_filter_project_stage(op->cx, stage_in, filters, cur_cols, out));
  }
  op->out_schema = op->stages.back()->out_schema;
}

// ---- host -> device import -----------------------------------------------------------------------------
static void copy_bits(uint8_t* dst, int64_t dst_off, const uint8_t* src, int64_t src_off, int64_t n) {
  // generic bit copy (dst bits beyond the range are preserved); byte-aligned fast path
  if (n <= 0) return;
  if ((dst_off & 7) == 0 && (src_off & 7) == 0) {
    memcpy(dst + dst_off / 8, src + src_off / 8, (size_t)(n / 8));
    for (int64_t i = n & ~7LL; i < n; i++) { const int b = (src[(src_off + i) >> 3] >> ((src_off + i) & 7)) & 1; uint8_t& d = dst[(dst_off + i) >> 3]; d = (uint8_t)((d & ~(1u << ((dst_off + i) & 7))) | (b << ((dst_off + i) & 7))); }
    return;
  }
  for (int64_t i = 0; i < n; i++) { const int b = (src[(src_off + i) >> 3] >> ((src_off + i) & 7)) & 1; uint8_t& d = dst[(dst_off + i) >> 3]; d = (uint8_t)((d & ~(1u << ((dst_off + i) & 7))) | (b << ((dst_off + i) & 7))); }
}
static void set_bits(uint8_t* dst, int64_t dst_off, int64_t n) {
  while (n > 0 && (dst_off & 7)) { dst[dst_off >> 3] |= (uint8_t)(1u << (dst_off & 7)); dst_off++; n--; }
  if (n >= 8) { memset(dst + dst_off / 8, 0xFF, (size_t)(n / 8)); dst_off += n & ~7LL; n &= 7; }
  for (; n > 0; n--, dst_off++) dst[dst_off >> 3] |= (uint8_t)(1u << (dst_off & 7));
}

static void validate_host_batch(b200q_op* op, const ArrowArray* batch) {
  if (!batch || !batch->release) throw ExecError(B200Q_ERR_INVALID_ARG, "push: released or null ArrowArray");
  if (batch->n_children != (int64_t)op->in_schema.fields.size())
    throw ExecError(B200Q_ERR_INVALID_ARG, "push: batch has " + std::to_string(batch->n_children) + " columns, the plan leaf declares " + std::to_string(op->in_schema.fields.size()));
  for (int64_t i = 0; i < batch->n_children; i++) {
    const ArrowArray* c = batch->children[i];
    if (!c) throw ExecError(B200Q_ERR_INVALID_ARG, "push: null child array");
    if (c->length + c->offset < batch->length + batch->offset) throw ExecError(B200Q_ERR_INVALID_ARG, "push: child array shorter than the struct");
    if (c->dictionary) throw ExecError(B200Q_ERR_UNSUPPORTED, "push: dictionary-encoded columns are not on the hot path");
    // the import paths dereference buffers[1] (and buffers[2] of Binary columns): a malformed / foreign batch must not crash the host process
    const DType& t = op->in_schema.fields[(size_t)i].type;
    if (t.id == T_NULL || batch->length == 0) continue;
    const int need = t.is_varlen() ? 3 : 2;
    if (c->n_buffers < need || !c->buffers) throw ExecError(B200Q_ERR_INVALID_ARG, "push: column " + std::to_string(i) + " has " + std::to_string(c->n_buffers) + " buffers, its type needs " + std::to_string(need));
    if (!c->buffers[1]) throw ExecError(B200Q_ERR_INVALID_ARG, "push: column " + std::to_string(i) + " has a null " + (t.is_varlen() ? "offsets" : "values") + " buffer");
    if (t.is_varlen() && !c->buffers[2] && ((const int32_t*)c->buffers[1])[c->offset + batch->offset + batch->length] != ((const int32_t*)c->buffers[1])[c->offset + batch->offset])
      throw ExecError(B200Q_ERR_INVALID_ARG, "push: " + t.str() + " column " + std::to_string(i) + " has a null data buffer");
  }
}

static void poll_pending(b200q_op* op, bool wait) {
  for (size_t i = 0; i < op->pending.size();) {
    PendingRelease& p = op->pending[i];
    cudaError_t q = wait ? cudaEventSynchronize(p.ev) : cudaEventQuery(p.ev);
    if (q == cudaSuccess || q != cudaErrorNotReady) {
      if (p.arr.release) p.arr.release(&p.arr);
      cudaEventDestroy(p.ev);
      op->pending.erase(op->pending.begin() + i);
    } else i++;
  }
}

// direct path: each used column is copied straight from the caller's buffers
static DevBatch import_direct(b200q_op* op, const ArrowArray* batch, const std::vector<int>& used) {
  OpContext& cx = op->cx;
  DevBatch db; db.num_rows = batch->length; db.cols.resize(op->in_schema.fields.size());
  for (size_t i = 0; i < db.cols.size(); i++) db.cols[i].type = op->in_schema.fields[i].type;
  for (int ci : used) {
    const ArrowArray* c = batch->children[ci];
    DevColumn& dc = db.cols[ci];
    const int64_t off = c->offset + batch->offset, len = batch->length;
    const int64_t a0 = off & ~7LL;                    // align down to a byte of the bitmaps
    dc.offset = off - a0;
    const int64_t cnt = dc.offset + len;
    const uint8_t* validity = c->n_buffers > 0 ? (const uint8_t*)c->buffers[0] : nullptr;
    if (validity && c->null_count != 0) {
      const size_t nb = (size_t)((cnt + 7) / 8);
      dc.validity = DevMem::alloc(nb + 4, cx.stream);
      B200Q_CUDA(cudaMemcpyAsync(dc.validity->ptr, validity + a0 / 8, nb, cudaMemcpyHostToDevice, cx.stream)); cx.m.h2d_bytes += (int64_t)nb;
    }
    if (dc.type.is_varlen()) {
      if (c->n_buffers < 3) throw ExecError(B200Q_ERR_INVALID_ARG, dc.type.str() + " column needs 3 buffers");
      const int32_t* offs = (const int32_t*)c->buffers[1]; const uint8_t* data = (const uint8_t*)c->buffers[2];
      const int32_t first = offs[a0], end = offs[off + len];
      dc.offsets = DevMem::alloc((size_t)(cnt + 1) * 4, cx.stream);
      // only [first, end) of the data is copied: the device offsets are rebased to start at 0, so every imported column indexes its
      // own allocation (columns may then be shared with the output and exported as they are)
      if (first == 0) B200Q_CUDA(cudaMemcpyAsync(dc.offsets->ptr, offs + a0, (size_t)(cnt + 1) * 4, cudaMemcpyHostToDevice, cx.stream));
      else {
        std::vector<int32_t> rebased(offs + a0, offs + a0 + cnt + 1);
        for (auto& o : rebased) o -= first;
        // a pageable source: the call returns once `rebased` has been staged, so it may go out of scope
        B200Q_CUDA(cudaMemcpyAsync(dc.offsets->ptr, rebased.data(), (size_t)(cnt + 1) * 4, cudaMemcpyHostToDevice, cx.stream));
      }
      dc.values = DevMem::alloc((size_t)(end - first), cx.stream);
      if (end > first) B200Q_CUDA(cudaMemcpyAsync(dc.values->ptr, data + first, (size_t)(end - first), cudaMemcpyHostToDevice, cx.stream));
      cx.m.h2d_bytes += (int64_t)(cnt + 1) * 4 + (end - first);
    } else if (dc.type.id == T_BOOL) {
      const size_t nb = (size_t)((cnt + 7) / 8);
      dc.values = DevMem::alloc(nb + 4, cx.stream);
      B200Q_CUDA(cudaMemcpyAsync(dc.values->ptr, (const uint8_t*)c->buffers[1] + a0 / 8, nb, cudaMemcpyHostToDevice, cx.stream)); cx.m.h2d_bytes += (int64_t)nb;
    } else if (dc.type.id != T_NULL) {
      const size_t w = (size_t)dc.type.byte_width();
      dc.values = DevMem::alloc((size_t)cnt * w, cx.stream);
      B200Q_CUDA(cudaMemcpyAsync(dc.values->ptr, (const uint8_t*)c->buffers[1] + (size_t)a0 * w, (size_t)cnt * w, cudaMemcpyHostToDevice, cx.stream)); cx.m.h2d_bytes += (int64_t)(cnt * w);
    }
  }
  return db;
}

// staging path: small host batches are appended to a pinned buffer set, flushed as one H2D + one launch
static void staging_init(b200q_op* op, const std::vector<int>& used) {
  const int64_t cap = op->cx.conf.staging_rows;
  for (int s = 0; s < 2; s++) {
    StagingSet& st = op->staging[s];
    st.cols.resize(op->in_schema.fields.size());
    B200Q_CUDA(cudaEventCreateWithFlags(&st.ev, cudaEventDisableTiming));
    for (int ci : used) {
      const DType& t = op->in_schema.fields[ci].type; StagingSet::Col& c = st.cols[ci];
      if (t.is_varlen()) {
        B200Q_CUDA(cudaMallocHost((void**)&c.offsets, (size_t)(cap + 1) * 4)); c.offsets[0] = 0;
        c.data_cap = (size_t)cap * 32; B200Q_CUDA(cudaMallocHost((void**)&c.data, c.data_cap));
      } else if (t.id == T_BOOL) { c.values_cap = (size_t)(cap + 7) / 8 + 8; B200Q_CUDA(cudaMallocHost(&c.values, c.values_cap)); memset(c.values, 0, c.values_cap); }
      else if (t.id != T_NULL) { c.values_cap = (size_t)cap * t.byte_width(); B200Q_CUDA(cudaMallocHost(&c.values, c.values_cap)); }
      if (op->in_schema.fields[ci].nullable) { B200Q_CUDA(cudaMallocHost((void**)&c.validity, (size_t)(cap + 7) / 8 + 8)); memset(c.validity, 0, (size_t)(cap + 7) / 8 + 8); }
    }
  }
  op->staging_ready = true;
}
static void staging_free(b200q_op* op) {
  for (int s = 0; s < 2; s++) {
    for (auto& c : op->staging[s].cols) { if (c.values) cudaFreeHost(c.values); if (c.validity) cudaFreeHost(c.validity); if (c.offsets) cudaFreeHost(c.offsets); if (c.data) cudaFreeHost(c.data); }
    if (op->staging[s].ev) cudaEventDestroy(op->staging[s].ev);
    op->staging[s].cols.clear();
  }
}

static void run_stages(b200q_op* op, DevBatch& b, size_t from);

static void staging_flush(b200q_op* op) {
  StagingSet& st = op->staging[op->cur_stage_set];
  if (st.rows == 0) return;
  OpContext& cx = op->cx;
  const std::vector<int>& used = op->stages[0]->used_input_cols;
  DevBatch db; db.num_rows = st.rows; db.cols.resize(op->in_schema.fields.size());
  for (size_t i = 0; i < db.cols.size(); i++) db.cols[i].type = op->in_schema.fields[i].type;
  for (int ci : used) {
    StagingSet::Col& c = st.cols[ci]; DevColumn& dc = db.cols[ci];
    const int64_t n = st.rows;
    if (c.validity && c.any_null) { const size_t nb = (size_t)(n + 7) / 8; dc.validity = DevMem::alloc(nb + 4, cx.stream); B200Q_CUDA(cudaMemcpyAsync(dc.validity->ptr, c.validity, nb, cudaMemcpyHostToDevice, cx.stream)); cx.m.h2d_bytes += (int64_t)nb; }
    if (dc.type.is_varlen()) {
      dc.offsets = DevMem::alloc((size_t)(n + 1) * 4, cx.stream); B200Q_CUDA(cudaMemcpyAsync(dc.offsets->ptr, c.offsets, (size_t)(n + 1) * 4, cudaMemcpyHostToDevice, cx.stream));
      dc.values = DevMem::alloc(c.data_len, cx.stream); if (c.data_len) B200Q_CUDA(cudaMemcpyAsync(dc.values->ptr, c.data, c.data_len, cudaMemcpyHostToDevice, cx.stream));
      cx.m.h2d_bytes += (int64_t)(n + 1) * 4 + (int64_t)c.data_len;
    } else if (dc.type.id == T_BOOL) { const size_t nb = (size_t)(n + 7) / 8; dc.values = DevMem::alloc(nb + 4, cx.stream); B200Q_CUDA(cudaMemcpyAsync(dc.values->ptr, c.values, nb, cudaMemcpyHostToDevice, cx.stream)); cx.m.h2d_bytes += (int64_t)nb; }
    else if (dc.type.id != T_NULL) { const size_t nb = (size_t)n * dc.type.byte_width(); dc.values = DevMem::alloc(nb, cx.stream); B200Q_CUDA(cudaMemcpyAsync(dc.values->ptr, c.values, nb, cudaMemcpyHostToDevice, cx.stream)); cx.m.h2d_bytes += (int64_t)nb; }
  }
  B200Q_CUDA(cudaEventRecord(st.ev, cx.stream)); st.in_flight = true;
  // switch to the other set; wait until its previous H2D has drained before it is overwritten
  op->cur_stage_set ^= 1;
  StagingSet& nx = op->staging[op->cur_stage_set];
  if (nx.in_flight) { B200Q_CUDA(cudaEventSynchronize(nx.ev)); nx.in_flight = false; }
  nx.rows = 0;
  for (auto& c : nx.cols) { c.data_len = 0; c.any_null = false; if (c.validity) memset(c.validity, 0, (size_t)(cx.conf.staging_rows + 7) / 8 + 8); if (c.values && c.values_cap < (size_t)cx.conf.staging_rows) memset(c.values, 0, c.values_cap); }
  run_stages(op, db, 0);
}

static void staging_append(b200q_op* op, const ArrowArray* batch) {
  const std::vector<int>& used = op->stages[0]->used_input_cols;
  if (!op->staging_ready) staging_init(op, used);
  int64_t done = 0;
  while (done < batch->length) {
    StagingSet& st = op->staging[op->cur_stage_set];
    const int64_t room = op->cx.conf.staging_rows - st.rows;
    if (room == 0) { staging_flush(op); continue; }
    const int64_t take = std::min(room, batch->length - done);
    bool need_flush = false;
    for (int ci : used) {
      const ArrowArray* c = batch->children[ci]; StagingSet::Col& sc = st.cols[ci]; const DType& t = op->in_schema.fields[ci].type;
      const int64_t off = c->offset + batch->offset + done;
      const uint8_t* validity = c->n_buffers > 0 ? (const uint8_t*)c->buffers[0] : nullptr;
      if (sc.validity) { if (validity && c->null_count != 0) { copy_bits(sc.validity, st.rows, validity, off, take); sc.any_null = true; } else set_bits(sc.validity, st.rows, take); }
      if (t.is_varlen()) {
        const int32_t* offs = (const int32_t*)c->buffers[1]; const uint8_t* data = (const uint8_t*)c->buffers[2];
        const size_t nbytes = (size_t)(offs[off + take] - offs[off]);
        if (sc.data_len + nbytes > sc.data_cap) {
          if (st.rows > 0) { need_flush = true; break; }
          uint8_t* nd; B200Q_CUDA(cudaMallocHost((void**)&nd, (sc.data_len + nbytes) * 2)); memcpy(nd, sc.data, sc.data_len); cudaFreeHost(sc.data); sc.data = nd; sc.data_cap = (sc.data_len + nbytes) * 2;
        }
        memcpy(sc.data + sc.data_len, data + offs[off], nbytes);
        const int32_t rebase = (int32_t)sc.data_len - offs[off];
        for (int64_t i = 0; i < take; i++) sc.offsets[st.rows + i + 1] = offs[off + i + 1] + rebase;
        sc.data_len += nbytes;
      } else if (t.id == T_BOOL) copy_bits((uint8_t*)sc.values, st.rows, (const uint8_t*)c->buffers[1], off, take);
      else if (t.id != T_NULL) { const size_t w = (size_t)t.byte_width(); memcpy((uint8_t*)sc.values + (size_t)st.rows * w, (const uint8_t*)c->buffers[1] + (size_t)off * w, (size_t)take * w); }
    }
    if (need_flush) { staging_flush(op); continue; }
    st.rows += take; done += take;
  }
}

// ---- stage driver ----------------------------------------------------------------------------------------
static void run_stages(b200q_op* op, DevBatch& b, size_t from) {
  std::vector<DevBatch> outs;
  op->cx.cur_stage = (int)from;
  op->stages[from]->push(op->cx, b, outs);
  for (auto& o : outs) {
    if (from + 1 < op->stages.size()) run_stages(op, o, from + 1);
    else { op->cx.m.output_rows += o.num_rows; op->out_queue.push_back(std::move(o)); }
  }
}

// ---- device -> host export ---------------------------------------------------------------------------------
static HostBatch to_host(b200q_op* op, DevBatch& db) {
  OpContext& cx = op->cx;
  HostBatch hb; hb.block = std::make_shared<HostBlock>(); hb.num_rows = db.num_rows;
  const int64_t n = db.num_rows;
  for (auto& dc : db.cols) {
    HostColumn hc; hc.type = dc.type;
    if (dc.offset != 0) throw ExecError(B200Q_ERR_EXECUTION, "internal: output column with non-zero offset");
    auto d2h = [&](const void* src, size_t bytes) { void* p = hb.block->alloc(bytes + 8); if (bytes) B200Q_CUDA(cudaMemcpyAsync(p, src, bytes, cudaMemcpyDeviceToHost, cx.stream)); cx.m.d2h_bytes += (int64_t)bytes; return p; };
    if (dc.validity) hc.validity = d2h(dc.validity->ptr, (size_t)(n + 7) / 8);
    if (dc.type.is_varlen()) {
      hc.offsets = d2h(dc.offsets->ptr, (size_t)(n + 1) * 4);
      B200Q_CUDA(cudaStreamSynchronize(cx.stream));
      int32_t* ho = (int32_t*)hc.offsets;
      const int32_t first = ho[0];                          // only the bytes the rows reference; the host copy starts at 0
      hc.values = d2h((const uint8_t*)dc.values->ptr + first, (size_t)(ho[n] - first));
      if (first) for (int64_t i = 0; i <= n; i++) ho[i] -= first;
    } else if (dc.type.id == T_BOOL) hc.values = d2h(dc.values->ptr, (size_t)(n + 7) / 8);
    else if (dc.type.id != T_NULL) hc.values = d2h(dc.values->ptr, (size_t)n * dc.type.byte_width());
    hb.cols.push_back(hc);
  }
  B200Q_CUDA(cudaStreamSynchronize(cx.stream));
  return hb;
}

struct ArrayPriv {
  std::shared_ptr<HostBlock> block;        // host export
  std::vector<DevMemP> dev;                // device export
  std::vector<const void*> buffers;
  std::vector<ArrowArray> children; std::vector<ArrowArray*> child_ptrs;
};
static void release_array(ArrowArray* a) {
  if (!a || !a->release) return;
  auto* p = (ArrayPriv*)a->private_data;
  for (auto& c : p->children) if (c.release) c.release(&c);
  delete p; a->release = nullptr;
}
static int64_t count_nulls(const uint8_t* bits, int64_t off, int64_t n) {
  int64_t set = 0;
  for (int64_t i = 0; i < n; i++) set += (bits[(off + i) >> 3] >> ((off + i) & 7)) & 1;
  return n - set;
}
static void export_host_slice(const HostBatch& hb, int64_t off, int64_t len, ArrowArray* out) {
  auto* top = new ArrayPriv(); top->block = hb.block;
  memset(out, 0, sizeof(*out));
  out->length = len; out->null_count = 0; out->offset = 0; out->n_buffers = 1;
  top->buffers.push_back(nullptr); out->buffers = top->buffers.data();
  top->children.resize(hb.cols.size()); top->child_ptrs.resize(hb.cols.size());
  for (size_t i = 0; i < hb.cols.size(); i++) {
    const HostColumn& hc = hb.cols[i];
    auto* cp = new ArrayPriv(); cp->block = hb.block;
    ArrowArray& c = top->children[i]; memset(&c, 0, sizeof(c));
    c.length = len; c.offset = off;
    c.null_count = hc.validity ? count_nulls((const uint8_t*)hc.validity, off, len) : 0;
    if (hc.type.id == T_NULL) { c.null_count = len; c.n_buffers = 0; }
    else if (hc.type.is_varlen()) { cp->buffers = {hc.validity, hc.offsets, hc.values}; c.n_buffers = 3; }
    else { cp->buffers = {hc.validity, hc.values}; c.n_buffers = 2; }
    c.buffers = cp->buffers.data(); c.release = release_array; c.private_data = cp;
    top->child_ptrs[i] = &c;
  }
  out->n_children = (int64_t)hb.cols.size(); out->children = top->child_ptrs.data();
  out->release = release_array; out->private_data = top;
}
void export_device(DevBatch& db, int device, ArrowDeviceArray* out) {
  auto* top = new ArrayPriv();
  memset(out, 0, sizeof(*out));
  ArrowArray& a = out->array;
  a.length = db.num_rows; a.n_buffers = 1; top->buffers.push_back(nullptr); a.buffers = top->buffers.data();
  top->children.resize(db.cols.size()); top->child_ptrs.resize(db.cols.size());
  for (size_t i = 0; i < db.cols.size(); i++) {
    DevColumn& dc = db.cols[i];
    auto* cp = new ArrayPriv();
    ArrowArray& c = top->children[i]; memset(&c, 0, sizeof(c));
    c.length = db.num_rows; c.offset = dc.offset; c.null_count = dc.validity ? -1 : 0;
    const void* v = dc.validity ? dc.validity->ptr : nullptr;
    if (dc.validity) cp->dev.push_back(dc.validity);
    if (dc.values) cp->dev.push_back(dc.values);
    if (dc.offsets) cp->dev.push_back(dc.offsets);
    if (dc.type.id == T_NULL) { c.n_buffers = 0; c.null_count = db.num_rows; }
    else if (dc.type.is_varlen()) { cp->buffers = {v, dc.offsets->ptr, dc.values->ptr}; c.n_buffers = 3; }
    else { cp->buffers = {v, dc.values ? dc.values->ptr : nullptr}; c.n_buffers = 2; }
    c.buffers = cp->buffers.data(); c.release = release_array; c.private_data = cp;
    top->child_ptrs[i] = &c;
  }
  a.n_children = (int64_t)db.cols.size(); a.children = top->child_ptrs.data();
  a.release = release_array; a.private_data = top;
  out->device_id = device; out->device_type = ARROW_DEVICE_CUDA; out->sync_event = nullptr;
}

static void conf_defaults(b200q_conf* c) {
  memset(c, 0, sizeof(*c));
  c->struct_size = sizeof(b200q_conf);
  c->batch_size = 10000;                               // commons/src/lib.rs:74-77
  c->suggested_batch_mem_size = 8388608;               // lib.rs:79-82
  c->partial_agg_skipping_enable = 1;
  c->partial_agg_skipping_ratio = 0.999;               // agg_ctx.rs:177
  c->partial_agg_skipping_min_rows = 20000;            // agg_ctx.rs:178
  c->staging_rows = 1 << 20;
  c->agg_initial_groups = 1 << 19;
  c->max_launch_rows = 1 << 27;
  c->partial_state_columnar = 0;
  c->force_generic_kernels = 0;
  c->agg_dense_keys = 1;
  c->agg_hot_key_cache = 1;                            // skew probe on the first batch -> CTA-private hot-key cache
}

}  // namespace b200q

// =====================================================================================================
// extern "C"
// =====================================================================================================
#define B200Q_STR2(x) #x
#define B200Q_STR(x) B200Q_STR2(x)

extern "C" {

int32_t b200q_version(void) { return 100; }
const char* b200q_build_info(void) { return "blaze_b200 hot path: Filter/Project/HashAgg, sm_90a, CUDA " B200Q_STR(CUDART_VERSION); }
const char* b200q_last_error(void) { return g_last_error.c_str(); }
int32_t b200q_device_count(void) { int n = 0; if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; } return n; }

b200q_status b200q_conf_init(b200q_conf* conf) {
  if (!conf) return fail(B200Q_ERR_INVALID_ARG, "conf is null");
  conf_defaults(conf); return B200Q_OK;
}

b200q_status b200q_plan_explain(const uint8_t* plan, size_t plan_len, int32_t plan_kind, char* buf, size_t cap, size_t* needed) {
  return guarded(nullptr, [&] {
    PlanP p = decode_plan(plan, plan_len, plan_kind);
    std::string s = explain_plan(p);
    if (needed) *needed = s.size() + 1;
    if (buf && cap) { const size_t n = std::min(cap - 1, s.size()); memcpy(buf, s.data(), n); buf[n] = 0; }
  });
}

b200q_status b200q_op_create(const uint8_t* plan, size_t plan_len, int32_t plan_kind, const struct ArrowSchema* input_schema,
                             const b200q_conf* conf, int32_t device, b200q_op** out) {
  if (!out) return fail(B200Q_ERR_INVALID_ARG, "out is null");
  *out = nullptr;
  b200q_op* op = nullptr;
  b200q_status st = guarded(nullptr, [&] {
    PlanP p = decode_plan(plan, plan_len, plan_kind);
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) { cudaGetLastError(); throw ExecError(B200Q_ERR_NO_DEVICE, "no CUDA device is visible: the sm_90a kernels cannot run and there is no CPU fallback"); }
    if (device < 0 || device >= ndev) throw ExecError(B200Q_ERR_INVALID_ARG, "invalid device ordinal");
    op = new b200q_op();
    op->plan = p; op->cx.device = device;
    conf_defaults(&op->cx.conf);
    if (conf) { const size_t n = std::min<size_t>(conf->struct_size ? conf->struct_size : sizeof(b200q_conf), sizeof(b200q_conf)); memcpy(&op->cx.conf, conf, n); op->cx.conf.struct_size = sizeof(b200q_conf); }
    if (op->cx.conf.batch_size <= 0) op->cx.conf.batch_size = 10000;
    if (op->cx.conf.max_launch_rows <= 0) op->cx.conf.max_launch_rows = 1 << 27;
    if (op->cx.conf.agg_initial_groups <= 0) op->cx.conf.agg_initial_groups = 1 << 19;
    B200Q_CUDA(cudaSetDevice(device));
    {   // keep freed blocks in the stream-ordered pool instead of returning them to the driver at every sync
      cudaMemPool_t pool; unsigned long long keep = ~0ULL;
      if (cudaDeviceGetDefaultMemPool(&pool, device) == cudaSuccess) cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &keep);
    }
    op->stream_ref = stream_ref_create(device);
    op->cx.stream = op->stream_ref->s;
    B200Q_CUDA(cudaEventCreate(&op->cx.ev0)); B200Q_CUDA(cudaEventCreate(&op->cx.ev1));
    build_pipeline(op);
    if (input_schema) {
      if (input_schema->n_children != (int64_t)op->in_schema.fields.size()) throw PlanError(B200Q_ERR_INVALID_ARG, "input_schema does not match the plan leaf: column count");
      for (int64_t i = 0; i < input_schema->n_children; i++)
        if (type_of_format(input_schema->children[i]->format) != op->in_schema.fields[i].type)
          throw PlanError(B200Q_ERR_INVALID_ARG, "input_schema does not match the plan leaf: type of column " + std::to_string(i));
    }
  });
  if (st != B200Q_OK) { if (op) { op->stages.clear(); delete op; } return st; }
  *out = op;
  return B200Q_OK;
}

b200q_status b200q_op_input_schema(b200q_op* op, struct ArrowSchema* out) {
  if (!op || !out) return fail(B200Q_ERR_INVALID_ARG, "null argument");
  return guarded(nullptr, [&] { export_schema(op->in_schema, out); });
}
b200q_status b200q_op_output_schema(b200q_op* op, struct ArrowSchema* out) {
  if (!op || !out) return fail(B200Q_ERR_INVALID_ARG, "null argument");
  return guarded(nullptr, [&] { export_schema(op->out_schema, out); });
}

b200q_status b200q_op_push(b200q_op* op, struct ArrowArray* batch) {
  if (!op) return fail(B200Q_ERR_INVALID_ARG, "op is null");
  b200q_status st = guarded(op, [&] {
    if (op->finished) throw ExecError(B200Q_ERR_STATE, "push after finish");
    B200Q_CUDA(cudaSetDevice(op->cx.device));
    validate_host_batch(op, batch);
    poll_pending(op, false);
    op->cx.m.input_rows += batch->length; op->cx.m.input_batches++;
    if (batch->length == 0) return;
    const std::vector<int>& used = op->stages[0]->used_input_cols;
    const int64_t srows = op->cx.conf.staging_rows;
    if (srows > 0 && batch->length < srows / 2) { staging_append(op, batch); return; }
    if (op->staging_ready) staging_flush(op);                       // keep arrival order
    DevBatch db = import_direct(op, batch, used);
    // the caller's buffers must outlive the async copies: release the batch when they have drained
    PendingRelease pr; pr.arr = *batch; batch->release = nullptr;
    B200Q_CUDA(cudaEventCreateWithFlags(&pr.ev, cudaEventDisableTiming));
    B200Q_CUDA(cudaEventRecord(pr.ev, op->cx.stream));
    op->pending.push_back(pr);
    run_stages(op, db, 0);
  });
  if (batch && batch->release) batch->release(batch);               // ownership moved to the library in every case
  return st;
}

b200q_status b200q_op_push_device(b200q_op* op, struct ArrowDeviceArray* dbatch) {
  if (!op) return fail(B200Q_ERR_INVALID_ARG, "op is null");
  b200q_status st = guarded(op, [&] {
    if (op->finished) throw ExecError(B200Q_ERR_STATE, "push after finish");
    if (!dbatch) throw ExecError(B200Q_ERR_INVALID_ARG, "null batch");
    if (dbatch->device_type != ARROW_DEVICE_CUDA || dbatch->device_id != op->cx.device) throw ExecError(B200Q_ERR_INVALID_ARG, "push_device: batch is not on this op's CUDA device");
    B200Q_CUDA(cudaSetDevice(op->cx.device));
    ArrowArray* batch = &dbatch->array;
    validate_host_batch(op, batch);
    poll_pending(op, false);
    if (op->staging_ready) staging_flush(op);
    if (dbatch->sync_event) B200Q_CUDA(cudaStreamWaitEvent(op->cx.stream, *(cudaEvent_t*)dbatch->sync_event, 0));
    op->cx.m.input_rows += batch->length; op->cx.m.input_batches++;
    if (batch->length == 0) return;
    DevBatch db; db.num_rows = batch->length; db.cols.resize(op->in_schema.fields.size());
    for (size_t i = 0; i < db.cols.size(); i++) {
      const ArrowArray* c = batch->children[i]; DevColumn& dc = db.cols[i];
      dc.type = op->in_schema.fields[i].type; dc.offset = c->offset + batch->offset;
      const size_t huge = (size_t)1 << 60;
      if (c->n_buffers > 0 && c->buffers[0] && c->null_count != 0) dc.validity = DevMem::borrow(c->buffers[0], huge, nullptr);
      if (dc.type.is_varlen()) { dc.offsets = DevMem::borrow(c->buffers[1], huge, nullptr); dc.values = DevMem::borrow(c->buffers[2], huge, nullptr); }
      else if (c->n_buffers > 1 && c->buffers[1]) dc.values = DevMem::borrow(c->buffers[1], huge, nullptr);
    }
    // queued BEFORE the stages run: if a stage throws, the array is still released (poll_pending) and the event destroyed;
    // in both cases the event is recorded behind the last kernel that reads the caller's buffers.
    PendingRelease pr; pr.arr = *batch;
    B200Q_CUDA(cudaEventCreateWithFlags(&pr.ev, cudaEventDisableTiming));
    batch->release = nullptr;
    op->pending.push_back(pr);
    const cudaEvent_t ev = pr.ev;
    try { run_stages(op, db, 0); } catch (...) { cudaEventRecord(ev, op->cx.stream); throw; }
    B200Q_CUDA(cudaEventRecord(ev, op->cx.stream));
  });
  if (dbatch && dbatch->array.release) dbatch->array.release(&dbatch->array);
  return st;
}

b200q_status b200q_op_finish(b200q_op* op) {
  if (!op) return fail(B200Q_ERR_INVALID_ARG, "op is null");
  return guarded(op, [&] {
    if (op->finished) return;
    B200Q_CUDA(cudaSetDevice(op->cx.device));
    {   // a ParquetScanExec leaf is the op's own source: read + decode the split now, one device batch per row group
      const PlanNode* leaf = op->plan.get();
      while (leaf->input) leaf = leaf->input.get();
      if (leaf->kind == N_LEAF && leaf->leaf_kind == "ParquetScan") {
        if (op->cx.m.input_batches) throw ExecError(B200Q_ERR_STATE, "an op whose leaf is a ParquetScanExecNode takes no pushed batches");
        run_parquet_scan(op->cx, *leaf, [&](DevBatch& b) { run_stages(op, b, 0); });
      }
    }
    if (op->staging_ready) staging_flush(op);
    for (size_t i = 0; i < op->stages.size(); i++) {
      std::vector<DevBatch> outs;
      op->cx.cur_stage = (int)i;
      op->stages[i]->finish(op->cx, outs);
      for (auto& o : outs) {
        if (i + 1 < op->stages.size()) run_stages(op, o, i + 1);
        else { op->cx.m.output_rows += o.num_rows; op->out_queue.push_back(std::move(o)); }
      }
    }
    B200Q_CUDA(cudaStreamSynchronize(op->cx.stream));
    poll_pending(op, true);
    op->finished = true;
  });
}

b200q_status b200q_op_pull(b200q_op* op, struct ArrowArray* out, int32_t* has_batch) {
  if (!op || !out || !has_batch) return fail(B200Q_ERR_INVALID_ARG, "null argument");
  *has_batch = 0;
  return guarded(op, [&] {
    B200Q_CUDA(cudaSetDevice(op->cx.device));
    if (!op->has_cur_host) {
      if (op->out_queue.empty()) return;
      op->cur_host = to_host(op, op->out_queue.front());
      op->out_queue.pop_front();
      op->has_cur_host = true;
    }
    HostBatch& hb = op->cur_host;
    const int64_t len = std::min<int64_t>(op->cx.conf.batch_size, hb.num_rows - hb.cursor);
    export_host_slice(hb, hb.cursor, len, out);
    hb.cursor += len;
    if (hb.cursor >= hb.num_rows) { op->has_cur_host = false; op->cur_host = HostBatch(); }
    op->cx.m.output_batches++;
    *has_batch = 1;
  });
}

b200q_status b200q_op_pull_device(b200q_op* op, struct ArrowDeviceArray* out, int32_t* has_batch) {
  if (!op || !out || !has_batch) return fail(B200Q_ERR_INVALID_ARG, "null argument");
  *has_batch = 0;
  return guarded(op, [&] {
    if (op->has_cur_host) throw ExecError(B200Q_ERR_STATE, "pull_device while a host batch is partially pulled");
    if (op->out_queue.empty()) return;
    B200Q_CUDA(cudaSetDevice(op->cx.device));
    B200Q_CUDA(cudaStreamSynchronize(op->cx.stream));
    export_device(op->out_queue.front(), op->cx.device, out);
    op->out_queue.pop_front();
    op->cx.m.output_batches++;
    *has_batch = 1;
  });
}

b200q_status b200q_op_sync(b200q_op* op) {
  if (!op) return fail(B200Q_ERR_INVALID_ARG, "op is null");
  return guarded(op, [&] { B200Q_CUDA(cudaSetDevice(op->cx.device)); B200Q_CUDA(cudaStreamSynchronize(op->cx.stream)); poll_pending(op, true); });
}

b200q_status b200q_op_metrics(b200q_op* op, b200q_metrics* out) {
  if (!op || !out) return fail(B200Q_ERR_INVALID_ARG, "null argument");
  const Metrics& m = op->cx.m;
  b200q_metrics r; memset(&r, 0, sizeof(r)); r.struct_size = sizeof(r);
  r.input_rows = m.input_rows; r.input_batches = m.input_batches; r.output_rows = m.output_rows; r.output_batches = m.output_batches;
  r.elapsed_compute_ns = (int64_t)(m.gpu_ms * 1e6); r.gpu_kernel_launches = m.launches; r.h2d_bytes = m.h2d_bytes; r.d2h_bytes = m.d2h_bytes;
  r.hot_kernel_ns = (int64_t)(m.hot_ms * 1e6); r.hot_kernel_rows = m.hot_rows; r.hot_kernel_launches = m.hot_launches;
  r.num_groups = m.num_groups; r.table_capacity_slots = m.table_capacity; r.table_grow_count = m.grow_count; r.fast_path_launches = m.fast_launches;
  const size_t n = std::min<size_t>(out->struct_size ? out->struct_size : sizeof(r), sizeof(r));
  memcpy(out, &r, n);
  return B200Q_OK;
}

void b200q_op_destroy(b200q_op* op) {
  if (!op) return;
  cudaSetDevice(op->cx.device);
  if (op->cx.stream) cudaStreamSynchronize(op->cx.stream);
  poll_pending(op, true);
  op->out_queue.clear(); op->has_cur_host = false; op->cur_host = HostBatch();
  op->stages.clear();
  staging_free(op);
  if (op->cx.ev0) cudaEventDestroy(op->cx.ev0);
  if (op->cx.ev1) cudaEventDestroy(op->cx.ev1);
  if (op->cx.stream) cudaStreamSynchronize(op->cx.stream);
  delete op;                     // the stream itself goes away with the last allocation that references it
}

b200q_status b200q_parquet_explain(const uint8_t* footer, size_t n, char* buf, size_t cap, size_t* needed) {
  return guarded(nullptr, [&] {
    const PqFileMeta m = parquet_parse_footer(footer, n);
    std::string o = "rows=" + std::to_string(m.num_rows) + " flat=" + (m.flat ? "true" : "false") + "\n";
    for (auto& c : m.columns) o += "column " + c.name + " physical=" + std::to_string(c.type) + (c.optional ? " optional" : " required") + " arrow=" + (c.arrow.id == T_NULL ? std::string("unsupported") : c.arrow.str()) + "\n";
    for (size_t g = 0; g < m.row_groups.size(); g++) {
      o += "row_group " + std::to_string(g) + " rows=" + std::to_string(m.row_groups[g].num_rows) + "\n";
      for (size_t c = 0; c < m.row_groups[g].columns.size(); c++) {
        const PqColumnChunk& cc = m.row_groups[g].columns[c];
        o += "  chunk " + std::to_string(c) + " codec=" + std::to_string(cc.codec) + " values=" + std::to_string(cc.num_values) + " start=" + std::to_string(cc.start()) + " bytes=" + std::to_string(cc.total_compressed_size) +
             " nulls=" + std::to_string(cc.stats.null_count) + " min_max=" + (cc.stats.has_min && cc.stats.has_max ? "yes" : "no") + "\n";
      }
    }
    if (needed) *needed = o.size() + 1;
    if (buf && cap) { const size_t k = std::min(cap - 1, o.size()); memcpy(buf, o.data(), k); buf[k] = 0; }
  });
}
b200q_status b200q_snappy_uncompress(const uint8_t* src, size_t n, uint8_t* dst, size_t cap, size_t* out_len) {
  if ((!src && n) || !out_len) return fail(B200Q_ERR_INVALID_ARG, "null argument");
  return guarded(nullptr, [&] {
    ByteBuf v; snappy_uncompress(src, n, v);
    *out_len = v.size();
    if (!dst || cap < v.size()) throw ExecError(B200Q_ERR_INVALID_ARG, "snappy output needs " + std::to_string(v.size()) + " bytes");
    if (v.size()) memcpy(dst, v.data(), v.size());
  });
}
b200q_status b200q_set_file_reader(b200q_file_reader_fn fn, void* ctx) { set_file_reader(fn, ctx); return B200Q_OK; }

b200q_status b200q_op_attach_build(b200q_op* probe_op, b200q_op* build_op) {
  if (!probe_op || !build_op) return fail(B200Q_ERR_INVALID_ARG, "null argument");
  return guarded(probe_op, [&] {
    const JoinBuildResult* b = build_op->stages.empty() ? nullptr : dynamic_cast<const JoinBuildResult*>(build_op->stages.back().get());
    if (!b) throw ExecError(B200Q_ERR_STATE, "attach_build: the build op's plan is not rooted at a BroadcastJoinBuildHashMapExecNode");
    if (!build_op->finished || !b->built()) throw ExecError(B200Q_ERR_STATE, "attach_build: finish the build op first");
    JoinProbeAttach* a = nullptr;
    for (auto& st : probe_op->stages) if (auto* j = dynamic_cast<JoinProbeAttach*>(st.get())) a = j;
    if (!a) throw ExecError(B200Q_ERR_STATE, "attach_build: the probe op's plan has no join");
    a->attach(b->built());
  });
}

b200q_status b200q_op_shuffle_chunk_count(b200q_op* op, int64_t* out_count) {
  if (!op || !out_count) return fail(B200Q_ERR_INVALID_ARG, "null argument");
  return guarded(op, [&] {
    const ShuffleResult* r = op->stages.empty() ? nullptr : dynamic_cast<const ShuffleResult*>(op->stages.back().get());
    if (!r) throw ExecError(B200Q_ERR_STATE, "the plan is not rooted at a ShuffleWriterExecNode");
    *out_count = r->chunk_count();
  });
}
b200q_status b200q_op_shuffle_chunk(b200q_op* op, int64_t index, b200q_shuffle_chunk* out) {
  if (!op || !out) return fail(B200Q_ERR_INVALID_ARG, "null argument");
  return guarded(op, [&] {
    const ShuffleResult* r = op->stages.empty() ? nullptr : dynamic_cast<const ShuffleResult*>(op->stages.back().get());
    if (!r) throw ExecError(B200Q_ERR_STATE, "the plan is not rooted at a ShuffleWriterExecNode");
    if (index < 0 || index >= r->chunk_count()) throw ExecError(B200Q_ERR_INVALID_ARG, "shuffle chunk index out of range");
    r->chunk(index, out);
  });
}
b200q_status b200q_lz4_frame_compress(const uint8_t* src, size_t n, uint8_t* dst, size_t cap, size_t* out_len) {
  if ((!src && n) || !out_len) return fail(B200Q_ERR_INVALID_ARG, "null argument");
  return guarded(nullptr, [&] {
    std::vector<uint8_t> v; lz4_frame_append(src, n, v);
    *out_len = v.size();
    if (!dst || cap < v.size()) throw ExecError(B200Q_ERR_INVALID_ARG, "lz4 frame needs " + std::to_string(v.size()) + " bytes");
    memcpy(dst, v.data(), v.size());
  });
}

b200q_status b200q_murmur3_partition(const struct ArrowSchema* key_schema, const struct ArrowDeviceArray* keys, int32_t num_partitions,
                                     uint32_t* out_pids_device, void* cuda_stream) {
  return guarded(nullptr, [&] {
    if (!key_schema || !keys || !out_pids_device) throw ExecError(B200Q_ERR_INVALID_ARG, "null argument");
    if (num_partitions <= 0) throw ExecError(B200Q_ERR_INVALID_ARG, "num_partitions must be positive");
    const ArrowArray& a = keys->array;
    if (a.n_children != key_schema->n_children || a.n_children > VM_MAX_COLS) throw ExecError(B200Q_ERR_INVALID_ARG, "key schema / array mismatch");
    ColTable ct{}; uint8_t phys[VM_MAX_COLS];
    for (int64_t i = 0; i < a.n_children; i++) {
      const DType t = type_of_format(key_schema->children[i]->format);
      if (t.is_varlen()) throw ExecError(B200Q_ERR_UNSUPPORTED, "murmur3 partition ids over a " + t.str() + " key are not on the GPU path");
      const ArrowArray* c = a.children[i];
      DevColumn dc; dc.type = t; dc.offset = c->offset + a.offset;
      phys[i] = phys_of(t);
      const int w = t.byte_width();
      ct.col[i].values = c->n_buffers > 1 ? (const uint8_t*)c->buffers[1] + (size_t)dc.offset * w : nullptr;
      ct.col[i].validity = (c->n_buffers > 0 && c->null_count != 0) ? (const uint8_t*)c->buffers[0] : nullptr;
      ct.col[i].bit_offset = (uint32_t)dc.offset;
    }
    launch_murmur3_partition(ct, phys, (int)a.n_children, a.length, num_partitions, out_pids_device, (cudaStream_t)cuda_stream);
    B200Q_CUDA(cudaGetLastError());
  });
}

}  // extern "C"
