// Stage implementations: FilterProjectStage and AggStage (see runtime.h).
#include <algorithm>
#include <chrono>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <unordered_map>

#include "runtime.h"
#include "kernels_fast.cuh"

namespace b200q {

// ---------------------------------------------------------------------------------------------------
static std::mutex g_stream_mu;
static std::unordered_map<cudaStream_t, std::weak_ptr<StreamRef>> g_streams;

StreamRef::~StreamRef() {
  { std::lock_guard<std::mutex> l(g_stream_mu); g_streams.erase(s); }
  if (s) { cudaSetDevice(device); cudaStreamSynchronize(s); cudaStreamDestroy(s); }
}
std::shared_ptr<StreamRef> stream_ref_create(int device) {
  auto r = std::make_shared<StreamRef>(); r->device = device;
  B200Q_CUDA(cudaStreamCreateWithFlags(&r->s, cudaStreamNonBlocking));
  std::lock_guard<std::mutex> l(g_stream_mu); g_streams[r->s] = r;
  return r;
}
std::shared_ptr<StreamRef> stream_ref_lookup(cudaStream_t s) {
  std::lock_guard<std::mutex> l(g_stream_mu);
  auto it = g_streams.find(s);
  return it == g_streams.end() ? nullptr : it->second.lock();
}

DevMem::~DevMem() {
  if (owned && ptr) {
    if (stream_keep) { cudaSetDevice(stream_keep->device); cudaFreeAsync(ptr, stream_keep->s); }
    else cudaFree(ptr);
  }
}
DevMemP DevMem::alloc(size_t bytes, cudaStream_t s, bool zero) {
  auto m = std::make_shared<DevMem>();
  m->bytes = bytes; m->stream = s; m->owned = true; m->stream_keep = stream_ref_lookup(s);
  if (bytes == 0) bytes = 16;
  {
    // HBM exhaustion is not a CUDA failure of the handle: the reference spills / skips under memory pressure
    // (agg_table.rs:108-120,540-588); here the op reports UNSUPPORTED so the host re-runs the task on its CPU operators
    const cudaError_t e = cudaMallocAsync(&m->ptr, bytes, s);
    if (e == cudaErrorMemoryAllocation) {
      cudaGetLastError(); m->ptr = nullptr; m->owned = false;
      throw ExecError(B200Q_ERR_UNSUPPORTED, "out of HBM: a device allocation of " + std::to_string(bytes) + " bytes failed; this task must fall back to the host path");
    }
    B200Q_CUDA(e);
  }
  if (zero) B200Q_CUDA(cudaMemsetAsync(m->ptr, 0, bytes, s));
  return m;
}
DevMemP DevMem::borrow(const void* p, size_t bytes, std::shared_ptr<void> owner) {
  auto m = std::make_shared<DevMem>();
  m->ptr = const_cast<void*>(p); m->bytes = bytes; m->owned = false; m->owner = std::move(owner);
  return m;
}

static inline size_t bitmap_bytes(int64_t n) { return (size_t)((n + 31) / 32) * 4; }

DevCol dev_col_of(const DevColumn& c) {
  DevCol d{};
  const int w = c.type.byte_width();
  d.values = c.values ? (const uint8_t*)c.values->ptr + (size_t)c.offset * (size_t)w : nullptr;
  if (c.type.is_varlen()) d.offsets = c.offsets ? (const int32_t*)c.offsets->ptr + c.offset : nullptr;   // values: the data base the offsets index
  d.validity = c.validity ? (const uint8_t*)c.validity->ptr : nullptr;
  d.bit_offset = (uint32_t)c.offset;
  if (c.offset > 0xFFFFFFFFLL) throw ExecError(B200Q_ERR_UNSUPPORTED, "column offset beyond 2^32 rows");
  return d;
}

// the program in device memory, its Utf8 constants relocated to their device addresses
static DevMemP upload_program(const CompiledProgram& cp, cudaStream_t s) {
  DevMemP d = DevMem::alloc(sizeof(VmProgram), s);
  const VmProgram p = relocated_program(cp, d->ptr);
  B200Q_CUDA(cudaMemcpyAsync(d->ptr, &p, sizeof(VmProgram), cudaMemcpyHostToDevice, s));
  B200Q_CUDA(cudaStreamSynchronize(s));                 // `p` lives on this stack frame
  return d;
}

static void check_device_error_flags(int flags) {
  if (flags & 1) throw ExecError(B200Q_ERR_EXECUTION, "Arrow error: Divide by zero error");
  if (flags & 2) throw ExecError(B200Q_ERR_EXECUTION, "Arrow error: Arithmetic overflow");
  if (flags & 4) throw ExecError(B200Q_ERR_EXECUTION, "corrupted accumulator row in the Binary agg buffer column");
}

// ---------------------------------------------------------------------------------------------------
// FilterProjectStage
// ---------------------------------------------------------------------------------------------------
class FilterProjectStage : public Stage {
  CompiledProgram cp_;
  DevMemP d_prog_;
  bool has_filters_;
  bool identity_ = false;            // no filter, output i = input column i: batches are forwarded as they are (no copy, no launch)
  bool lean_possible_ = false;
  LeanFpSpec lean_{};
  // variable-width outputs (Utf8 / Binary column references): gathered from the input column, not evaluated by the VM program.
  // out_src_[i] >= 0: output i is input column out_src_[i]; vm_out_[i]: index among the program's outputs otherwise
  std::vector<int> out_src_, vm_out_;
  bool varlen_ = false;
  int sel_out_ = -1;                 // program output holding the source row of each survivor (filtered plans with varlen outputs)

  int slot_of(int col_index) const { for (size_t i = 0; i < cp_.used_cols.size(); i++) if (cp_.used_cols[i] == col_index) return (int)i; return -1; }
  static bool is_i64(const DType& t) { return t.id == T_INT64 || t.id == T_TIMESTAMP_US; }

  // M0-class plans: `col cmp literal` conjuncts and column / column-op-column|literal projections over int64
  void detect_lean(const std::vector<ExprP>& filters, const std::vector<ExprP>& outs) {
    lean_possible_ = false;
    if (filters.size() > 4 || outs.size() > 8 || outs.empty() || cp_.used_cols.empty() || cp_.used_cols.size() > 4) return;
    LeanFpSpec sp{}; sp.nfilt = (int)filters.size(); sp.nout = (int)outs.size();
    for (size_t f = 0; f < filters.size(); f++) {
      const ExprP& p = filters[f];
      if (p->kind != E_BINARY || p->op < OP_EQ || p->op > OP_GE) return;
      ExprP l = p->children[0], r = p->children[1]; int op = p->op - OP_EQ;
      if (l->kind == E_LITERAL && r->kind == E_COLUMN) { std::swap(l, r); static const int flip[] = {CMP_EQ, CMP_NE, CMP_GT, CMP_GE, CMP_LT, CMP_LE}; op = flip[op]; }
      if (l->kind != E_COLUMN || r->kind != E_LITERAL || r->lit_null || !is_i64(l->type) || !is_i64(r->type)) return;
      const int s = slot_of(l->col_index); if (s < 0 || s > 127) return;
      sp.filt[f].col = (int8_t)s; sp.filt[f].op = (uint8_t)op; sp.filt[f].lit = (long long)r->lit_lo;
    }
    for (size_t o = 0; o < outs.size(); o++) {
      const ExprP& e = outs[o];
      if (!is_i64(e->type)) return;
      if (e->kind == E_COLUMN) { const int s = slot_of(e->col_index); if (s < 0 || s > 127) return; sp.out[o].kind = 0; sp.out[o].a = (int8_t)s; sp.out[o].b = -1; continue; }
      if (e->kind != E_BINARY || (e->op != OP_PLUS && e->op != OP_MINUS && e->op != OP_MUL)) return;
      const ExprP &l = e->children[0], &r = e->children[1];
      if (l->kind != E_COLUMN || !is_i64(l->type)) return;
      const int sa = slot_of(l->col_index); if (sa < 0 || sa > 127) return;
      sp.out[o].kind = (uint8_t)(e->op == OP_PLUS ? 1 : e->op == OP_MINUS ? 2 : 3); sp.out[o].a = (int8_t)sa;
      if (r->kind == E_COLUMN && is_i64(r->type)) { const int sb = slot_of(r->col_index); if (sb < 0 || sb > 127) return; sp.out[o].b = (int8_t)sb; }
      else if (r->kind == E_LITERAL && !r->lit_null && is_i64(r->type)) { sp.out[o].b = -1; sp.out[o].lit = (long long)r->lit_lo; }
      else return;
    }
    lean_ = sp; lean_possible_ = true;
  }

 public:
  FilterProjectStage(OpContext& cx, const SchemaDef& in, const std::vector<ExprP>& filters, const std::vector<ExprP>& outs, const SchemaDef& out) {
    in_schema = in; out_schema = out;
    has_filters_ = !filters.empty();
    identity_ = !has_filters_ && outs.size() == in.fields.size();
    for (size_t i = 0; identity_ && i < outs.size(); i++) identity_ = outs[i]->kind == E_COLUMN && outs[i]->col_index == (int)i && outs[i]->type == in.fields[i].type;
    std::vector<ExprP> vm_outs;
    for (const ExprP& o : outs) {
      ExprP e = o;
      while ((e->kind == E_TRY_CAST || e->kind == E_CAST) && e->children[0]->type == e->type) e = e->children[0];
      if (!e->type.is_varlen()) { out_src_.push_back(-1); vm_out_.push_back((int)vm_outs.size()); vm_outs.push_back(o); continue; }
      if (e->kind != E_COLUMN)
        throw PlanError(B200Q_ERR_UNSUPPORTED, "ProjectExec: " + explain_expr(o) + " produces a " + e->type.str() + " value; only " + e->type.str() + " column references are on the hot path");
      out_src_.push_back(e->col_index); vm_out_.push_back(-1);
    }
    varlen_ = vm_outs.size() != outs.size();
    if (varlen_ && has_filters_) sel_out_ = (int)vm_outs.size();
    cp_ = compile_program(filters, vm_outs, has_filters_, sel_out_);
    used_input_cols = cp_.used_cols;
    for (int c : out_src_) if (c >= 0 && std::find(used_input_cols.begin(), used_input_cols.end(), c) == used_input_cols.end()) used_input_cols.push_back(c);
    if (!cx.conf.force_generic_kernels && !varlen_ && !cp_.has_strings) detect_lean(filters, outs);
    d_prog_ = upload_program(cp_, cx.stream);
  }

  void push(OpContext& cx, DevBatch& in, std::vector<DevBatch>& outs) override {
    const int64_t n = in.num_rows;
    if (n == 0) return;
    if (n > 0x7FFFFFFFLL) throw ExecError(B200Q_ERR_UNSUPPORTED, "batches above 2^31-1 rows must be split by the caller");
    if (identity_) {
      bool plain = true;
      auto ours = [](const DevMemP& m) { return !m || m->owned || m->owner; };          // borrowed caller memory (push_device) is only valid until the batch is released
      for (auto& c : in.cols) plain = plain && c.offset == 0 && ours(c.values) && ours(c.validity) && ours(c.offsets);
      if (plain) { outs.push_back(in); return; }
    }
    ColTable ct{};
    for (size_t i = 0; i < cp_.used_cols.size(); i++) ct.col[i] = dev_col_of(in.cols[cp_.used_cols[i]]);
    OutTable ot{};
    DevBatch ob;
    for (size_t i = 0; i < cp_.outs.size(); i++) {
      const OutDesc& od = cp_.outs[i];
      DevColumn c; c.type = od.type;
      const bool is_bool = od.type.id == T_BOOL;
      c.values = is_bool ? DevMem::alloc(bitmap_bytes(n), cx.stream, true) : DevMem::alloc((size_t)n * od.type.byte_width(), cx.stream);
      if (od.nullable) c.validity = DevMem::alloc(bitmap_bytes(n), cx.stream, true);
      ot.values[i] = c.values->ptr; ot.validity[i] = c.validity ? (uint32_t*)c.validity->ptr : nullptr; ot.phys[i] = phys_of(od.type);
      ob.cols.push_back(c);
    }
    DevMemP sel;
    if (sel_out_ >= 0) { sel = DevMem::alloc((size_t)n * 4, cx.stream); ot.values[sel_out_] = sel->ptr; ot.validity[sel_out_] = nullptr; ot.phys[sel_out_] = PH_SEL; }
    bool lean = lean_possible_;
    for (size_t i = 0; lean && i < cp_.used_cols.size(); i++) lean = ct.col[i].validity == nullptr;
    DevMemP scratch = DevMem::alloc(32, cx.stream, true);
    DevMemP status;
    B200Q_CUDA(cudaEventRecord(cx.ev0, cx.stream));
    if (lean) {
      // outputs of non-null inputs are never NULL: the (zeroed) validity bitmaps become all-ones
      for (auto& c : ob.cols) if (c.validity) B200Q_CUDA(cudaMemsetAsync(c.validity->ptr, 0xFF, c.validity->bytes, cx.stream));
      if (has_filters_) status = DevMem::alloc((size_t)filter_project_lean_scratch_bytes(n), cx.stream, true);
      long long* outp[8]; for (size_t i = 0; i < cp_.outs.size(); i++) outp[i] = (long long*)ot.values[i];
      cx.m.launches += launch_filter_project_lean(ct, (int)cp_.used_cols.size(), lean_, outp, n, status ? status->ptr : nullptr, (unsigned long long*)scratch->ptr, cx.stream);
      cx.m.fast_launches++;
    } else {
      if (has_filters_) status = DevMem::alloc((size_t)filter_project_num_tiles(n) * 8, cx.stream, true);
      cx.m.launches += launch_filter_project((const VmProgram*)d_prog_->ptr, ct, ot, (int)cp_.outs.size(), n, has_filters_,
                                             status ? (unsigned long long*)status->ptr : nullptr, (unsigned long long*)scratch->ptr, cx.stream);
    }
    B200Q_CUDA(cudaEventRecord(cx.ev1, cx.stream));
    B200Q_CUDA(cudaGetLastError());
    unsigned long long h[4];
    B200Q_CUDA(cudaMemcpyAsync(h, scratch->ptr, 32, cudaMemcpyDeviceToHost, cx.stream));
    B200Q_CUDA(cudaStreamSynchronize(cx.stream));
    { float ms = 0; B200Q_CUDA(cudaEventElapsedTime(&ms, cx.ev0, cx.ev1)); cx.m.gpu_ms += ms; if (cx.cur_stage == 0) { cx.m.hot_ms += ms; cx.m.hot_rows += n; cx.m.hot_launches++; } }
    check_device_error_flags((int)h[2]);
    ob.num_rows = (int64_t)h[1];
    if (ob.num_rows == 0) return;                            // sender.send drops empty batches (execution_context.rs:713-716)
    if (!varlen_) { outs.push_back(std::move(ob)); return; }
    DevBatch res; res.num_rows = ob.num_rows;
    for (size_t i = 0; i < out_src_.size(); i++) res.cols.push_back(out_src_[i] < 0 ? ob.cols[(size_t)vm_out_[i]] : DevColumn());
    gather_varlen(cx, in, sel ? (const uint32_t*)sel->ptr : nullptr, res);
    outs.push_back(std::move(res));
  }

  // the Utf8 / Binary outputs of `res` = rows sel[0..m) (sel null: rows 0..m) of their input columns.  Lengths, validity and offsets
  // of every column are computed first, so that one host round trip brings back all byte totals before the data is allocated.
  void gather_varlen(OpContext& cx, const DevBatch& in, const uint32_t* sel, DevBatch& res) {
    const int64_t m = res.num_rows;
    auto ours = [](const DevMemP& p) { return !p || p->owned || p->owner; };           // borrowed caller memory (push_device) must be copied
    struct Job { size_t out; DevCol src; };
    std::vector<Job> jobs;
    for (size_t i = 0; i < out_src_.size(); i++) {
      if (out_src_[i] < 0) continue;
      const DevColumn& c = in.cols[(size_t)out_src_[i]];
      // no filter: share the buffers (imported offsets always start at 0, so the column indexes its own allocation)
      if (!sel && c.offset == 0 && ours(c.values) && ours(c.offsets) && ours(c.validity)) { res.cols[i] = c; continue; }
      jobs.push_back(Job{i, dev_col_of(c)});
    }
    if (jobs.empty()) return;
    const size_t nj = jobs.size();
    DevMemP totals = DevMem::alloc(nj * 8, cx.stream, true);
    std::vector<DevMemP> keep;
    for (size_t j = 0; j < nj; j++) {
      DevColumn& o = res.cols[jobs[j].out];
      const DevColumn& c = in.cols[(size_t)out_src_[jobs[j].out]];
      o.type = c.type;
      o.offsets = DevMem::alloc((size_t)(m + 1) * 4, cx.stream);
      if (c.validity && out_schema.fields[jobs[j].out].nullable) o.validity = DevMem::alloc(bitmap_bytes(m), cx.stream);
      DevMemP lengths = DevMem::alloc((size_t)m * 4 + 16, cx.stream), sums = DevMem::alloc((size_t)scan_num_blocks(m) * 4 + 16, cx.stream);
      cx.m.launches += launch_varlen_lengths(jobs[j].src, sel, m, (int32_t*)lengths->ptr, o.validity ? (uint32_t*)o.validity->ptr : nullptr,
                                             (unsigned long long*)totals->ptr + j, cx.stream);
      cx.m.launches += launch_exclusive_scan_i32((const int32_t*)lengths->ptr, (int32_t*)o.offsets->ptr, m, (int32_t*)sums->ptr, cx.stream);
      keep.push_back(lengths); keep.push_back(sums);                  // released stream-ordered after the scans
    }
    std::vector<unsigned long long> bytes(nj);
    B200Q_CUDA(cudaMemcpyAsync(bytes.data(), totals->ptr, nj * 8, cudaMemcpyDeviceToHost, cx.stream));
    B200Q_CUDA(cudaStreamSynchronize(cx.stream));
    for (size_t j = 0; j < nj; j++) {
      DevColumn& o = res.cols[jobs[j].out];
      if (bytes[j] > 0x7FFFFFFFULL) throw ExecError(B200Q_ERR_UNSUPPORTED, "a " + o.type.str() + " output column of one batch exceeds 2 GiB (32-bit Arrow offsets); push smaller batches");
      o.values = DevMem::alloc((size_t)bytes[j], cx.stream);
      cx.m.launches += launch_varlen_copy(jobs[j].src, sel, m, (const int32_t*)o.offsets->ptr, (uint8_t*)o.values->ptr, cx.stream);
    }
    B200Q_CUDA(cudaGetLastError());
  }
  void finish(OpContext&, std::vector<DevBatch>&) override {}
};

std::unique_ptr<Stage> make_filter_project_stage(OpContext& cx, const SchemaDef& in_schema, const std::vector<ExprP>& filters,
                                                 const std::vector<ExprP>& outs, const SchemaDef& out_schema) {
  return std::unique_ptr<Stage>(new FilterProjectStage(cx, in_schema, filters, outs, out_schema));
}

// ---------------------------------------------------------------------------------------------------
// ExpandStage: one FilterProjectStage per projection, run in order over every pushed batch (the pending filters below the Expand
// are evaluated by each of them).  Outputs that share the input's buffers hold their own references, so `in` outlives them all.
// ---------------------------------------------------------------------------------------------------
class ExpandStage : public Stage {
  std::vector<std::unique_ptr<FilterProjectStage>> sets_;
 public:
  ExpandStage(OpContext& cx, const SchemaDef& in, const std::vector<ExprP>& filters, const std::vector<std::vector<ExprP>>& projections, const SchemaDef& out) {
    in_schema = in; out_schema = out;
    for (auto& p : projections) {
      sets_.emplace_back(new FilterProjectStage(cx, in, filters, p, out));
      for (int c : sets_.back()->used_input_cols) if (std::find(used_input_cols.begin(), used_input_cols.end(), c) == used_input_cols.end()) used_input_cols.push_back(c);
    }
    std::sort(used_input_cols.begin(), used_input_cols.end());
  }
  void push(OpContext& cx, DevBatch& in, std::vector<DevBatch>& outs) override { for (auto& s : sets_) s->push(cx, in, outs); }
  void finish(OpContext&, std::vector<DevBatch>&) override {}
};

std::unique_ptr<Stage> make_expand_stage(OpContext& cx, const SchemaDef& in_schema, const std::vector<ExprP>& filters,
                                         const std::vector<std::vector<ExprP>>& projections, const SchemaDef& out_schema) {
  return std::unique_ptr<Stage>(new ExpandStage(cx, in_schema, filters, projections, out_schema));
}

// ---------------------------------------------------------------------------------------------------
// AggStage
// ---------------------------------------------------------------------------------------------------
static uint64_t host_mix64(uint64_t x) { x ^= x >> 33; x *= 0xff51afd7ed558ccdULL; x ^= x >> 33; x *= 0xc4ceb9fe1a85ec53ULL; x ^= x >> 33; return x; }

StateCols state_columns_of(const AggDef& a) {
  StateCols s; DType i64; i64.id = T_INT64;
  switch (a.fn) {
    case AGG_COUNT: s.fields.push_back(FieldDef{a.field_name, i64, false}); break;
    case AGG_AVG:
      s.fields.push_back(FieldDef{a.field_name + "#sum", a.data_type, true});
      s.fields.push_back(FieldDef{a.field_name + "#count", i64, false});
      break;
    default: s.fields.push_back(FieldDef{a.field_name, a.data_type, true}); break;
  }
  return s;
}

// can this expression evaluate to NULL?  (conservative; used to drop validity tracking)
static bool cast_may_fail(const DType& f, const DType& t) {
  if (f == t) return false;
  auto ii = [](const DType& d) { return d.is_integer() || d.id == T_DATE32 || d.id == T_TIMESTAMP_US || d.id == T_BOOL; };
  if (ii(f) && ii(t)) return t.int_bits() < f.int_bits();
  if (ii(f) && t.is_float()) return false;
  if (f.is_float() && (t.is_float() || t.is_integer() || t.id == T_BOOL)) return false;
  return true;
}
static bool can_be_null(const ExprP& e) {
  switch (e->kind) {
    case E_COLUMN: return e->nullable;
    case E_LITERAL: return e->lit_null || e->type.id == T_NULL;
    case E_BINARY:
      if (e->op == OP_AND || e->op == OP_OR) return e->nullable;
      return can_be_null(e->children[0]) || can_be_null(e->children[1]);
    case E_IS_NULL: case E_IS_NOT_NULL: return false;
    case E_NOT: case E_NEGATIVE: return can_be_null(e->children[0]);
    case E_CAST: case E_TRY_CAST: return can_be_null(e->children[0]) || cast_may_fail(e->children[0]->type, e->type);
    default: return true;
  }
}

static bool same_expr(const ExprP& a, const ExprP& b) {
  if (a == b) return true;
  if (a->kind != b->kind || a->type != b->type || a->children.size() != b->children.size()) return false;
  if (a->kind == E_COLUMN) return a->col_index == b->col_index;
  if (a->kind == E_LITERAL) return a->lit_null == b->lit_null && a->lit_lo == b->lit_lo && a->lit_hi == b->lit_hi && a->lit_str == b->lit_str;
  if (a->kind == E_STR_MATCH && (a->str_match != b->str_match || a->lit_str != b->lit_str)) return false;
  if (a->kind == E_BINARY && a->op != b->op) return false;
  if (a->kind == E_SCALAR_FN && a->name != b->name) return false;
  if (a->kind == E_IN_LIST && a->negated != b->negated) return false;
  if (a->kind == E_CASE && (a->case_has_base != b->case_has_base || a->case_has_else != b->case_has_else)) return false;
  for (size_t i = 0; i < a->children.size(); i++) if (!same_expr(a->children[i], b->children[i])) return false;
  return true;
}
// strip casts that change nothing on the device (same 64-bit representation, cannot fail)
static ExprP strip_noop_casts(ExprP e) {
  while ((e->kind == E_CAST || e->kind == E_TRY_CAST) && !cast_may_fail(e->children[0]->type, e->type)) {
    const DType &f = e->children[0]->type, &t = e->type;
    const bool same_repr = (f == t) || (f.is_intlike() && t.is_intlike());
    if (!same_repr) break;
    e = e->children[0];
  }
  return e;
}

// NULL whatever the row: a NULL literal, through any casts
static bool is_null_literal(ExprP e) {
  while (e->kind == E_CAST || e->kind == E_TRY_CAST) e = e->children[0];
  return e->kind == E_LITERAL && (e->lit_null || e->type.id == T_NULL);
}
// a grouping key that is one value for every row of a grouping set (the rolled-up NULLs and the grouping id of an Expand):
// folded into the set's constant key words, in the representation the VM gives the same value
static bool const_key(const ExprP& e0, bool& null, uint64_t& lo, uint64_t& hi) {
  if (is_null_literal(e0)) { null = true; lo = hi = 0; return true; }
  const ExprP e = strip_noop_casts(e0);
  if (e->kind != E_LITERAL || !(e->type.is_intlike() || e->type.is_decimal())) return false;
  null = false; lo = e->lit_lo; hi = e->lit_hi;
  return true;
}

// Small pinned host slots (counter snapshots).  cudaMallocHost / cudaFreeHost cost milliseconds once tens of GB are mapped in the process, so
// ops never call them on their own: one pinned page per process, 32-byte slots, recycled.
class PinnedSlots {
  std::mutex mu_; std::vector<unsigned long long*> free_; 
 public:
  unsigned long long* get() {
    std::lock_guard<std::mutex> l(mu_);
    if (free_.empty()) {
      unsigned long long* page = nullptr;
      B200Q_CUDA(cudaMallocHost((void**)&page, 4096));
      for (int i = 0; i < 4096 / 32; i++) free_.push_back(page + i * 4);
    }
    unsigned long long* p = free_.back(); free_.pop_back(); return p;
  }
  void put(unsigned long long* p) { std::lock_guard<std::mutex> l(mu_); free_.push_back(p); }
};
static PinnedSlots& pinned_slots() { static PinnedSlots* p = new PinnedSlots(); return *p; }

class AggStage : public Stage {
  PlanNode node_;                       // copy of the Agg node (exprs already rewritten over the stage input)
  std::vector<ExprP> filters_;
  std::vector<ExprP> vm_outs_;          // keys, then accumulator arguments
  CompiledProgram cp_;
  DevMemP d_prog_;
  AggLayout lay_{};
  bool merge_mode_ = false, columnar_ = false, final_ = false;
  int n_in_ = 0;                        // input columns
  std::vector<FieldDef> merge_state_fields_;   // state columns fed by the merge-mode aggs (in agg order)
  int first_state_col_ = 0;             // index of the first state column in the program's column space
  // grouping sets of a fused ExpandExec (nsets_ > 1): per-set keys and arguments over the shared VM outputs
  int nsets_ = 1;
  std::vector<AggSetDesc> sets_;
  DevMemP d_sets_;

  // table
  DevMemP keys_, accs_, counters_, deferred_[2];
  uint64_t capacity_ = 0;
  int64_t deferred_cap_ = 0;
  int64_t ngroups_ = 0;

  // specialised kernels (kernels_fast.cu)
  bool fast_ok_ = false, dense_possible_ = false, dense_decided_ = false;
  bool acc_arg_nullable_[2] = {true, true};
  FastSpec fs_{};
  DenseEmitMap dmap_{};
  DevMemP dense_tab_, sink_;
  // wide tile aggregates (f64 / decimal / MIN / MAX accumulators over a dense table, kernels_tile.cu)
  bool wide_possible_ = false;
  TileAggSpec ws_{};
  int64_t wide_rows_since_norm_ = 0;

  // emit plan (per output/state column)
  struct EmitSpec { EmitCol ec; FieldDef field; bool frozen_count = false; };
  std::vector<EmitSpec> emit_;          // key columns first, then per-agg result or state columns
  std::vector<FrozenField> frozen_fields_;     // non-final, reference format: how the state columns freeze

  int add_out(const ExprP& e) {
    ExprP s = strip_noop_casts(e);
    for (size_t i = 0; i < vm_outs_.size(); i++) if (same_expr(vm_outs_[i], s)) return (int)i;
    if (nsets_ > 1 && (int)vm_outs_.size() >= VM_MAX_OUT)
      throw PlanError(B200Q_ERR_UNSUPPORTED, "ExpandExec below AggExec: the grouping sets need more than " + std::to_string(VM_MAX_OUT) + " distinct key and argument expressions (VM_MAX_OUT)");
    vm_outs_.push_back(s);
    return (int)vm_outs_.size() - 1;
  }

  static uint8_t frozen_width(const DType& t) { return (uint8_t)t.byte_width(); }

 public:
  AggStage(OpContext& cx, const SchemaDef& in, const std::vector<ExprP>& filters, const PlanNode& agg,
           const std::vector<ExprP>& group_exprs, const std::vector<std::vector<ExprP>>& agg_args, const std::vector<AggSetExprs>& sets) : node_(agg), filters_(filters) {
    in_schema = in; out_schema = agg.schema;
    n_in_ = (int)in.fields.size();
    merge_mode_ = agg.need_partial_merge; final_ = agg.need_final_merge;
    columnar_ = cx.conf.partial_state_columnar != 0;
    if (agg.exec_mode != 0 && !agg.group_exprs.empty()) {
      // SortAgg over sorted input produces the same multiset of groups; the GPU always hashes.
    }
    if ((int)group_exprs.size() > AGG_MAX_KEYS) throw PlanError(B200Q_ERR_UNSUPPORTED, "more than 8 grouping columns");
    if (merge_mode_ && !filters.empty()) throw PlanError(B200Q_ERR_UNSUPPORTED, "Filter fused below a merge-mode aggregate");
    const bool multi = sets.size() > 1;
    if (multi) {
      if ((int)sets.size() > AGG_MAX_SETS)
        throw PlanError(B200Q_ERR_UNSUPPORTED, "ExpandExec below AggExec: " + std::to_string(sets.size()) + " projections exceed the limit of " + std::to_string(AGG_MAX_SETS) + " grouping sets (AGG_MAX_SETS)");
      if (merge_mode_) throw PlanError(B200Q_ERR_UNSUPPORTED, "ExpandExec fused below a merge-mode aggregate");
      nsets_ = (int)sets.size();
      sets_.resize(nsets_);
      for (auto& d : sets_) { memset(&d, 0, sizeof(d)); memset(d.acc_arg, AGG_NO_ARG, sizeof(d.acc_arg)); }
    }

    // ---- state columns consumed by merge-mode aggs
    for (auto& a : agg.aggs) if (a.mode != MODE_PARTIAL) for (auto& f : state_columns_of(a).fields) merge_state_fields_.push_back(f);
    if (merge_mode_) {
      if (columnar_) {
        first_state_col_ = n_in_ - (int)merge_state_fields_.size();
        if (first_state_col_ < (int)0) throw PlanError(B200Q_ERR_INVALID_PLAN, "columnar partial state: input has too few columns");
        for (size_t k = 0; k < merge_state_fields_.size(); k++)
          if (in.fields[first_state_col_ + k].type != merge_state_fields_[k].type)
            throw PlanError(B200Q_ERR_INVALID_PLAN, "columnar partial state: column " + in.fields[first_state_col_ + k].name + " has type " +
                                                        in.fields[first_state_col_ + k].type.str() + ", expected " + merge_state_fields_[k].type.str());
      } else {
        first_state_col_ = n_in_;
        if (in.fields.empty() || in.fields.back().type.id != T_BINARY)
          throw PlanError(B200Q_ERR_INVALID_PLAN, "merge-mode aggregate: the last input column must be the Binary agg buffer column (agg_ctx.rs:280)");
      }
    }

    // ---- slot layout
    lay_.nkeys = (int)group_exprs.size();
    int word = 1;
    for (int k = 0; k < lay_.nkeys; k++) {
      const ExprP& g = group_exprs[k];
      if (!multi) {
        lay_.key_out[k] = (uint8_t)add_out(g);
        if (lay_.key_out[k] != k) throw PlanError(B200Q_ERR_UNSUPPORTED, "duplicate grouping expressions");
      } else lay_.key_out[k] = AGG_KEY_CONST;                      // per set: sets_[s].key_out[k]
      lay_.key_word[k] = (uint8_t)word; lay_.key_nwords[k] = g->type.is_decimal() ? 2 : 1;
      word += lay_.key_nwords[k];
    }
    // grouping sets: a key that is a literal in a set is folded into the set's constant words; every other key expression is a
    // (deduplicated) VM output, so two key positions of one set may share one output and still keep their own key words
    for (int s = 0; multi && s < nsets_; s++)
      for (int k = 0; k < lay_.nkeys; k++) {
        AggSetDesc& d = sets_[s];
        bool null = false; uint64_t lo = 0, hi = 0;
        if (const_key(sets[s].group_exprs[k], null, lo, hi)) {
          d.key_out[k] = AGG_KEY_CONST;
          if (null) d.key_null |= 1u << k;
          else { d.key_const[lay_.key_word[k] - 1] = lo; if (lay_.key_nwords[k] == 2) d.key_const[lay_.key_word[k]] = hi; }
        } else d.key_out[k] = (uint8_t)add_out(sets[s].group_exprs[k]);
      }
    lay_.nkw = word - 1;
    const int key_entry_words = word;
    word = 0;                                                     // from here on `word` counts words of the accumulator entry
    for (int i = 0; i < AGG_MAX_SLOT_WORDS; i++) lay_.init[i] = 0;
    lay_.init_flags = 0;
    int vbits = 0, state_k = 0;
    auto new_vbit = [&]() { if (vbits >= 15) throw PlanError(B200Q_ERR_UNSUPPORTED, "too many nullable accumulators in one aggregate"); return (uint8_t)vbits++; };
    auto state_col_expr = [&](const FieldDef& f) {
      auto e = std::make_shared<Expr>(); e->kind = E_COLUMN; e->col_index = first_state_col_ + state_k++; e->name = f.name; e->type = f.type; e->nullable = f.nullable;
      return ExprP(e);
    };
    auto add_acc = [&](AccKind kind, int nwords, uint8_t vbit, const std::vector<int>& args, uint64_t init_lo, uint64_t init_hi) {
      if (lay_.nacc >= AGG_MAX_ACC) throw PlanError(B200Q_ERR_UNSUPPORTED, "too many accumulators in one aggregate");
      if (word + nwords > AGG_MAX_SLOT_WORDS) throw PlanError(B200Q_ERR_UNSUPPORTED, "aggregate state too wide for one table slot");
      AccOp& a = lay_.acc[lay_.nacc++];
      a.kind = kind; a.word = (uint8_t)word; a.vbit = vbit; a.nargs = (uint8_t)args.size();
      for (size_t i = 0; i < args.size() && i < 4; i++) a.arg_out[i] = (uint8_t)args[i];
      lay_.init[word] = init_lo; if (nwords == 2) lay_.init[word + 1] = init_hi;
      const int w = word; word += nwords; return w;
    };

    // key emit columns
    for (int k = 0; k < lay_.nkeys; k++) {
      EmitSpec es{}; es.ec.kind = EMIT_KEY; es.ec.phys = phys_of(group_exprs[k]->type); es.ec.word = lay_.key_word[k]; es.ec.key = (uint8_t)k; es.ec.vbit = 0xFF;
      es.field = agg.schema.fields[k];
      emit_.push_back(es);
    }

    for (size_t ai = 0; ai < agg.aggs.size(); ai++) {
      const AggDef& a = agg.aggs[ai];
      const bool partial = a.mode == MODE_PARTIAL;
      const DType& dt = a.data_type;
      if ((a.fn == AGG_MIN || a.fn == AGG_MAX) && dt.id == T_BOOL) throw PlanError(B200Q_ERR_UNSUPPORTED, "min/max over boolean is not on the hot path");
      int sum_word = -1, cnt_word = -1; uint8_t sum_vbit = 0xFF;
      // --- sum-like part (Sum, Avg, Min, Max)
      if (a.fn != AGG_COUNT) {
        ExprP arg;
        if (partial) { arg = agg_args[ai][0]; }
        else { arg = state_col_expr(state_columns_of(a).fields[0]); }
        // grouping sets: each set's argument is its own VM output; a set whose argument is a NULL literal skips the accumulator
        std::vector<int> set_o(nsets_, -1);
        bool set_nullable = false;
        for (int s = 0; multi && s < nsets_; s++) {
          const ExprP& e = sets[s].agg_args[ai][0];
          if (is_null_literal(e)) { set_nullable = true; continue; }
          set_o[s] = add_out(e); set_nullable = set_nullable || can_be_null(e);
        }
        int o = 0;
        if (!multi) o = add_out(arg);
        else for (int s = nsets_ - 1; s >= 0; s--) if (set_o[s] >= 0) o = set_o[s];
        // no-grouping aggregates always emit one (pre-seeded) row: with no valid input the accumulator stays NULL
        // (AccPrimColumn valids stay false, agg_exec.rs:280-323), so it needs a validity bit even for never-NULL arguments
        const bool nullable_arg = (multi ? set_nullable : can_be_null(arg)) || lay_.nkeys == 0;
        const uint8_t vbit = nullable_arg ? new_vbit() : (uint8_t)0xFF;
        AccKind kind; int nwords = 1; uint64_t ilo = 0, ihi = 0;
        if (a.fn == AGG_SUM || a.fn == AGG_AVG) {
          if (dt.is_decimal()) { kind = ACC_ADD_DEC; nwords = 2; }
          else if (dt.id == T_FLOAT64) { kind = ACC_ADD_F64; ilo = 0x8000000000000000ULL; }   // -0.0: see tile_identity
          else if (dt.is_integer()) kind = ACC_ADD_I64;
          else throw PlanError(B200Q_ERR_UNSUPPORTED, "sum/avg accumulating at " + dt.str() + " is not on the hot path");
        } else {
          const bool mn = a.fn == AGG_MIN;
          if (dt.is_decimal()) { kind = mn ? ACC_MIN_DEC : ACC_MAX_DEC; nwords = 2; ilo = mn ? ~0ULL : 0ULL; ihi = mn ? 0x7FFFFFFFFFFFFFFFULL : 0x8000000000000000ULL; }
          else if (dt.is_float()) { kind = mn ? ACC_MIN_F64 : ACC_MAX_F64; ilo = mn ? 0x7FFFFFFFFFFFFFFFULL : 0x8000000000000000ULL; }
          else if (dt.is_intlike()) { kind = mn ? ACC_MIN_I64 : ACC_MAX_I64; ilo = mn ? 0x7FFFFFFFFFFFFFFFULL : 0x8000000000000000ULL; }
          else throw PlanError(B200Q_ERR_UNSUPPORTED, "min/max over " + dt.str() + " is not on the hot path");
        }
        sum_word = add_acc(kind, nwords, vbit, {o}, ilo, ihi); sum_vbit = vbit;
        for (int s = 0; multi && s < nsets_; s++) {
          if (set_o[s] < 0) sets_[s].acc_skip |= 1u << (lay_.nacc - 1);
          else sets_[s].acc_arg[lay_.nacc - 1][0] = (uint8_t)set_o[s];
        }
      }
      // --- count part (Count, Avg)
      if (a.fn == AGG_COUNT || a.fn == AGG_AVG) {
        if (multi) {
          std::vector<std::vector<int>> set_args(nsets_);
          std::vector<bool> skip(nsets_, false);
          for (int s = 0; s < nsets_; s++) {
            const auto& srcs = a.fn == AGG_AVG ? std::vector<ExprP>{sets[s].agg_args[ai][0]} : sets[s].agg_args[ai];
            for (auto& e : srcs) {
              if (is_null_literal(e)) skip[s] = true;
              else if (can_be_null(e)) set_args[s].push_back(add_out(e));
            }
            if (set_args[s].size() > 4) throw PlanError(B200Q_ERR_UNSUPPORTED, "count over more than 4 nullable arguments");
          }
          cnt_word = add_acc(ACC_COUNT, 1, 0xFF, set_args[0], 0, 0);
          for (int s = 0; s < nsets_; s++) {
            if (skip[s]) { sets_[s].acc_skip |= 1u << (lay_.nacc - 1); continue; }
            for (size_t i = 0; i < set_args[s].size(); i++) sets_[s].acc_arg[lay_.nacc - 1][i] = (uint8_t)set_args[s][i];
          }
        } else if (partial) {
          std::vector<int> args;
          const auto& srcs = a.fn == AGG_AVG ? std::vector<ExprP>{agg_args[ai][0]} : agg_args[ai];
          for (auto& e : srcs) if (can_be_null(e)) args.push_back(add_out(e));      // agg.rs:178-189 + never-NULL arguments dropped
          if (args.size() > 4) throw PlanError(B200Q_ERR_UNSUPPORTED, "count over more than 4 nullable arguments");
          cnt_word = add_acc(ACC_COUNT, 1, 0xFF, args, 0, 0);
        } else {
          const auto sc = state_columns_of(a);
          const int o = add_out(state_col_expr(sc.fields.back()));
          cnt_word = add_acc(ACC_ADD_I64, 1, 0xFF, {o}, 0, 0);
        }
      }
      // --- emit columns
      auto value_spec = [&](const FieldDef& f, int w, uint8_t vbit, bool order_key) {
        EmitSpec es{}; es.ec.kind = EMIT_ACC_VALUE; es.ec.phys = phys_of(f.type); es.ec.word = (uint8_t)w; es.ec.vbit = vbit; es.ec.is_order_key = order_key; es.field = f; return es;
      };
      const bool order_key = (a.fn == AGG_MIN || a.fn == AGG_MAX) && dt.is_float();
      if (final_) {
        const FieldDef& of = agg.schema.fields[lay_.nkeys + ai];
        if (a.fn == AGG_COUNT) emit_.push_back(value_spec(of, cnt_word, 0xFF, false));
        else if (a.fn == AGG_AVG) {
          EmitSpec es{}; es.field = of; es.ec.word = (uint8_t)sum_word; es.ec.word2 = (uint8_t)cnt_word; es.ec.vbit = sum_vbit;
          if (dt.is_decimal()) { es.ec.kind = EMIT_AVG_DEC; es.ec.phys = PH_DEC128; }
          else { es.ec.kind = EMIT_AVG_F64; es.ec.phys = PH_F64; es.ec.sum_is_f64 = dt.id == T_FLOAT64; }
          emit_.push_back(es);
        } else emit_.push_back(value_spec(of, sum_word, sum_vbit, order_key));
      } else {
        const auto sc = state_columns_of(a);
        if (a.fn == AGG_COUNT) { emit_.push_back(value_spec(sc.fields[0], cnt_word, 0xFF, false)); emit_.back().frozen_count = true; }
        else {
          emit_.push_back(value_spec(sc.fields[0], sum_word, sum_vbit, order_key));
          if (a.fn == AGG_AVG) { emit_.push_back(value_spec(sc.fields[1], cnt_word, 0xFF, false)); emit_.back().frozen_count = true; }
        }
      }
    }
    if (lay_.nkeys == 0 && lay_.nacc == 0) throw PlanError(B200Q_ERR_UNSUPPORTED, "aggregate without groupings and aggregates");
    // entry strides: powers of two up to a 32-byte sector (an entry never straddles a sector), multiples of 4 words beyond
    auto stride_of = [](int words) { return words <= 1 ? 1 : words <= 2 ? 2 : words <= 4 ? 4 : (words + 3) & ~3; };
    lay_.kstride = std::max(2, stride_of(key_entry_words));      // {hdr, key0} is probed with one 16-byte load
    lay_.astride = stride_of(std::max(word, 1));
    if (lay_.kstride > AGG_MAX_SLOT_WORDS || lay_.astride > AGG_MAX_SLOT_WORDS) throw PlanError(B200Q_ERR_UNSUPPORTED, "aggregate state too wide for one table slot");

    if (!final_ && columnar_) {          // typed state columns instead of the Binary agg-buffer column
      out_schema.fields.resize(lay_.nkeys);
      for (size_t i = lay_.nkeys; i < emit_.size(); i++) out_schema.fields.push_back(emit_[i].field);
    }

    // ---- program
    cp_ = compile_program(filters_, vm_outs_, false);
    lay_.nouts = (int)cp_.outs.size();
    int ow = 0;
    for (size_t i = 0; i < cp_.outs.size(); i++) { lay_.out_word[i] = (uint8_t)ow; ow += cp_.outs[i].slots; }
    if (ow > AGG_MAX_ROW_WORDS) {
      if (multi) throw PlanError(B200Q_ERR_UNSUPPORTED, "ExpandExec below AggExec: the grouping sets need " + std::to_string(ow) + " key/argument words per row, more than " + std::to_string(AGG_MAX_ROW_WORDS) + " (AGG_MAX_ROW_WORDS)");
      throw PlanError(B200Q_ERR_UNSUPPORTED, "too many key/argument words per row");
    }
    for (int c : cp_.used_cols) if (c < n_in_) used_input_cols.push_back(c);
    if (merge_mode_ && !columnar_) used_input_cols.push_back(n_in_ - 1);
    std::sort(used_input_cols.begin(), used_input_cols.end());
    used_input_cols.erase(std::unique(used_input_cols.begin(), used_input_cols.end()), used_input_cols.end());
    d_prog_ = upload_program(cp_, cx.stream);
    if (multi) {                              // the set descriptors travel next to the program (they do not fit the kernel parameters)
      d_sets_ = DevMem::alloc(sizeof(AggSetDesc) * sets_.size(), cx.stream);
      B200Q_CUDA(cudaMemcpyAsync(d_sets_->ptr, sets_.data(), sizeof(AggSetDesc) * sets_.size(), cudaMemcpyHostToDevice, cx.stream));
    }

    if (!cp_.has_strings && !multi) {         // the specialised kernels read fixed-width columns only: string programs stay on the VM kernel;
                                              // they insert one key per row, so grouping sets stay on the VM kernel too
      detect_fast(cx);
      if (!fast_ok_) detect_wide(cx);
    }

    // ---- frozen-row descriptors of the state columns (non-final output in the reference format)
    if (!final_) {
      for (size_t i = lay_.nkeys; i < emit_.size(); i++) {
        FrozenField f{}; const FieldDef& fd = emit_[i].field;
        f.kind = emit_[i].frozen_count ? FZ_COUNT : FZ_PRIM; f.width = frozen_width(fd.type); f.phys = phys_of(fd.type);
        frozen_fields_.push_back(f);
      }
    }

    // ---- table
    // capacity: any size (slot = mulhi(hash, capacity)); sized for a load of ~0.6 at the hinted group count so that
    // key area + accumulator area stay L2-resident; floor 2^20 keeps the slack above the load limit (0.3 * capacity)
    // larger than the concurrent-insert overshoot bound (resident threads ~ 303K)
    capacity_ = std::max<uint64_t>(1ULL << 20, (uint64_t)((double)std::max<int64_t>(cx.conf.agg_initial_groups, 1) * AGG_SLOTS_PER_GROUP));
    if (capacity_ >= (1ULL << 32)) throw PlanError(B200Q_ERR_UNSUPPORTED, "agg_initial_groups too large");
    alloc_table(cx, capacity_, keys_, accs_, counters_);
    if (lay_.nkeys == 0) seed_global_group(cx);
    B200Q_CUDA(cudaStreamSynchronize(cx.stream));
    cx.m.table_capacity = (int64_t)capacity_;
  }


  // ---- specialised-kernel eligibility -------------------------------------------------------------------
  int prog_col_slot(int col_index) const {
    for (size_t i = 0; i < cp_.used_cols.size(); i++) if (cp_.used_cols[i] == col_index) return (int)i;
    return -1;
  }
  static bool int_phys(const DType& t) { return t.is_intlike(); }

  // the 1-2 integer key columns and the `col cmp literal` conjuncts of the specialised kernels (key slots, filt[], merged
  // into frange[] by merge_conjuncts); false: a key or a conjunct they cannot read
  bool parse_keys_and_conjuncts(FastSpec& fs) const {
    if (lay_.nkeys < 1 || lay_.nkeys > 2 || filters_.size() > 4) return false;
    fs.nkeys = lay_.nkeys; fs.nfilt = (int)filters_.size();
    for (int k = 0; k < lay_.nkeys; k++) {
      const ExprP& e = vm_outs_[lay_.key_out[k]];
      if (e->kind != E_COLUMN || !int_phys(e->type) || lay_.key_nwords[k] != 1) return false;
      const int s = prog_col_slot(e->col_index); if (s < 0 || s > 127) return false;
      fs.key_col[k] = (int8_t)s; fs.key_phys[k] = phys_of(e->type);
    }
    for (size_t f = 0; f < filters_.size(); f++) {
      const ExprP& p = filters_[f];
      if (p->kind != E_BINARY || p->op < OP_EQ || p->op > OP_GE) return false;
      ExprP l = strip_noop_casts(p->children[0]), r = strip_noop_casts(p->children[1]);
      int op = p->op - OP_EQ;
      if (l->kind == E_LITERAL && r->kind == E_COLUMN) { std::swap(l, r); static const int flip[] = {CMP_EQ, CMP_NE, CMP_GT, CMP_GE, CMP_LT, CMP_LE}; op = flip[op]; }
      if (l->kind != E_COLUMN || r->kind != E_LITERAL || r->lit_null || !int_phys(l->type) || !int_phys(r->type)) return false;
      const int s = prog_col_slot(l->col_index); if (s < 0 || s > 127) return false;
      fs.filt[f].col = (int8_t)s; fs.filt[f].phys = phys_of(l->type); fs.filt[f].op = (uint8_t)op; fs.filt[f].lit = (long long)r->lit_lo;
    }
    merge_conjuncts(fs);
    return true;
  }

  void detect_fast(OpContext& cx) {
    fast_ok_ = false;
    if (cx.conf.force_generic_kernels) return;
    if (lay_.nacc < 1 || lay_.nacc > 2) return;
    FastSpec fs{};
    if (!parse_keys_and_conjuncts(fs)) return;
    fs.nacc = lay_.nacc;
    for (int j = 0; j < lay_.nacc; j++) {
      const AccOp& a = lay_.acc[j];
      fs.acc[j].vbit = a.vbit; fs.acc[j].word = a.word; fs.acc[j].col = -1; fs.acc[j].phys = PH_I64;
      if (a.kind == ACC_ADD_I64) {
        const ExprP& e = vm_outs_[a.arg_out[0]];
        if (e->kind != E_COLUMN || !int_phys(e->type)) return;
        const int s = prog_col_slot(e->col_index); if (s < 0 || s > 127) return;
        fs.acc[j].kind = FAST_ACC_ADD; fs.acc[j].col = (int8_t)s; fs.acc[j].phys = phys_of(e->type);
        acc_arg_nullable_[j] = e->nullable;
      } else if (a.kind == ACC_COUNT && a.nargs <= 1) {
        fs.acc[j].kind = FAST_ACC_COUNT;
        if (a.nargs == 1) {
          const ExprP& e = vm_outs_[a.arg_out[0]];
          if (e->kind != E_COLUMN || !(e->type.is_intlike() || e->type.is_float() || e->type.is_decimal())) return;
          const int s = prog_col_slot(e->col_index); if (s < 0 || s > 127) return;
          fs.acc[j].col = (int8_t)s; fs.acc[j].phys = phys_of(e->type);
        }
      } else return;
    }
    if (lay_.nacc == 2 && lay_.acc[0].word / 4 != lay_.acc[1].word / 4) return;
    sink_ = DevMem::alloc((size_t)FAST_SINK_WARPS * 32, cx.stream, true);
    fs.sink = (unsigned long long*)sink_->ptr;
    fs_ = fs; fast_ok_ = true;
    // DENSE mode needs: integer keys with small value ranges (decided on the first batch) and an entry of at most 4 words
    dense_possible_ = cx.conf.agg_dense_keys != 0;
    if (dense_possible_) {
      for (size_t c = 0; c < emit_.size(); c++) {
        const EmitCol& ec = emit_[c].ec;
        if (ec.kind == EMIT_KEY) continue;
        bool found = false; for (int i = 0; i < lay_.nacc; i++) found |= fs_.acc[i].word == ec.word;
        if (ec.kind != EMIT_ACC_VALUE || ec.is_order_key || !found) { dense_possible_ = false; break; }
      }
    }
    if (dense_possible_) dense_possible_ = dense_layout();
  }

  // FilterExec conjuncts arrive pre-split as `col cmp literal` terms (NativeFilterBase.scala:66-87): all terms on one
  // column intersect to one closed interval [lo, lo + span], tested by the tile kernels with one subtract + one
  // unsigned compare.  `!=` terms or more than two filter columns keep the per-conjunct kernels (nfcol = -1).
  static void merge_conjuncts(FastSpec& fs) {
    fs.nfcol = 0; fs.filt_never = 0;
    long long lo[2] = {INT64_MIN, INT64_MIN}, hi[2] = {INT64_MAX, INT64_MAX}; bool never = false;
    for (int f = 0; f < fs.nfilt; f++) {
      int c = -1;
      for (int i = 0; i < fs.nfcol; i++) if (fs.frange[i].col == fs.filt[f].col) c = i;
      if (c < 0) { if (fs.nfcol == 2) { fs.nfcol = -1; return; } c = fs.nfcol++; fs.frange[c].col = fs.filt[f].col; fs.frange[c].phys = fs.filt[f].phys; }
      const long long lit = fs.filt[f].lit;
      switch (fs.filt[f].op) {
        case CMP_EQ: lo[c] = std::max(lo[c], lit); hi[c] = std::min(hi[c], lit); break;
        case CMP_LT: if (lit == INT64_MIN) never = true; else hi[c] = std::min(hi[c], lit - 1); break;
        case CMP_LE: hi[c] = std::min(hi[c], lit); break;
        case CMP_GT: if (lit == INT64_MAX) never = true; else lo[c] = std::max(lo[c], lit + 1); break;
        case CMP_GE: lo[c] = std::max(lo[c], lit); break;
        default: fs.nfcol = -1; return;                              // CMP_NE
      }
    }
    for (int c = 0; c < fs.nfcol; c++) {
      if (lo[c] > hi[c]) never = true;
      fs.frange[c].lo = lo[c]; fs.frange[c].span = (unsigned long long)hi[c] - (unsigned long long)lo[c];
    }
    fs.filt_never = never ? 1 : 0;
  }

  // ---- WIDE tile aggregates: everything the FAST_ACC_ADD / FAST_ACC_COUNT family does not cover --------------------
  // 1-2 integer key columns, mergeable conjuncts, up to 4 accumulators of ONE RED flavour over at most two argument columns
  // (a decimal128 argument takes both value registers).  Dense keys only (decided on the first batch like DENSE mode).
  void detect_wide(OpContext& cx) {
    wide_possible_ = false;
    if (cx.conf.force_generic_kernels || !cx.conf.agg_dense_keys) return;
    if (lay_.nacc < 1 || lay_.nacc > 4) return;
    TileAggSpec ts{};
    {
      FastSpec fs{};
      if (!parse_keys_and_conjuncts(fs) || fs.nfcol < 0) return;
      ts.nkeys = fs.nkeys; ts.nfcol = fs.nfcol; ts.filt_never = fs.filt_never;
      for (int k = 0; k < 2; k++) { ts.key_col[k] = fs.key_col[k]; ts.key_phys[k] = fs.key_phys[k]; ts.frange[k] = fs.frange[k]; }
    }
    ts.nacc = lay_.nacc; ts.dec_word = 0xFF;
    // flavour
    bool any_f64 = false, any_min = false, any_int = false;
    for (int j = 0; j < lay_.nacc; j++) {
      switch (lay_.acc[j].kind) {
        case ACC_ADD_F64: any_f64 = true; break;
        case ACC_MIN_I64: case ACC_MAX_I64: case ACC_MIN_F64: case ACC_MAX_F64: any_min = true; break;
        case ACC_ADD_I64: case ACC_ADD_DEC: any_int = true; break;
        case ACC_COUNT: break;
        default: return;                                               // 128-bit MIN / MAX stay on the generic kernel
      }
    }
    if ((int)any_f64 + (int)any_min + (int)any_int > 1) return;
    ts.flavour = any_f64 ? TF_ADD_F64 : any_min ? TF_MIN_S64 : TF_ADD_U64;
    const unsigned long long ONE = ts.flavour == TF_ADD_F64 ? 0x3FF0000000000000ULL : ts.flavour == TF_MIN_S64 ? 0ULL : 1ULL;
    const unsigned long long NOOP = tile_identity(ts.flavour);
    // argument columns
    struct ArgInfo { int col_index; int cvt; bool nullable; bool values; };
    std::vector<ArgInfo> args; std::vector<ExprP> arg_cols;
    unsigned long long dec_mul = 1; bool dec_mul_seen = false;
    auto arg_of = [&](const ExprP& e0, int want_cvt, bool values, bool dec) -> int {
      ExprP e = strip_noop_casts(e0); int cvt = TC_NONE;
      const bool nullable = can_be_null(e0);
      if ((e->kind == E_CAST || e->kind == E_TRY_CAST)) {
        const ExprP& c = e->children[0];
        if (c->kind == E_COLUMN && c->type.is_intlike() && e->type.id == T_FLOAT64) { cvt = TC_I2F; e = c; }                     // Rust `as f64` (arrow/cast.rs test_int_to_float)
        else if (c->kind == E_COLUMN && c->type.is_decimal() && e->type.is_decimal() && e->type.scale >= c->type.scale && e->type.scale - c->type.scale <= 18 &&
                 (int)e->type.precision - (int)c->type.precision >= (int)e->type.scale - (int)c->type.scale) {
          // decimal -> decimal with at least as many extra digits as extra scale: an exact multiplication that cannot overflow
          unsigned long long mul = 1; for (int i = c->type.scale; i < e->type.scale; i++) mul *= 10ULL;
          if (dec_mul_seen && dec_mul != mul) return -1;
          dec_mul = mul; dec_mul_seen = true; e = c;
        }
        else return -1;
      }
      if (e->kind != E_COLUMN) return -1;
      if (!values) { for (size_t i = 0; i < args.size(); i++) if (args[i].col_index == e->col_index) { args[i].nullable = args[i].nullable || nullable; return (int)i; } }
      if (values) {
        if (dec) { if (!e->type.is_decimal()) return -1; }
        else if (want_cvt == TC_ORDER) { if (e->type.id != T_FLOAT64 || cvt != TC_NONE) return -1; cvt = TC_ORDER; }
        else if (ts.flavour == TF_ADD_F64) { if (!(e->type.id == T_FLOAT64 && cvt == TC_NONE) && cvt != TC_I2F) return -1; }
        else if (!e->type.is_intlike() || cvt != TC_NONE) return -1;
      }
      for (size_t i = 0; i < args.size(); i++)
        if (args[i].col_index == e->col_index && (!values || !args[i].values || args[i].cvt == cvt)) { args[i].nullable = args[i].nullable || nullable; if (values && !args[i].values) { args[i].values = true; args[i].cvt = cvt; } return (int)i; }
      if (args.size() == 2) return -1;
      args.push_back(ArgInfo{e->col_index, cvt, nullable, values}); arg_cols.push_back(e);
      return (int)args.size() - 1;
    };
    int acc_arg[4] = {-1, -1, -1, -1};
    for (int j = 0; j < lay_.nacc; j++) {
      const AccOp& a = lay_.acc[j];
      if (a.kind == ACC_COUNT) { if (a.nargs > 1) return; if (a.nargs == 1) { acc_arg[j] = arg_of(vm_outs_[a.arg_out[0]], TC_NONE, false, false); if (acc_arg[j] < 0) return; } continue; }
      const bool dec = a.kind == ACC_ADD_DEC, order = a.kind == ACC_MIN_F64 || a.kind == ACC_MAX_F64;
      acc_arg[j] = arg_of(vm_outs_[a.arg_out[0]], order ? TC_ORDER : TC_NONE, true, dec);
      if (acc_arg[j] < 0) return;
      if (dec) { if ((ts.arg_is_dec && acc_arg[j] != 0) || acc_arg[j] != 0) return; ts.arg_is_dec = 1; }
    }
    if (ts.arg_is_dec && args.size() > 1) return;                       // a decimal argument takes both value registers
    ts.nargs = (int)args.size(); ts.dec_mul = dec_mul;
    for (size_t i = 0; i < args.size(); i++) {
      const int s = prog_col_slot(args[i].col_index); if (s < 0 || s > 127) return;
      const DType& t = arg_cols[i]->type;
      if (args[i].values && !ts.arg_is_dec && !(t.is_intlike() || t.id == T_FLOAT64)) return;
      ts.arg_col[i] = (int8_t)s; ts.arg_phys[i] = t.id == T_FLOAT64 ? (uint8_t)PH_I64 : phys_of(t); ts.arg_cvt[i] = (uint8_t)args[i].cvt; ts.arg_values[i] = args[i].values ? 1 : 0;
    }
    // entry words: [presence] [valid-argument mark per nullable argument] [accumulator words]
    int w = 0;
    auto constant_word = [&](unsigned long long cst, int gate) { TileWord tw{}; tw.srcsel = 2; tw.gate = (uint8_t)gate; tw.cst = cst; return tw; };
    ts.presence_word = 0; ts.word[w++] = constant_word(ONE, 30);
    int valid_word[2] = {-1, -1};
    for (size_t i = 0; i < args.size(); i++) if (args[i].nullable) { valid_word[i] = w; ts.word[w++] = constant_word(ONE, 28 + (int)i); }
    for (int j = 0; j < lay_.nacc; j++) {
      const AccOp& a = lay_.acc[j]; const int arg = acc_arg[j];
      auto& out = ts.acc[j]; out.arg = (int8_t)arg; out.lay_acc = (uint8_t)j; out.valid_word = 0xFF; out.recon = TR_COPY;
      if (a.kind == ACC_COUNT) {
        if (ts.flavour == TF_MIN_S64) return;
        out.w0 = (uint8_t)(arg >= 0 && valid_word[arg] >= 0 ? valid_word[arg] : 0);
        out.recon = ts.flavour == TF_ADD_F64 ? TR_F2I : TR_COPY;
        continue;
      }
      if (a.vbit != 0xFF) { if (valid_word[arg] < 0) return; out.valid_word = (uint8_t)valid_word[arg]; }
      if (w + (a.kind == ACC_ADD_DEC ? 3 : 1) > 8) return;
      out.w0 = (uint8_t)w;
      TileWord tw{}; tw.srcsel = (uint8_t)arg; tw.gate = (uint8_t)(28 + arg); tw.msk = ~0ULL;
      if (a.kind == ACC_ADD_DEC) {
        ts.dec_word = (uint8_t)w; out.recon = TR_DEC3;
        TileWord lo = tw; lo.srcsel = 0; lo.msk = 0xFFFFFFFFULL; ts.word[w++] = lo;
        TileWord mid = lo; mid.sh = 32; ts.word[w++] = mid;
        TileWord hi = tw; hi.srcsel = 1; ts.word[w++] = hi;
      } else {
        if (a.kind == ACC_MAX_I64 || a.kind == ACC_MAX_F64) { tw.inv = ~0ULL; out.recon = TR_NOT; }
        ts.word[w++] = tw;
      }
    }
    if (w > 8) return;
    ts.G = w <= 2 ? 2 : w <= 4 ? 4 : 8;
    for (; w < ts.G; w++) ts.word[w] = constant_word(NOOP, 30);
    // every emit column must be something the hashed-slot view can produce (always true for these accumulator kinds)
    sink_ = DevMem::alloc((size_t)FAST_SINK_WARPS * 32, cx.stream);
    { std::vector<unsigned long long> fill((size_t)FAST_SINK_WARPS * 4, NOOP); B200Q_CUDA(cudaMemcpyAsync(sink_->ptr, fill.data(), fill.size() * 8, cudaMemcpyHostToDevice, cx.stream)); B200Q_CUDA(cudaStreamSynchronize(cx.stream)); }
    ts.sink = (unsigned long long*)sink_->ptr;
    ws_ = ts; wide_possible_ = true;
  }

  // DENSE decision from the key ranges of (a sample of) the first batch.  The range kernel of every key (and, with
  // probe_skew, the skew probe) are enqueued back to back and their results come back in ONE host round trip.  Each
  // key's range is padded to [min - margin, max + margin]; false: the keys are too sparse for a table of entry_words
  // words per entry, or it would exceed agg_max_table_bytes (stay on the hash table)
  struct DenseRange { long long base[2] = {0, 0}; uint64_t span[2] = {1, 1}; uint64_t entries = 1; bool hot = false; };
  bool dense_range(OpContext& cx, const ColTable& ct, int64_t n, int nkeys, const int8_t* key_col, const uint8_t* key_phys, int entry_words,
                   bool probe_skew, DenseRange& dr) {
    const int64_t sample = std::min<int64_t>(n, 1 << 22);
    DevMemP d = DevMem::alloc(64, cx.stream);
    { const long long init[8] = {INT64_MAX, INT64_MIN, 0, INT64_MAX, INT64_MIN, 0, 0, 0};
      B200Q_CUDA(cudaMemcpyAsync(d->ptr, init, 64, cudaMemcpyHostToDevice, cx.stream)); }
    for (int k = 0; k < nkeys; k++) cx.m.launches += launch_key_range(ct.col[key_col[k]], key_phys[k], sample, (long long*)d->ptr + 3 * k, cx.stream);
    DevMemP hist;
    if (probe_skew) {
      hist = DevMem::alloc((65536 + 1) * 4, cx.stream, true);
      DevCol kc[2] = {ct.col[key_col[0]], ct.col[key_col[nkeys == 2 ? 1 : 0]]};
      cx.m.launches += launch_key_skew_probe(kc, key_phys, nkeys, sample, (unsigned*)hist->ptr, cx.stream);
    }
    long long hr[6] = {0}; unsigned mx = 0;
    B200Q_CUDA(cudaMemcpyAsync(hr, d->ptr, 48, cudaMemcpyDeviceToHost, cx.stream));
    if (probe_skew) B200Q_CUDA(cudaMemcpyAsync(&mx, (unsigned*)hist->ptr + 65536, 4, cudaMemcpyDeviceToHost, cx.stream));
    B200Q_CUDA(cudaStreamSynchronize(cx.stream));
    long long nonnull = 0;
    for (int k = 0; k < nkeys; k++) {
      const long long* h = hr + 3 * k;                                     // {min, max, non-null rows}
      if (h[2] <= 0 || h[1] < h[0]) return false;
      const unsigned __int128 range = (unsigned __int128)((__int128)h[1] - (__int128)h[0]) + 1;
      if (range > ((uint64_t)1 << 26)) return false;
      const uint64_t r = (uint64_t)range, margin = r / 8 + std::min<uint64_t>(64, r / 2 + 1);
      dr.base[k] = h[0] > INT64_MIN + (long long)margin ? h[0] - (long long)margin : INT64_MIN;
      dr.span[k] = r + 2 * margin;
      nonnull = std::max(nonnull, h[2]);
    }
    const unsigned __int128 entries = (unsigned __int128)dr.span[0] * dr.span[1];
    const uint64_t budget = 8 * (uint64_t)std::max<int64_t>(std::max<int64_t>(nonnull, cx.conf.agg_initial_groups), 1 << 16);
    if (entries > budget || entries > ((uint64_t)1 << 26)) return false;               // sparse keys: stay on the hash table
    if (cx.conf.agg_max_table_bytes > 0 && entries * entry_words * 8 > (unsigned __int128)cx.conf.agg_max_table_bytes) return false;
    dr.entries = (uint64_t)entries;
    // do a few keys dominate the sample?  one hash bucket holds > 0.4 % of the rows
    dr.hot = probe_skew && dr.entries * entry_words > 4096 && (uint64_t)mx * 256 > (uint64_t)sample;
    return true;
  }

  void decide_wide(OpContext& cx, const ColTable& ct, int64_t n) {
    dense_decided_ = true;
    if (!wide_possible_ || n == 0) { wide_possible_ = false; return; }
    DenseRange dr;
    if (!dense_range(cx, ct, n, ws_.nkeys, ws_.key_col, ws_.key_phys, ws_.G, false, dr)) { wide_possible_ = false; return; }
    ws_.dense_base = dr.base[0]; ws_.dense_cap0 = dr.span[0]; ws_.dense_base1 = dr.base[1]; ws_.dense_r1 = dr.span[1]; ws_.dense_cap = dr.entries;
    dense_tab_ = DevMem::alloc((size_t)ws_.dense_cap * ws_.G * 8, cx.stream);
    ws_.dense_tab = (unsigned long long*)dense_tab_->ptr;
    cx.m.launches += launch_tile_wide_init(ws_, cx.stream);
  }

  // dense entry layout (2 or 4 words): [row counter unless a COUNT(*) accumulator doubles as the presence marker]
  // [accumulators] [one "valid arguments" counter per nullable SUM that has no COUNT over the same column beside it]
  bool dense_layout() {
    int star = -1;
    for (int j = 0; j < lay_.nacc; j++) if (fs_.acc[j].kind == FAST_ACC_COUNT && fs_.acc[j].col < 0) star = j;
    int word_of_acc[2] = {0, 0}, valid_word_of_acc[2] = {0xFF, 0xFF}, w = 0;
    for (int i = 0; i < 4; i++) fs_.dense_word_src[i] = -2;
    int8_t src[8]; for (int i = 0; i < 8; i++) src[i] = -2;
    if (star < 0) src[w++] = -1;
    for (int j = 0; j < lay_.nacc; j++) { word_of_acc[j] = w; src[w++] = (int8_t)j; }
    for (int j = 0; j < lay_.nacc; j++) {
      if (fs_.acc[j].kind != FAST_ACC_ADD || fs_.acc[j].vbit == 0xFF) continue;
      for (int i = 0; i < lay_.nacc; i++) if (i != j && fs_.acc[i].kind == FAST_ACC_COUNT && fs_.acc[i].col == fs_.acc[j].col) valid_word_of_acc[j] = word_of_acc[i];
      // a never-NULL argument: the SUM has a value as soon as the entry holds a row
      if (valid_word_of_acc[j] == 0xFF && !acc_arg_nullable_[j]) valid_word_of_acc[j] = star >= 0 ? word_of_acc[star] : 0;
      if (valid_word_of_acc[j] == 0xFF) { valid_word_of_acc[j] = w; src[w++] = (int8_t)(2 + j); }
    }
    if (w > 4) return false;
    fs_.dense_stride = w <= 2 ? 2 : 4;
    for (int i = 0; i < 4; i++) fs_.dense_word_src[i] = src[i];
    fs_.dense_presence_word = (uint8_t)(star >= 0 ? word_of_acc[star] : 0);
    for (size_t c = 0; c < emit_.size(); c++) {
      dmap_.word[c] = 0; dmap_.valid_word[c] = 0xFF;
      const EmitCol& ec = emit_[c].ec;
      if (ec.kind == EMIT_KEY) continue;
      int j = 0; for (int i = 0; i < lay_.nacc; i++) if (fs_.acc[i].word == ec.word) j = i;
      dmap_.word[c] = (uint8_t)word_of_acc[j];
      if (ec.vbit != 0xFF) dmap_.valid_word[c] = (uint8_t)valid_word_of_acc[j];
    }
    return true;
  }

  // decide DENSE mode from the key range of (a sample of) the first batch; dense_layout() already ran in detect_fast
  void decide_dense(OpContext& cx, const ColTable& ct, int64_t n) {
    dense_decided_ = true;
    if (!fast_ok_ || !dense_possible_ || n == 0) return;
    DenseRange dr;
    if (!dense_range(cx, ct, n, fs_.nkeys, fs_.key_col, fs_.key_phys, fs_.dense_stride, cx.conf.agg_hot_key_cache != 0, dr)) return;
    fs_.dense_base = dr.base[0]; fs_.dense_cap0 = dr.span[0];
    fs_.dense_base1 = dr.base[1]; fs_.dense_r1 = dr.span[1];
    fs_.dense_cap = dr.entries;
    // the key with the shorter span indexes the rows of the table: short rows would interleave the dead entries of their
    // margins with the live ones in every cache line (M2: 163,968 x 20 entries, 52 MB, whose live third then no longer
    // stays in L2 beside the input stream; as 20 rows of 163,968 the live entries are 8 runs of 2 MB)
    fs_.dense_key0_minor = fs_.nkeys == 2 && dr.span[1] < dr.span[0];
    dense_tab_ = DevMem::alloc((size_t)fs_.dense_cap * fs_.dense_stride * 8, cx.stream, true);
    fs_.dense_tab = (unsigned long long*)dense_tab_->ptr;
    fs_.dense = 1;
    fs_.hot_cache = dr.hot ? 1 : 0;
  }

  // LEAN kernels: every referenced column is a non-null, 32-byte aligned int64 column
  bool lean_ok(const ColTable& ct, int64_t begin) const {
    if (begin % 4) return false;
    auto ok = [&](int slot, uint8_t phys) {
      const DevCol& c = ct.col[slot];
      return phys == PH_I64 && c.validity == nullptr && ((uintptr_t)c.values & 31) == 0;
    };
    for (int k = 0; k < fs_.nkeys; k++) if (!ok(fs_.key_col[k], fs_.key_phys[k])) return false;
    for (int j = 0; j < fs_.nacc; j++) {
      if (fs_.acc[j].col < 0) continue;
      if (fs_.acc[j].kind == FAST_ACC_ADD) { if (!ok(fs_.acc[j].col, fs_.acc[j].phys)) return false; }
      else if (ct.col[fs_.acc[j].col].validity != nullptr) return false;       // COUNT(col): needs no data, only "no NULLs"
    }
    for (int f = 0; f < fs_.nfilt; f++) if (!ok(fs_.filt[f].col, fs_.filt[f].phys)) return false;
    return true;
  }

  int launch_update(OpContext& cx, const ColTable& ct, const AggTable& t, int64_t begin, int64_t m, const uint32_t* list) {
    if (nsets_ > 1) return launch_agg_update_sets((const VmProgram*)d_prog_->ptr, ct, lay_, t, begin, m, list, (const AggSetDesc*)d_sets_->ptr, nsets_, cx.stream);
    // deferred-row replays (arbitrary row lists, rare) always take the generic kernel: same table, same semantics
    if (wide_possible_ && ws_.dense_tab && !list) {
      cx.m.fast_launches++;
      if (ws_.dec_word != 0xFF) {                                    // carry-free decimal pieces: normalise before 2^31 rows could have met in one entry
        if (wide_rows_since_norm_ + m > (1LL << 31)) { cx.m.launches += launch_tile_wide_normalise(ws_, cx.stream); wide_rows_since_norm_ = 0; }
        wide_rows_since_norm_ += m;
      }
      return launch_agg_tile_wide(ct, ws_, lay_, t, begin, m, cx.stream);
    }
    if (fast_ok_ && !list) {
      cx.m.fast_launches++;
      FastSpec fs = fs_;
      fs.lean = lean_ok(ct, begin) ? 1 : 0;
      return launch_agg_fast_update(ct, fs, lay_, t, begin, m, cx.stream);
    }
    return launch_agg_update((const VmProgram*)d_prog_->ptr, ct, lay_, t, begin, m, list, cx.stream);
  }

  // A12: the GPU table never spills; when it would outgrow its HBM budget (b200q_conf.agg_max_table_bytes, or the
  // device itself) the op returns B200Q_ERR_UNSUPPORTED and the host falls back (INTEGRATION.md §3)
  void check_table_budget(OpContext& cx, unsigned __int128 bytes, const char* what) const {
    const int64_t budget = cx.conf.agg_max_table_bytes;
    if (budget > 0 && bytes > (unsigned __int128)budget)
      throw ExecError(B200Q_ERR_UNSUPPORTED, std::string("aggregate ") + what + " of " + std::to_string((unsigned long long)bytes) + " bytes exceeds the HBM budget (agg_max_table_bytes = " +
                                                 std::to_string(budget) + "): the table cannot spill on the GPU, fall back to the host path (agg_table.rs:540-588)");
  }
  void alloc_table(OpContext& cx, uint64_t cap, DevMemP& keys, DevMemP& accs, DevMemP& counters) {
    check_table_budget(cx, (unsigned __int128)cap * (lay_.kstride + lay_.astride) * 8, "hash table");
    keys = DevMem::alloc((size_t)cap * lay_.kstride * 8, cx.stream, true);
    accs = DevMem::alloc((size_t)cap * lay_.astride * 8, cx.stream);       // initialised at insertion
    counters = DevMem::alloc(64, cx.stream, true);
  }

  // no-grouping aggregation always yields exactly one row (agg_exec.rs:280-323): pre-insert the empty key
  void seed_global_group(OpContext& cx) {
    const uint64_t h = host_mix64(0x9E3779B97F4A7C15ULL);        // == agg_hash_words(nullptr, 0, 0)
    const uint64_t s = ((h >> 32) * (uint64_t)(uint32_t)capacity_) >> 32;          // == agg_first_slot
    const uint32_t tag2 = (uint32_t)h | 0x80000000u;                             // == agg_tag
    std::vector<uint64_t> kimg(lay_.kstride, 0), aimg(lay_.astride, 0);
    for (int i = 0; i < lay_.astride; i++) aimg[i] = lay_.init[i];
    kimg[0] = (uint64_t)tag2 | ((uint64_t)lay_.init_flags << 32);
    B200Q_CUDA(cudaMemcpyAsync((uint8_t*)keys_->ptr + s * lay_.kstride * 8, kimg.data(), kimg.size() * 8, cudaMemcpyHostToDevice, cx.stream));
    B200Q_CUDA(cudaMemcpyAsync((uint8_t*)accs_->ptr + s * lay_.astride * 8, aimg.data(), aimg.size() * 8, cudaMemcpyHostToDevice, cx.stream));
    const unsigned long long one = 1;
    B200Q_CUDA(cudaMemcpyAsync(counters_->ptr, &one, 8, cudaMemcpyHostToDevice, cx.stream));
    B200Q_CUDA(cudaStreamSynchronize(cx.stream));
  }

  // probe chains cost one dependent L2 round trip per extra slot: the table is kept at most half full (measured on
  // M1-hash: load 0.3 -> 6.7e10 rows/s, load 0.6 -> 5.6e10; only the sectors holding occupied slots are L2-resident)
  static constexpr double AGG_SLOTS_PER_GROUP = 3.0, AGG_LOAD_LIMIT = 0.5;
  static uint64_t load_limit(uint64_t cap) {
    const uint64_t lim = (uint64_t)((double)cap * AGG_LOAD_LIMIT);
    return cap > (1ULL << 19) ? std::min<uint64_t>(lim, cap - (1ULL << 19)) : lim;      // slack above the limit > the concurrent-insert overshoot bound (resident threads)
  }

  AggTable table_view(int deferred_idx) const {
    AggTable t{};
    t.keys = (unsigned long long*)keys_->ptr; t.accs = (unsigned long long*)accs_->ptr; t.capacity = capacity_; t.max_groups = load_limit(capacity_);
    t.counters = (unsigned long long*)counters_->ptr;
    t.deferred = deferred_[deferred_idx] ? (uint32_t*)deferred_[deferred_idx]->ptr : nullptr;
    return t;
  }

  void grow(OpContext& cx, uint64_t min_groups) {
    uint64_t cap = capacity_;
    do cap <<= 1; while (load_limit(cap) < min_groups);
    if (cap >= (1ULL << 32)) throw ExecError(B200Q_ERR_UNSUPPORTED, "aggregate hash table beyond 2^32 slots");
    DevMemP nkeys, naccs, ncounters;
    alloc_table(cx, cap, nkeys, naccs, ncounters);
    AggTable oldt = table_view(0);
    AggTable newt{}; newt.keys = (unsigned long long*)nkeys->ptr; newt.accs = (unsigned long long*)naccs->ptr; newt.capacity = cap; newt.max_groups = load_limit(cap); newt.counters = (unsigned long long*)ncounters->ptr;
    cx.m.launches += launch_agg_rehash(lay_, oldt, newt, cx.stream);
    B200Q_CUDA(cudaGetLastError());
    keys_ = nkeys; accs_ = naccs; counters_ = ncounters; capacity_ = cap;
    cx.m.grow_count++; cx.m.table_capacity = (int64_t)cap;
  }

  void read_counters(OpContext& cx, unsigned long long (&h)[3]) {
    B200Q_CUDA(cudaMemcpyAsync(h, counters_->ptr, 24, cudaMemcpyDeviceToHost, cx.stream));
    B200Q_CUDA(cudaStreamSynchronize(cx.stream));
    check_device_error_flags((int)h[2]);
    ngroups_ = (int64_t)h[0];
    cx.m.num_groups = ngroups_;
  }

  // The counters of a chunk (groups, deferred rows, error flags) are copied into a pinned snapshot right behind its kernel and read
  // while the NEXT chunk's kernel already runs: no host round trip between the launches of a batch.
  struct Snap { unsigned long long* h = nullptr; cudaEvent_t ready = nullptr, k0 = nullptr, k1 = nullptr; };
  Snap snap_[2];
 public:
  ~AggStage() override { for (auto& s : snap_) { if (s.h) pinned_slots().put(s.h); if (s.ready) cudaEventDestroy(s.ready); if (s.k0) cudaEventDestroy(s.k0); if (s.k1) cudaEventDestroy(s.k1); } }
  void ensure_snaps() {
    if (snap_[0].h) return;
    for (auto& s : snap_) {
      s.h = pinned_slots().get();
      B200Q_CUDA(cudaEventCreateWithFlags(&s.ready, cudaEventDisableTiming)); B200Q_CUDA(cudaEventCreate(&s.k0)); B200Q_CUDA(cudaEventCreate(&s.k1));
    }
  }
  void account(OpContext& cx, const Snap& s, int64_t rows) {
    float ms = 0; B200Q_CUDA(cudaEventElapsedTime(&ms, s.k0, s.k1));
    cx.m.gpu_ms += ms; if (cx.cur_stage == 0) { cx.m.hot_ms += ms; cx.m.hot_rows += rows; cx.m.hot_launches++; }
  }
  // rows of [begin, ...) that could not be inserted (the table was at its load limit): grow, then replay only those rows
  void replay(OpContext& cx, const ColTable& ct, int64_t begin, const uint32_t* list, uint64_t ndef, bool grow_first) {
    // new deferrals go to the buffer the list does not live in; the second buffer only exists once a replay needs it (the slow path is rare, and
    // a buffer is 8 bytes per row of a launch)
    if (!deferred_[1] || deferred_[1]->bytes < (size_t)deferred_cap_ * 4) deferred_[1] = DevMem::alloc((size_t)deferred_cap_ * 4, cx.stream);
    int wr = list == (const uint32_t*)deferred_[0]->ptr ? 1 : 0;
    while (ndef > 0) {
      if (grow_first) grow(cx, (uint64_t)ngroups_ + ndef);
      grow_first = true;
      B200Q_CUDA(cudaMemsetAsync((uint8_t*)counters_->ptr + 8, 0, 8, cx.stream));
      cx.m.launches += launch_update(cx, ct, table_view(wr), begin, (int64_t)ndef, list);
      B200Q_CUDA(cudaGetLastError());
      unsigned long long h[3];
      read_counters(cx, h);
      ndef = h[1]; list = (const uint32_t*)deferred_[wr]->ptr; wr ^= 1;
    }
  }

  void update_rows(OpContext& cx, const ColTable& ct, int64_t n) {
    int64_t chunk = std::max<int64_t>(1 << 16, std::min<int64_t>(cx.conf.max_launch_rows, 0x7FFFFFFFLL));
    // grouping sets: a launch inserts rows x sets keys; its rows are clamped so that a deferred entry (row * nsets + set) fits in 32 bits
    // and the deferred buffers stay as large as a single-set launch of `chunk` rows would make them
    if (nsets_ > 1) chunk = std::max<int64_t>(1 << 16, chunk / nsets_);
    static const bool dbg = getenv("B200Q_AGG_TIMING") != nullptr;
    auto hnow = [] { return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now().time_since_epoch()).count(); };
    const double tA = hnow();
    ensure_snaps();
    const double tB = hnow();
    const int64_t m_max = std::min(chunk, n);
    if (deferred_cap_ < 2 * m_max * nsets_) {                             // two chunks' worth: a chunk is launched before the counters of the one before it are back
      deferred_cap_ = 2 * m_max * nsets_;
      deferred_[0] = DevMem::alloc((size_t)deferred_cap_ * 4, cx.stream);
      deferred_[1] = nullptr;
    }
    const double tC = hnow(); double t_launch = 0, t_settle = 0;
    int64_t prev_begin = 0, prev_m = 0; bool have_prev = false;
    int idx = 0;
    // settles the chunk whose snapshot is snap_[pi]; `cur` (when >= 0): the chunk launched behind it, whose snapshot is snap_[pi ^ 1]
    auto settle = [&](int pi, int64_t pb, int64_t pm, bool cur_in_flight, int64_t cb, int64_t cm) -> bool {
      Snap& sp = snap_[pi];
      B200Q_CUDA(cudaEventSynchronize(sp.ready));
      account(cx, sp, pm);
      check_device_error_flags((int)sp.h[2]);
      ngroups_ = (int64_t)sp.h[0]; cx.m.num_groups = ngroups_;
      const uint64_t d_prev = sp.h[1];
      if (d_prev == 0) return false;
      // slow path: the table hit its load limit.  The chunk behind (if any) appended its own deferred rows after ours.
      uint64_t d_cur = 0; DevMemP list_cur;
      if (cur_in_flight) {
        Snap& sc = snap_[pi ^ 1];
        B200Q_CUDA(cudaEventSynchronize(sc.ready));
        account(cx, sc, cm);
        check_device_error_flags((int)sc.h[2]);
        ngroups_ = (int64_t)sc.h[0]; cx.m.num_groups = ngroups_;
        d_cur = sc.h[1] - d_prev;
        if (d_cur) { list_cur = DevMem::alloc((size_t)d_cur * 4, cx.stream); B200Q_CUDA(cudaMemcpyAsync(list_cur->ptr, (const uint32_t*)deferred_[0]->ptr + d_prev, (size_t)d_cur * 4, cudaMemcpyDeviceToDevice, cx.stream)); }
      }
      replay(cx, ct, pb, (const uint32_t*)deferred_[0]->ptr, d_prev, true);
      if (d_cur) replay(cx, ct, cb, (const uint32_t*)list_cur->ptr, d_cur, false);
      return true;
    };
    for (int64_t begin = 0; begin < n; begin += chunk, idx++) {
      const int64_t m = std::min(chunk, n - begin);
      Snap& s = snap_[idx & 1];
      const double tl = hnow();
      B200Q_CUDA(cudaEventRecord(s.k0, cx.stream));
      cx.m.launches += launch_update(cx, ct, table_view(0), begin, m, nullptr);
      B200Q_CUDA(cudaEventRecord(s.k1, cx.stream));
      B200Q_CUDA(cudaGetLastError());
      B200Q_CUDA(cudaMemcpyAsync(s.h, counters_->ptr, 24, cudaMemcpyDeviceToHost, cx.stream));
      B200Q_CUDA(cudaEventRecord(s.ready, cx.stream));
      const double ts = hnow(); t_launch += ts - tl;
      const bool slow = have_prev && settle((idx & 1) ^ 1, prev_begin, prev_m, true, begin, m);
      t_settle += hnow() - ts;
      if (slow) { have_prev = false; continue; }                          // the slow path settled this chunk too
      prev_begin = begin; prev_m = m; have_prev = true;
    }
    const double tD = hnow();
    if (have_prev) settle((idx & 1) ^ 1, prev_begin, prev_m, false, 0, 0);
    if (dbg) fprintf(stderr, "update_rows: snaps %.3f ms, deferred buffers %.3f ms, launches %.3f ms, settles %.3f ms, last settle %.3f ms (%d chunks)\n", tB - tA, tC - tB, t_launch, t_settle, hnow() - tD, idx);
  }

  void push(OpContext& cx, DevBatch& in, std::vector<DevBatch>&) override {
    const int64_t n = in.num_rows;
    if (n == 0) return;
    ColTable ct{};
    std::vector<DevColumn> state_cols;
    if (merge_mode_ && !columnar_) unfreeze(cx, in, state_cols);
    for (size_t i = 0; i < cp_.used_cols.size(); i++) {
      const int c = cp_.used_cols[i];
      ct.col[i] = dev_col_of(c < n_in_ ? in.cols[c] : state_cols[c - n_in_]);
    }
    if (!dense_decided_) { if (wide_possible_) decide_wide(cx, ct, n); else decide_dense(cx, ct, n); }
    update_rows(cx, ct, n);
  }

  // Binary agg-buffer column -> typed state columns (AccColumn::unfreeze_from_rows, agg_ctx.rs:276-296)
  void unfreeze(OpContext& cx, DevBatch& in, std::vector<DevColumn>& state_cols) {
    const int64_t n = in.num_rows;
    const DevColumn& bc = in.cols.back();
    if (!bc.offsets || !bc.values) throw ExecError(B200Q_ERR_INVALID_ARG, "agg buffer column without offsets/data");
    FrozenTable ft{}; ft.nfields = (int)merge_state_fields_.size();
    if (ft.nfields > FROZEN_MAX_FIELDS) throw ExecError(B200Q_ERR_UNSUPPORTED, "too many accumulator fields");
    std::vector<DevMemP> valid_bytes(ft.nfields);
    for (int k = 0; k < ft.nfields; k++) {
      const FieldDef& f = merge_state_fields_[k];
      DevColumn c; c.type = f.type; c.values = DevMem::alloc((size_t)n * f.type.byte_width(), cx.stream);
      FrozenField& ff = ft.f[k];
      ff.kind = f.nullable ? FZ_PRIM : FZ_COUNT; ff.width = frozen_width(f.type); ff.phys = phys_of(f.type); ff.values = c.values->ptr;
      if (f.nullable) { valid_bytes[k] = DevMem::alloc((size_t)n, cx.stream); ff.valid = (const uint8_t*)valid_bytes[k]->ptr; c.validity = DevMem::alloc(bitmap_bytes(n), cx.stream); }
      state_cols.push_back(c);
    }
    int* d_err = (int*)((unsigned long long*)counters_->ptr + 2);
    cx.m.launches += launch_frozen_read(ft, n, (const int32_t*)bc.offsets->ptr, bc.offset, (const uint8_t*)bc.values->ptr, d_err, cx.stream);
    for (int k = 0; k < ft.nfields; k++)
      if (valid_bytes[k]) cx.m.launches += launch_pack_valid((const uint8_t*)valid_bytes[k]->ptr, (uint32_t*)state_cols[k].validity->ptr, n, cx.stream);
    B200Q_CUDA(cudaGetLastError());
    // valid_bytes buffers are released stream-ordered after the pack kernels
  }

  void finish(OpContext& cx, std::vector<DevBatch>& outs) override {
    // ONE host round trip for the group counts: the hash table's counters and the occupied entries of the dense / wide table land in one pinned slot
    const bool wide = wide_possible_ && ws_.dense_tab;
    ensure_snaps();
    unsigned long long* hs = snap_[0].h;
    DevMemP dc;
    if (fs_.dense || wide) {
      dc = DevMem::alloc(8, cx.stream, true);
      if (wide) cx.m.launches += launch_tile_wide_normalise(ws_, cx.stream);
      cx.m.launches += fs_.dense ? launch_dense_count(fs_, (unsigned long long*)dc->ptr, cx.stream) : launch_tile_wide_count(ws_, (unsigned long long*)dc->ptr, cx.stream);
      B200Q_CUDA(cudaMemcpyAsync(hs + 3, dc->ptr, 8, cudaMemcpyDeviceToHost, cx.stream));
    } else hs[3] = 0;
    B200Q_CUDA(cudaMemcpyAsync(hs, counters_->ptr, 24, cudaMemcpyDeviceToHost, cx.stream));
    B200Q_CUDA(cudaStreamSynchronize(cx.stream));
    check_device_error_flags((int)hs[2]);
    ngroups_ = (int64_t)hs[0];
    const int64_t g = ngroups_ + (int64_t)hs[3];
    cx.m.num_groups = g;
    if (g == 0) return;                                             // no records (agg_table.rs:154-156)
    EmitTable et{}; et.ncols = (int)emit_.size();
    if (et.ncols > EMIT_MAX_COLS) throw ExecError(B200Q_ERR_UNSUPPORTED, "too many output columns");
    DevBatch ob; ob.num_rows = g;
    std::vector<DevMemP> valid_bytes(emit_.size()), bool_bytes(emit_.size());
    for (size_t i = 0; i < emit_.size(); i++) {
      EmitCol ec = emit_[i].ec; const FieldDef& f = emit_[i].field;
      DevColumn c; c.type = f.type;
      if (f.type.id == T_BOOL) { bool_bytes[i] = DevMem::alloc((size_t)g, cx.stream); ec.values = bool_bytes[i]->ptr; c.values = DevMem::alloc(bitmap_bytes(g), cx.stream); }
      else { c.values = DevMem::alloc((size_t)g * f.type.byte_width(), cx.stream); ec.values = c.values->ptr; }
      if (f.nullable) { valid_bytes[i] = DevMem::alloc((size_t)g, cx.stream); ec.valid_bytes = (uint8_t*)valid_bytes[i]->ptr; c.validity = DevMem::alloc(bitmap_bytes(g), cx.stream); }
      et.col[i] = ec;
      ob.cols.push_back(c);
    }
    DevMemP out_count = DevMem::alloc(8, cx.stream, true);
    cx.m.launches += launch_agg_emit(lay_, table_view(0), et, (unsigned long long*)out_count->ptr, cx.stream);
    if (fs_.dense) cx.m.launches += launch_agg_emit_dense(fs_, et, dmap_, (unsigned long long*)out_count->ptr, cx.stream);
    if (wide) cx.m.launches += launch_tile_wide_emit(ws_, lay_, et, (unsigned long long*)out_count->ptr, cx.stream);
    for (size_t i = 0; i < emit_.size(); i++) {
      if (valid_bytes[i]) cx.m.launches += launch_pack_valid((const uint8_t*)valid_bytes[i]->ptr, (uint32_t*)ob.cols[i].validity->ptr, g, cx.stream);
      if (bool_bytes[i]) cx.m.launches += launch_pack_valid((const uint8_t*)bool_bytes[i]->ptr, (uint32_t*)ob.cols[i].values->ptr, g, cx.stream);
    }
    B200Q_CUDA(cudaGetLastError());
    if (!final_ && !columnar_) {
      // freeze the state columns into the reference's Binary agg-buffer column (freeze_acc_table, agg_ctx.rs:407-426)
      FrozenTable ft{}; ft.nfields = (int)frozen_fields_.size();
      for (int k = 0; k < ft.nfields; k++) {
        ft.f[k] = frozen_fields_[k];
        ft.f[k].values = ob.cols[lay_.nkeys + k].values->ptr;
        ft.f[k].valid = valid_bytes[lay_.nkeys + k] ? (const uint8_t*)valid_bytes[lay_.nkeys + k]->ptr : nullptr;
      }
      DevMemP lengths = DevMem::alloc((size_t)g * 4, cx.stream);
      DevMemP offsets = DevMem::alloc((size_t)(g + 1) * 4, cx.stream);
      DevMemP block_sums = DevMem::alloc((size_t)scan_num_blocks(g) * 4 + 16, cx.stream);
      cx.m.launches += launch_frozen_lengths(ft, g, (int32_t*)lengths->ptr, cx.stream);
      cx.m.launches += launch_exclusive_scan_i32((const int32_t*)lengths->ptr, (int32_t*)offsets->ptr, g, (int32_t*)block_sums->ptr, cx.stream);
      int32_t total = 0;
      B200Q_CUDA(cudaMemcpyAsync(&total, (int32_t*)offsets->ptr + g, 4, cudaMemcpyDeviceToHost, cx.stream));
      B200Q_CUDA(cudaStreamSynchronize(cx.stream));
      if (total < 0) throw ExecError(B200Q_ERR_UNSUPPORTED, "frozen accumulator column exceeds 2 GiB; emit in smaller batches");
      DevMemP data = DevMem::alloc((size_t)total, cx.stream);
      cx.m.launches += launch_frozen_write(ft, g, (const int32_t*)offsets->ptr, (uint8_t*)data->ptr, cx.stream);
      B200Q_CUDA(cudaGetLastError());
      DevColumn bc; bc.type.id = T_BINARY; bc.values = data; bc.offsets = offsets;
      ob.cols.resize(lay_.nkeys);
      ob.cols.push_back(bc);
    }
    B200Q_CUDA(cudaStreamSynchronize(cx.stream));
    outs.push_back(std::move(ob));
  }
};

std::unique_ptr<Stage> make_agg_stage(OpContext& cx, const SchemaDef& in_schema, const std::vector<ExprP>& filters, const PlanNode& agg,
                                      const std::vector<ExprP>& group_exprs, const std::vector<std::vector<ExprP>>& agg_args,
                                      const std::vector<AggSetExprs>& sets) {
  return std::unique_ptr<Stage>(new AggStage(cx, in_schema, filters, agg, group_exprs, agg_args, sets));
}

}  // namespace b200q
