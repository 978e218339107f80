// SortMergeJoinStage: SortMergeJoinExecNode (DESIGN.md §3.14).
//
// Reference (paths relative to the reference's native-engine/datafusion-ext-plans/src/): SortMergeJoinExec::execute
// sort_merge_join_exec.rs:200-330 (both children streamed in key order through one of the joiners of joins/smj/*.rs),
// compare_cursor! :357-365 (a key with a NULL never matches; outer / anti / existence forms still emit its row).
// Shape on the GPU: the op's pushed input is the LEFT child (usually the rows a SortExec below it emits); the RIGHT child runs as
// its own op and its queued device batches are attached by reference (b200q_op_attach_right), normalised and checked once.
// Every pushed left batch is joined at once against the whole right side (kernels_merge.cu): normalise + sortedness check, merge
// path co-ranking, counts, 64-bit scan, pair emission in output order, and one gather per 16 columns of each side.  For Right /
// Full joins, right rows whose key sorts strictly before the batch's last left key are settled by that batch: its unmatched ones
// are merged into the batch's output at their key position; the others wait for a later batch or for finish().
#include <cstring>

#include "kernels_join.cuh"
#include "kernels_merge.cuh"
#include "runtime.h"

namespace b200q {

namespace {

enum { SJ_INNER = 0, SJ_LEFT, SJ_RIGHT, SJ_FULL, SJ_SEMI, SJ_ANTI, SJ_EXISTENCE };   // protobuf JoinType (auron.proto:475-483)

SortKeyCol key_col(const DType& t, const void* values, const uint8_t* vbits, uint32_t bit_offset, const uint8_t* vbytes, const PlanNode::SortOptionsDef& o) {
  SortKeyCol k{};
  k.values = values; k.valid_bytes = vbytes; k.valid_bits = vbytes ? nullptr : vbits; k.bit_offset = bit_offset;
  k.phys = (uint8_t)phys_of(t); k.descending = !o.asc; k.nulls_first = o.nulls_first; k.dec_word = 0;
  const int w = t.byte_width();
  k.mask = w >= 8 ? ~0ull : ((1ull << (8 * w)) - 1);
  return k;
}

class SmjStage : public Stage, public SmjRightAttach {
  int jt_;
  SchemaDef left_, right_;
  std::vector<int> lkeys_, rkeys_;
  std::vector<PlanNode::SortOptionsDef> opts_;
  bool left_outer_, right_outer_, semi_like_;
  // the right side, after attach
  bool attached_ = false;
  int64_t m_ = 0;
  std::vector<GatherSrc> rsrc_;                      // its columns as gather sources
  std::vector<DevMemP> rkeep_;                       // the allocations they point into
  DevMemP rw0_, rw1_, rflags_, matched_;
  // the left stream
  DevMemP carry_, status_, zero_;
  int64_t settled_ = 0;                              // right rows [0, settled_) have been settled (Right / Full)

  MergeKeys right_keys() const { return MergeKeys{(const unsigned long long*)rw0_->ptr, rw1_ ? (const unsigned long long*)rw1_->ptr : nullptr, (const uint8_t*)rflags_->ptr}; }

  SmjStatus read_status(OpContext& cx) {
    SmjStatus st{};
    B200Q_CUDA(cudaMemcpyAsync(&st, status_->ptr, sizeof(st), cudaMemcpyDeviceToHost, cx.stream));
    B200Q_CUDA(cudaStreamSynchronize(cx.stream));
    return st;
  }
  unsigned long long read_word(OpContext& cx, const void* p) {
    unsigned long long v = 0;
    B200Q_CUDA(cudaMemcpyAsync(&v, p, 8, cudaMemcpyDeviceToHost, cx.stream));
    B200Q_CUDA(cudaStreamSynchronize(cx.stream));
    return v;
  }
  // exclusive scan of n u64 -> out (n + 1 words)
  DevMemP scan(OpContext& cx, const DevMemP& in, int64_t n) {
    DevMemP out = DevMem::alloc((size_t)(n + 1) * 8, cx.stream), tmp = DevMem::alloc((size_t)smj_scan_tmp_words(n) * 8 + 16, cx.stream);
    cx.m.launches += launch_smj_scan(in ? (const unsigned long long*)in->ptr : nullptr, (unsigned long long*)out->ptr, n, (unsigned long long*)tmp->ptr, cx.stream);
    return out;
  }

 public:
  SmjStage(OpContext& cx, const SchemaDef& in, const PlanNode& node) {
    jt_ = node.join_type; left_ = node.join_left_schema; right_ = node.join_right_schema; opts_ = node.smj_sort_options;
    in_schema = in; out_schema = node.schema;
    for (auto& p : node.join_on) { lkeys_.push_back(p.first->col_index); rkeys_.push_back(p.second->col_index); }
    left_outer_ = jt_ == SJ_LEFT || jt_ == SJ_FULL;
    right_outer_ = jt_ == SJ_RIGHT || jt_ == SJ_FULL;
    semi_like_ = jt_ >= SJ_SEMI;
    if (in.fields.size() != left_.fields.size()) throw PlanError(B200Q_ERR_INVALID_PLAN, "SortMergeJoinExec: the left input does not have the left schema");
    for (size_t i = 0; i < in.fields.size(); i++) used_input_cols.push_back((int)i);
    carry_ = DevMem::alloc(sizeof(SmjCarry), cx.stream, true);
    status_ = DevMem::alloc(sizeof(SmjStatus), cx.stream, true);
    zero_ = DevMem::alloc(16, cx.stream, true);
  }

  bool right_attached() const override { return attached_; }

  void attach_right(OpContext& cx, const std::vector<DevBatch>& batches, const SchemaDef& schema) override {
    if (attached_) throw ExecError(B200Q_ERR_STATE, "attach_right: a right side is already attached");
    if (schema.fields.size() != right_.fields.size()) throw ExecError(B200Q_ERR_INVALID_ARG, "attach_right: the right op's schema does not match the join's right side");
    for (size_t i = 0; i < schema.fields.size(); i++)
      if (schema.fields[i].type != right_.fields[i].type) throw ExecError(B200Q_ERR_INVALID_ARG, "attach_right: type of right column " + std::to_string(i) + " differs");
    std::vector<const DevBatch*> parts;
    int64_t m = 0;
    for (auto& b : batches) if (b.num_rows > 0) { parts.push_back(&b); m += b.num_rows; }
    if (m >= (1LL << 31)) throw ExecError(B200Q_ERR_UNSUPPORTED, "SortMergeJoinExec: the right side has 2^31 rows or more");
    const size_t ncols = right_.fields.size();
    std::vector<GatherSrc> src(ncols);
    std::vector<DevMemP> keep;
    for (size_t c = 0; c < ncols; c++) src[c] = GatherSrc{right_.fields[c].type, nullptr, nullptr, 0, nullptr, false};
    if (parts.size() == 1) {                        // one batch (what a SortExec emits): used where it lies
      for (size_t c = 0; c < ncols; c++) {
        const DevColumn& dc = parts[0]->cols[c];
        src[c] = gather_src_of(dc, false); keep.push_back(dc.values);
        if (dc.validity) keep.push_back(dc.validity);
      }
    } else if (parts.size() > 1) {                  // several: concatenated once, validity as one byte per row
      const ByteCols bc = to_byte_cols(cx, right_, parts);
      for (size_t c = 0; c < ncols; c++) {
        src[c].values = bc.values[c]->ptr; keep.push_back(bc.values[c]);
        if (bc.valid[c]) { src[c].vbytes = (const uint8_t*)bc.valid[c]->ptr; src[c].may_be_null = true; keep.push_back(bc.valid[c]); }
      }
    }
    // normalise the right keys once and check their order
    const int nk = (int)rkeys_.size();
    DevMemP w0 = DevMem::alloc((size_t)m * 8 + 16, cx.stream), w1 = nk > 1 ? DevMem::alloc((size_t)m * 8 + 16, cx.stream) : nullptr, fl = DevMem::alloc((size_t)m + 16, cx.stream);
    SortKeyCol kc[2];
    for (int i = 0; i < nk; i++) { const GatherSrc& g = src[(size_t)rkeys_[(size_t)i]]; kc[i] = key_col(g.type, g.values, g.vbits, g.bit_offset, g.vbytes, opts_[(size_t)i]); }
    B200Q_CUDA(cudaMemsetAsync(status_->ptr, 0, sizeof(SmjStatus), cx.stream));
    cx.m.launches += launch_smj_normalise(kc, nk, m, (unsigned long long*)w0->ptr, w1 ? (unsigned long long*)w1->ptr : nullptr, (uint8_t*)fl->ptr, nullptr, (SmjStatus*)status_->ptr, cx.stream);
    if (read_status(cx).unsorted) throw ExecError(B200Q_ERR_INVALID_ARG, "SortMergeJoinExec: the right input not sorted by the join keys under the node's sort_options");
    rsrc_ = src; rkeep_ = keep; rw0_ = w0; rw1_ = w1; rflags_ = fl; m_ = m;
    if (right_outer_) matched_ = DevMem::alloc((size_t)m + 16, cx.stream, true);
    B200Q_CUDA(cudaStreamSynchronize(cx.stream));
    attached_ = true;
  }

  void push(OpContext& cx, DevBatch& in, std::vector<DevBatch>& outs) override {
    if (!attached_) throw ExecError(B200Q_ERR_STATE, "SortMergeJoinExec: no right side attached (b200q_op_attach_right) before the first left batch");
    for_each_window(in, 1LL << 26, [&](DevBatch& part) { join_batch(cx, part, outs); });      // bounds the per-launch index vectors
  }

  void join_batch(OpContext& cx, DevBatch& in, std::vector<DevBatch>& outs) {
    const int64_t n = in.num_rows;
    if (n == 0) return;
    const int nk = (int)lkeys_.size();
    SortKeyCol kc[2];
    for (int i = 0; i < nk; i++) {
      const DevColumn& c = in.cols[(size_t)lkeys_[(size_t)i]];
      if (c.offset > 0xFFFFFFFFLL) throw ExecError(B200Q_ERR_UNSUPPORTED, "column offset beyond 2^32 rows");
      kc[i] = key_col(c.type, (const uint8_t*)c.values->ptr + (size_t)c.offset * c.type.byte_width(), c.validity ? (const uint8_t*)c.validity->ptr : nullptr, (uint32_t)c.offset, nullptr, opts_[(size_t)i]);
    }
    DevMemP w0 = DevMem::alloc((size_t)n * 8 + 16, cx.stream), w1 = nk > 1 ? DevMem::alloc((size_t)n * 8 + 16, cx.stream) : nullptr, fl = DevMem::alloc((size_t)n + 16, cx.stream);
    const MergeKeys lk{(const unsigned long long*)w0->ptr, w1 ? (const unsigned long long*)w1->ptr : nullptr, (const uint8_t*)fl->ptr};
    const MergeKeys rk = right_keys();
    B200Q_CUDA(cudaMemsetAsync(status_->ptr, 0, sizeof(SmjStatus), cx.stream));
    B200Q_CUDA(cudaEventRecord(cx.ev0, cx.stream));
    cx.m.launches += launch_smj_normalise(kc, nk, n, (unsigned long long*)w0->ptr, w1 ? (unsigned long long*)w1->ptr : nullptr, (uint8_t*)fl->ptr, (SmjCarry*)carry_->ptr, (SmjStatus*)status_->ptr, cx.stream);
    cx.m.launches += launch_smj_bounds(lk, n, rk, m_, (SmjStatus*)status_->ptr, cx.stream);
    const SmjStatus st = read_status(cx);
    if (st.unsorted) throw ExecError(B200Q_ERR_INVALID_ARG, "SortMergeJoinExec: the left input not sorted by the join keys under the node's sort_options");
    const int64_t rb0 = (int64_t)st.rb0, rb1 = (int64_t)st.rb1;
    DevMemP lo = DevMem::alloc((size_t)n * 4 + 16, cx.stream), hi = DevMem::alloc((size_t)n * 4 + 16, cx.stream), pr = DevMem::alloc((size_t)(rb1 - rb0) * 4 + 16, cx.stream);
    cx.m.launches += launch_smj_merge(lk, n, rk, rb0, rb1, (uint32_t*)lo->ptr, (uint32_t*)hi->ptr, (uint32_t*)pr->ptr, cx.stream);
    DevMemP counts = DevMem::alloc((size_t)n * 8 + 16, cx.stream);
    cx.m.launches += launch_smj_counts(lk, n, (const uint32_t*)lo->ptr, (const uint32_t*)hi->ptr, jt_, (unsigned long long*)counts->ptr, cx.stream);
    DevMemP L = scan(cx, counts, n);
    B200Q_CUDA(cudaEventRecord(cx.ev1, cx.stream));
    const int64_t lt = (int64_t)read_word(cx, (const unsigned long long*)L->ptr + n);
    SmjEmit e{};
    e.n = n; e.lo = (const uint32_t*)lo->ptr; e.hi = (const uint32_t*)hi->ptr; e.lflags = (const uint8_t*)fl->ptr; e.L = (const unsigned long long*)L->ptr;
    e.rb0 = rb0; e.pr = (const uint32_t*)pr->ptr; e.s0 = settled_;
    int64_t total = lt;
    DevMemP U;
    if (right_outer_) {                              // settle the right rows before the batch's last key: [settled_, lo[n - 1])
      uint32_t s_new = 0;
      B200Q_CUDA(cudaMemcpyAsync(&s_new, (const uint32_t*)lo->ptr + n - 1, 4, cudaMemcpyDeviceToHost, cx.stream));
      cx.m.launches += launch_smj_mark(lk, rk, rb0, rb1, (const uint32_t*)pr->ptr, (uint8_t*)matched_->ptr, cx.stream);
      B200Q_CUDA(cudaStreamSynchronize(cx.stream));
      const int64_t nw = (int64_t)s_new - settled_;
      U = unmatched_scan(cx, settled_, nw);
      total += (int64_t)read_word(cx, (const unsigned long long*)U->ptr + nw);
      e.nw = nw; e.U = (const unsigned long long*)U->ptr; e.matched = (const uint8_t*)matched_->ptr;
      settled_ = s_new;
    }
    add_kernel_time(cx, n, cx.cur_stage == 0);
    cx.m.fast_launches++;
    emit_chunks(cx, outs, &in, e, total);
  }

  DevMemP unmatched_scan(OpContext& cx, int64_t s0, int64_t nw) {
    DevMemP f = DevMem::alloc((size_t)nw * 8 + 16, cx.stream);
    cx.m.launches += launch_smj_unmatched((const uint8_t*)matched_->ptr, s0, nw, (unsigned long long*)f->ptr, cx.stream);
    return scan(cx, f, nw);
  }

  // the output rows [0, total) of one batch (in: its left rows; null: none), in chunks of at most max_launch_rows rows
  void emit_chunks(OpContext& cx, std::vector<DevBatch>& outs, const DevBatch* in, SmjEmit e, int64_t total) {
    const int64_t step = std::max<int64_t>(1, cx.conf.max_launch_rows);
    for (int64_t o0 = 0; o0 < total; o0 += step) {
      const int64_t cnt = std::min(step, total - o0);
      DevMemP pidx = DevMem::alloc((size_t)cnt * 4 + 16, cx.stream);
      DevMemP bidx = semi_like_ ? nullptr : DevMem::alloc((size_t)cnt * 4 + 16, cx.stream);
      DevMemP ex = jt_ == SJ_EXISTENCE ? DevMem::alloc((size_t)cnt + 16, cx.stream) : nullptr;
      e.o0 = o0; e.o1 = o0 + cnt; e.pidx = (uint32_t*)pidx->ptr; e.bidx = bidx ? (uint32_t*)bidx->ptr : nullptr; e.exists = ex ? (uint8_t*)ex->ptr : nullptr;
      cx.m.launches += launch_smj_emit(e, cx.stream);
      DevBatch ob; ob.num_rows = cnt;
      if (in) {
        std::vector<GatherSrc> ls;
        for (auto& c : in->cols) ls.push_back(gather_src_of(c, right_outer_));
        ob.cols = gather_columns(cx, ls, (const uint32_t*)pidx->ptr, cnt);
      } else {                                       // right-only rows: NULL left columns
        ob.cols = null_columns(cx, left_, cnt);
      }
      if (jt_ == SJ_EXISTENCE) {
        DevColumn x; x.type.id = T_BOOL; x.values = pack_bits(cx, ex->ptr, cnt);
        ob.cols.push_back(x);
      } else if (!semi_like_) {
        std::vector<GatherSrc> rs = rsrc_;
        for (auto& g : rs) g.may_be_null = g.may_be_null || left_outer_;
        for (auto& c : gather_columns(cx, rs, (const uint32_t*)bidx->ptr, cnt)) ob.cols.push_back(c);
      }
      B200Q_CUDA(cudaStreamSynchronize(cx.stream));   // the left batch's buffers are released when push returns
      outs.push_back(std::move(ob));
    }
  }

  void finish(OpContext& cx, std::vector<DevBatch>& outs) override {
    if (!attached_) throw ExecError(B200Q_ERR_STATE, "SortMergeJoinExec: no right side attached (b200q_op_attach_right) before finish");
    if (!right_outer_ || settled_ >= m_) return;
    const int64_t nw = m_ - settled_;                // the right rows no left batch settled: in right order, after everything
    DevMemP U = unmatched_scan(cx, settled_, nw);
    const int64_t total = (int64_t)read_word(cx, (const unsigned long long*)U->ptr + nw);
    SmjEmit e{};
    e.n = 0; e.L = (const unsigned long long*)zero_->ptr; e.U = (const unsigned long long*)U->ptr; e.s0 = settled_; e.nw = nw; e.rb0 = m_; e.matched = (const uint8_t*)matched_->ptr;
    settled_ = m_;
    emit_chunks(cx, outs, nullptr, e, total);
  }
};

}  // namespace

std::unique_ptr<Stage> make_smj_stage(OpContext& cx, const SchemaDef& in_schema, const PlanNode& node) { return std::unique_ptr<Stage>(new SmjStage(cx, in_schema, node)); }

}  // namespace b200q
