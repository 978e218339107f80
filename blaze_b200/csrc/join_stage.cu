// Hash join stages (SURVEY.md §8(f) rank 2): JoinBuildStage (BroadcastJoinBuildHashMapExecNode) and JoinProbeStage
// (BroadcastJoinExecNode / HashJoinExecNode).
//
// Reference (paths relative to the reference's native-engine/datafusion-ext-plans/src/):
//   BroadcastJoinBuildHashMapExec::execute    broadcast_join_build_hash_map_exec.rs:148-236 (collect the side, build ONE map)
//   BroadcastJoinExec::execute / execute_join broadcast_join_exec.rs:226-298, 496-560 (map side = broadcast / build side; the
//                                             other child is streamed through a Joiner)
//   joiner selection                          broadcast_join_exec.rs:333-358
//   FullJoiner / SemiJoiner                   joins/bhj/full_join.rs:90-379, joins/bhj/semi_join.rs:100-327
//   cached map shared by the tasks of a process  broadcast_join_exec.rs:640-677
// Shape on the GPU: the build side is its OWN op handle (as it is its own plan node in the reference): pushing the side's
// batches and finishing it leaves the table + the side's columns in HBM; any number of probe ops attach to it
// (b200q_op_attach_build — the counterpart of the process-wide map cache) and stream their batches.  A probe batch costs:
// one lookup pass, one scan, one pair-emit pass and one gather per output column; `map_joined` (rows of the build side
// that found a partner) belongs to the probe op, like the joiner's BitVec, and feeds finish() for the outer / semi forms.
#include <cstring>

#include "kernels_join.cuh"
#include "runtime.h"

namespace b200q {

namespace {

void fill_keys(JoinKeys& k, const std::vector<ExprP>& exprs, const DevBatch& in) {
  k.nkeys = (int)exprs.size();
  for (int i = 0; i < k.nkeys; i++) {
    const DevColumn& c = in.cols[(size_t)exprs[(size_t)i]->col_index];
    k.phys[i] = (uint8_t)phys_of(c.type);
    const int w = c.type.byte_width();
    if (c.offset > 0xFFFFFFFFLL) throw ExecError(B200Q_ERR_UNSUPPORTED, "column offset beyond 2^32 rows");
    k.col[i].values = (const uint8_t*)c.values->ptr + (size_t)c.offset * (size_t)w;
    k.col[i].validity = c.validity ? (const uint8_t*)c.validity->ptr : nullptr;
    k.col[i].bit_offset = (uint32_t)c.offset;
  }
}

}  // namespace

// all columns of one side through one index vector: one kernel per 16 columns
std::vector<DevColumn> gather_columns(OpContext& cx, const std::vector<GatherSrc>& srcs, const uint32_t* idx, int64_t n) {
  std::vector<DevColumn> out; std::vector<DevMemP> valid_bytes;
  for (size_t c0 = 0; c0 < srcs.size(); c0 += 16) {
    GatherSpec g{}; g.ncols = (int)std::min<size_t>(16, srcs.size() - c0);
    for (int c = 0; c < g.ncols; c++) {
      const GatherSrc& s = srcs[c0 + (size_t)c];
      DevColumn o; o.type = s.type;
      const int w = s.type.byte_width();
      o.values = DevMem::alloc((size_t)n * w + 16, cx.stream);
      DevMemP ob = s.may_be_null ? DevMem::alloc((size_t)n + 16, cx.stream) : nullptr;
      g.col[c] = GatherCol{s.values, s.vbits, s.vbytes, o.values->ptr, ob ? (uint8_t*)ob->ptr : nullptr, s.bit_offset, w};
      out.push_back(o); valid_bytes.push_back(ob);
    }
    cx.m.launches += launch_join_gather_multi(g, idx, n, cx.stream);
  }
  for (size_t c = 0; c < out.size(); c++)
    if (valid_bytes[c]) out[c].validity = pack_bits(cx, valid_bytes[c]->ptr, n);
  return out;
}

// ---- what a finished build op holds (shared with the probe ops that attach to it) -------------------------------------
struct JoinBuilt {
  SchemaDef schema;                               // the side's data schema
  std::vector<DType> key_types;
  ByteCols cols;                                  // the side's rows
  JoinTable table{};
  DevMemP t_keys, t_state, t_head, t_count, t_next, t_stats, t_packed;
  uint32_t max_dup = 0;                           // rows of the most duplicated key
  int device = 0;
};

namespace {

class JoinBuildStage : public Stage, public JoinBuildResult {
  std::vector<ExprP> keys_;
  std::vector<ByteCols> parts_;                   // owned copies of the pushed batches
  std::shared_ptr<JoinBuilt> built_;

 public:
  JoinBuildStage(OpContext& cx, const SchemaDef& in, const PlanNode& node) {
    in_schema = in; out_schema = node.schema;
    keys_ = node.join_build_keys;
    check_keys(keys_, "BroadcastJoinBuildHashMapExec");
    check_data_schema(in, "BroadcastJoinBuildHashMapExec");
    for (size_t i = 0; i < in.fields.size(); i++) used_input_cols.push_back((int)i);
    (void)cx;
  }

  void push(OpContext& cx, DevBatch& in, std::vector<DevBatch>&) override {
    if (built_) throw ExecError(B200Q_ERR_STATE, "join build side: push after finish");
    if (in.num_rows == 0) return;
    parts_.push_back(to_byte_cols(cx, in_schema, {&in}));         // the caller's buffers are released when push returns: keep an owned copy
  }

  void finish(OpContext& cx, std::vector<DevBatch>&) override {
    if (built_) return;
    auto b = std::make_shared<JoinBuilt>();
    b->schema = in_schema; b->device = cx.device;
    for (auto& e : keys_) b->key_types.push_back(e->type);
    int64_t total = 0;
    for (auto& p : parts_) total += p.rows;
    if (total >= (1LL << 30)) throw ExecError(B200Q_ERR_UNSUPPORTED, "join hash table: number of rows exceeded 2^30");     // join_hash_map.rs:107-110
    b->cols = concat(cx, in_schema, std::move(parts_));
    // table: a power of two >= 2 x rows slots
    uint64_t cap = 1024;
    while (cap < (uint64_t)total * 2) cap <<= 1;
    JoinTable& t = b->table;
    t.nkw = (int)keys_.size(); t.mask = (uint32_t)(cap - 1);
    b->t_keys = DevMem::alloc((size_t)cap * t.nkw * 8, cx.stream);
    b->t_state = DevMem::alloc((size_t)cap * 4, cx.stream, true);
    b->t_head = DevMem::alloc((size_t)cap * 4, cx.stream);
    b->t_count = DevMem::alloc((size_t)cap * 4, cx.stream, true);
    b->t_next = DevMem::alloc((size_t)total * 4 + 16, cx.stream);
    b->t_stats = DevMem::alloc(16, cx.stream, true);
    b->t_packed = DevMem::alloc((size_t)cap * (keys_.size() == 1 ? 2 : 4) * 8 + 16, cx.stream);
    B200Q_CUDA(cudaMemsetAsync(b->t_head->ptr, 0xFF, (size_t)cap * 4, cx.stream));
    t.keys = (unsigned long long*)b->t_keys->ptr; t.state = (uint32_t*)b->t_state->ptr; t.head = (uint32_t*)b->t_head->ptr;
    t.count = (uint32_t*)b->t_count->ptr; t.next = (uint32_t*)b->t_next->ptr; t.stats = (uint32_t*)b->t_stats->ptr; t.packed = (unsigned long long*)b->t_packed->ptr;
    if (total > 0) {
      JoinKeys k{}; k.nkeys = (int)keys_.size();
      for (int i = 0; i < k.nkeys; i++) {
        const size_t c = (size_t)keys_[(size_t)i]->col_index;
        k.phys[i] = (uint8_t)phys_of(in_schema.fields[c].type);
        k.col[i].values = b->cols.values[c]->ptr; k.col[i].validity = nullptr; k.col[i].bit_offset = 0;
      }
      // NULL keys: the build kernel reads validity bitmaps; the side keeps bytes -> pack the keys' bytes once
      std::vector<DevMemP> key_bits;
      for (int i = 0; i < k.nkeys; i++) {
        const size_t c = (size_t)keys_[(size_t)i]->col_index;
        if (!b->cols.valid[c]) continue;
        DevMemP bits = pack_bits(cx, b->cols.valid[c]->ptr, total);
        k.col[i].validity = (const uint8_t*)bits->ptr; key_bits.push_back(bits);
      }
      B200Q_CUDA(cudaEventRecord(cx.ev0, cx.stream));
      cx.m.launches += launch_join_build(k, total, t, cx.stream);
      B200Q_CUDA(cudaEventRecord(cx.ev1, cx.stream));
      B200Q_CUDA(cudaMemcpyAsync(&b->max_dup, b->t_stats->ptr, 4, cudaMemcpyDeviceToHost, cx.stream));
      B200Q_CUDA(cudaStreamSynchronize(cx.stream));
      add_kernel_time(cx, total, true);
      cx.m.fast_launches++;
    }
    if (total == 0) { JoinKeys k0{}; cx.m.launches += launch_join_build(k0, 0, t, cx.stream); }      // an empty map side still needs its (all-empty) probe view
    B200Q_CUDA(cudaStreamSynchronize(cx.stream));           // probe ops run on their own streams
    cx.m.num_groups = total; cx.m.table_capacity = (int64_t)cap;
    built_ = b;
  }

  std::shared_ptr<JoinBuilt> built() const override { return built_; }
};

enum ProtoJoinType { PJ_INNER = 0, PJ_LEFT = 1, PJ_RIGHT = 2, PJ_FULL = 3, PJ_SEMI = 4, PJ_ANTI = 5, PJ_EXISTENCE = 6 };   // auron.proto:475-483; Semi/Anti = LeftSemi/LeftAnti (auron-serde/src/lib.rs:104-116)

class JoinProbeStage : public Stage, public JoinProbeAttach {
  int jt_; bool build_is_left_;
  SchemaDef left_, right_;
  std::vector<ExprP> probe_keys_;
  std::vector<DType> build_key_types_;
  std::shared_ptr<JoinBuilt> built_;
  DevMemP map_joined_;                               // one byte per build row
  bool probe_outer_ = false, build_outer_ = false, semi_like_ = false, probe_is_join_side_ = false;

  const SchemaDef& probe_schema() const { return build_is_left_ ? right_ : left_; }
  const SchemaDef& build_schema() const { return build_is_left_ ? left_ : right_; }

 public:
  JoinProbeStage(OpContext&, const SchemaDef& in, const PlanNode& node) {
    jt_ = node.join_type; build_is_left_ = node.join_build_is_left;
    left_ = node.join_left_schema; right_ = node.join_right_schema;
    in_schema = in; out_schema = node.schema;
    if (jt_ < PJ_INNER || jt_ > PJ_EXISTENCE) throw PlanError(B200Q_ERR_INVALID_PLAN, "invalid JoinType");
    std::vector<ExprP> lk, rk;
    for (auto& p : node.join_on) { lk.push_back(p.first); rk.push_back(p.second); }
    check_keys(lk, "join"); check_keys(rk, "join");
    for (size_t i = 0; i < lk.size(); i++)
      if (lk[i]->type.is_integer() != rk[i]->type.is_integer() || (!lk[i]->type.is_integer() && lk[i]->type.id != rk[i]->type.id))
        throw PlanError(B200Q_ERR_UNSUPPORTED, "join keys of different type classes (" + lk[i]->type.str() + " vs " + rk[i]->type.str() + ")");
    probe_keys_ = build_is_left_ ? rk : lk;
    for (auto& e : (build_is_left_ ? lk : rk)) build_key_types_.push_back(e->type);
    check_data_schema(left_, "join"); check_data_schema(right_, "join");
    const bool probe_is_left = !build_is_left_;
    probe_outer_ = jt_ == PJ_FULL || (jt_ == PJ_LEFT && probe_is_left) || (jt_ == PJ_RIGHT && !probe_is_left);        // full_join.rs:71-79
    build_outer_ = jt_ == PJ_FULL || (jt_ == PJ_LEFT && !probe_is_left) || (jt_ == PJ_RIGHT && probe_is_left);
    semi_like_ = jt_ == PJ_SEMI || jt_ == PJ_ANTI || jt_ == PJ_EXISTENCE;
    probe_is_join_side_ = semi_like_ && probe_is_left;                                                                     // semi_join.rs:78-87 (the wire carries the Left forms only)
    // output = left ++ right (or left [++ exists#0]); types must agree with the declared schema
    const size_t want = jt_ == PJ_EXISTENCE ? left_.fields.size() + 1 : (semi_like_ ? left_.fields.size() : left_.fields.size() + right_.fields.size());
    if (out_schema.fields.size() != want) throw PlanError(B200Q_ERR_INVALID_PLAN, "join schema has " + std::to_string(out_schema.fields.size()) + " fields, the join produces " + std::to_string(want));
    for (size_t i = 0; i < want; i++) {
      const DType& got = out_schema.fields[i].type;
      DType exp; if (i < left_.fields.size()) exp = left_.fields[i].type; else if (jt_ == PJ_EXISTENCE) exp.id = T_BOOL; else exp = right_.fields[i - left_.fields.size()].type;
      if (got != exp) throw PlanError(B200Q_ERR_INVALID_PLAN, "join schema field " + std::to_string(i) + " is " + got.str() + ", the inputs give " + exp.str());
    }
    for (size_t i = 0; i < in.fields.size(); i++) used_input_cols.push_back((int)i);
  }

  void attach(std::shared_ptr<JoinBuilt> b) override {
    if (!b) throw ExecError(B200Q_ERR_STATE, "attach_build: the build op has not finished");
    if (b->schema.fields.size() != build_schema().fields.size()) throw ExecError(B200Q_ERR_INVALID_ARG, "attach_build: the build op's schema does not match the join's build side");
    for (size_t i = 0; i < b->schema.fields.size(); i++)
      if (b->schema.fields[i].type != build_schema().fields[i].type) throw ExecError(B200Q_ERR_INVALID_ARG, "attach_build: type of build column " + std::to_string(i) + " differs");
    if (b->key_types.size() != build_key_types_.size()) throw ExecError(B200Q_ERR_INVALID_ARG, "attach_build: the build op was keyed on a different number of columns");
    built_ = b;
  }

  void need_built(OpContext& cx) {
    if (!built_) throw ExecError(B200Q_ERR_STATE, "join: no build side attached (b200q_op_attach_build) before the first probe batch");
    if (built_->device != cx.device) throw ExecError(B200Q_ERR_INVALID_ARG, "join: the build side lives on another device");
    if (!map_joined_ && (build_outer_ || (semi_like_ && !probe_is_join_side_))) map_joined_ = DevMem::alloc((size_t)built_->cols.rows + 16, cx.stream, true);
  }

  std::vector<DevColumn> gather_probe(OpContext& cx, const DevBatch& in, const uint32_t* idx, int64_t n, bool nil_possible) {
    std::vector<GatherSrc> srcs;
    for (auto& c : in.cols) srcs.push_back(gather_src_of(c, nil_possible));
    return gather_columns(cx, srcs, idx, n);
  }
  std::vector<DevColumn> gather_build(OpContext& cx, const uint32_t* idx, int64_t n, bool nil_possible) {
    const ByteCols& b = built_->cols;
    std::vector<GatherSrc> srcs;
    for (size_t c = 0; c < built_->schema.fields.size(); c++)
      srcs.push_back(GatherSrc{built_->schema.fields[c].type, b.values[c]->ptr, nullptr, 0, b.valid[c] ? (const uint8_t*)b.valid[c]->ptr : nullptr, nil_possible || (bool)b.valid[c]});
    return gather_columns(cx, srcs, idx, n);
  }
  void emit(std::vector<DevBatch>& outs, std::vector<DevColumn> pcols, std::vector<DevColumn> bcols, int64_t n) {
    DevBatch ob; ob.num_rows = n;
    std::vector<DevColumn>& first = build_is_left_ ? bcols : pcols; std::vector<DevColumn>& second = build_is_left_ ? pcols : bcols;
    for (auto& c : first) ob.cols.push_back(c);
    for (auto& c : second) ob.cols.push_back(c);
    outs.push_back(std::move(ob));
  }
  // exclusive scan of n int32 -> offs[n + 1]; returns the total (host)
  int64_t scan(OpContext& cx, const int32_t* in, int64_t n, DevMemP& offs) {
    offs = DevMem::alloc((size_t)(n + 1) * 4, cx.stream);
    DevMemP sums = DevMem::alloc((size_t)scan_num_blocks(n) * 4 + 16, cx.stream);
    cx.m.launches += launch_exclusive_scan_i32(in, (int32_t*)offs->ptr, n, (int32_t*)sums->ptr, cx.stream);
    int32_t total = 0;
    B200Q_CUDA(cudaMemcpyAsync(&total, (const int32_t*)offs->ptr + n, 4, cudaMemcpyDeviceToHost, cx.stream));
    B200Q_CUDA(cudaStreamSynchronize(cx.stream));
    if (total < 0) throw ExecError(B200Q_ERR_UNSUPPORTED, "join: more than 2^31-1 output rows from one probe batch; push smaller batches");
    return total;
  }

  void push(OpContext& cx, DevBatch& in, std::vector<DevBatch>& outs) override {
    need_built(cx);
    for_each_window(in, 1LL << 26, [&](DevBatch& part) { probe(cx, part, outs); });      // bounds the per-launch index vectors / output columns
  }

  void probe(OpContext& cx, DevBatch& in, std::vector<DevBatch>& outs) {
    const int64_t n = in.num_rows;
    if (n == 0) return;
    JoinKeys k{}; fill_keys(k, probe_keys_, in);
    DevMemP cursor = DevMem::alloc(16, cx.stream, true);
    auto read_cursor = [&]() { unsigned long long v = 0; B200Q_CUDA(cudaMemcpyAsync(&v, cursor->ptr, 8, cudaMemcpyDeviceToHost, cx.stream)); B200Q_CUDA(cudaStreamSynchronize(cx.stream)); return (int64_t)v; };
    B200Q_CUDA(cudaEventRecord(cx.ev0, cx.stream));
    if (!semi_like_) {
      // pass 1 looks every probe row up (keys only: 8 B/row in, for unique map keys 4 B/row of chain heads out) and counts the output rows, then
      //   unique map keys (the PK side of a PK-FK join): ONE fused gather pass writes the output columns of both sides in probe-row order;
      //   duplicated map keys: (probe row, map row) pairs, then one gather pass per side
      const bool fused = built_->max_dup <= 1 && in.cols.size() <= 16 && built_->schema.fields.size() <= 16;
      DevMemP head = fused ? DevMem::alloc((size_t)n * 4 + 16, cx.stream) : nullptr;
      if (fused) cx.m.launches += launch_join_probe_count(k, n, built_->table, probe_outer_ ? 1 : 0, (uint32_t*)head->ptr, nullptr, cx.stream, (unsigned long long*)cursor->ptr);
      else cx.m.launches += launch_join_probe_pairs(k, n, built_->table, probe_outer_ ? 1 : 0, (unsigned long long*)cursor->ptr, nullptr, nullptr, nullptr, cx.stream);
      const int64_t total = read_cursor();
      if (total > 0x7FFFFFFFLL) throw ExecError(B200Q_ERR_UNSUPPORTED, "join: more than 2^31-1 output rows from one probe batch; push smaller batches");
      B200Q_CUDA(cudaMemsetAsync(cursor->ptr, 0, 8, cx.stream));
      uint8_t* mark = build_outer_ ? (uint8_t*)map_joined_->ptr : nullptr;
      if (total > 0 && fused) {
        GatherSpec pc{}, bc{};
        std::vector<DevColumn> pcols, bcols; std::vector<DevMemP> pvb, bvb;
        auto out_col = [&](const DType& t, bool may_be_null, GatherCol& g, std::vector<DevColumn>& cols, std::vector<DevMemP>& vbs) {
          DevColumn o; o.type = t;
          o.values = DevMem::alloc((size_t)total * t.byte_width() + 16, cx.stream);
          DevMemP vb = may_be_null ? DevMem::alloc((size_t)total + 16, cx.stream) : nullptr;
          g.out = o.values->ptr; g.out_valid = vb ? (uint8_t*)vb->ptr : nullptr; g.width = t.byte_width();
          cols.push_back(o); vbs.push_back(vb);
        };
        pc.ncols = (int)in.cols.size();
        for (int c = 0; c < pc.ncols; c++) {
          const DevColumn& sc = in.cols[(size_t)c];
          GatherCol& g = pc.col[c];
          g.src = (const uint8_t*)sc.values->ptr + (size_t)sc.offset * sc.type.byte_width(); g.vbits = sc.validity ? (const uint8_t*)sc.validity->ptr : nullptr; g.bit_offset = (uint32_t)sc.offset; g.vbytes = nullptr;
          out_col(sc.type, (bool)sc.validity, g, pcols, pvb);
        }
        bc.ncols = (int)built_->schema.fields.size();
        for (int c = 0; c < bc.ncols; c++) {
          GatherCol& g = bc.col[c];
          const DevMemP& vb = built_->cols.valid[(size_t)c];
          g.src = built_->cols.values[(size_t)c]->ptr; g.vbits = nullptr; g.bit_offset = 0; g.vbytes = vb ? (const uint8_t*)vb->ptr : nullptr;
          out_col(built_->schema.fields[(size_t)c].type, probe_outer_ || vb, g, bcols, bvb);
        }
        cx.m.launches += launch_join_probe_fused((const uint32_t*)head->ptr, n, probe_outer_ ? 1 : 0, (unsigned long long*)cursor->ptr, pc, bc, mark, cx.stream);
        auto pack = [&](std::vector<DevColumn>& cols, std::vector<DevMemP>& vbs) {
          for (size_t c = 0; c < cols.size(); c++)
            if (vbs[c]) cols[c].validity = pack_bits(cx, vbs[c]->ptr, total);
        };
        pack(pcols, pvb); pack(bcols, bvb);
        emit(outs, pcols, bcols, total);
      } else if (total > 0) {
        DevMemP pidx = DevMem::alloc((size_t)total * 4 + 16, cx.stream), bidx = DevMem::alloc((size_t)total * 4 + 16, cx.stream);
        cx.m.launches += launch_join_probe_pairs(k, n, built_->table, probe_outer_ ? 1 : 0, (unsigned long long*)cursor->ptr, (uint32_t*)pidx->ptr, (uint32_t*)bidx->ptr, mark, cx.stream);
        emit(outs, gather_probe(cx, in, (const uint32_t*)pidx->ptr, total, false), gather_build(cx, (const uint32_t*)bidx->ptr, total, probe_outer_), total);
      }
    } else {
      if (!probe_is_join_side_) cx.m.launches += launch_join_probe_mark(k, n, built_->table, (uint8_t*)map_joined_->ptr, cx.stream);
      else if (jt_ == PJ_EXISTENCE) {                  // every probe row + exists#0 (semi_join.rs:252-258)
        DevBatch ob; ob.num_rows = n;
        for (auto& c : in.cols) {
          DevColumn o = c;
          if (c.offset != 0) {                         // outputs carry offset 0
            const int w = c.type.byte_width();
            o.values = DevMem::alloc((size_t)n * w + 16, cx.stream); o.offset = 0;
            B200Q_CUDA(cudaMemcpyAsync(o.values->ptr, (const uint8_t*)c.values->ptr + (size_t)c.offset * w, (size_t)n * w, cudaMemcpyDeviceToDevice, cx.stream));
            if (c.validity) { DevMemP vb = DevMem::alloc((size_t)n + 16, cx.stream); cx.m.launches += launch_unpack_bits((const uint8_t*)c.validity->ptr, (uint32_t)c.offset, n, (uint8_t*)vb->ptr, cx.stream);
                              o.validity = pack_bits(cx, vb->ptr, n); }
          } else {                                     // the caller's buffers are released after push: copy
            const int w = c.type.byte_width();
            o.values = DevMem::alloc((size_t)n * w + 16, cx.stream);
            B200Q_CUDA(cudaMemcpyAsync(o.values->ptr, c.values->ptr, (size_t)n * w, cudaMemcpyDeviceToDevice, cx.stream));
            if (c.validity) { o.validity = DevMem::alloc(bitmap_bytes(n), cx.stream, true); B200Q_CUDA(cudaMemcpyAsync(o.validity->ptr, c.validity->ptr, (size_t)(n + 7) / 8, cudaMemcpyDeviceToDevice, cx.stream)); }
          }
          ob.cols.push_back(o);
        }
        DevMemP head = DevMem::alloc((size_t)n * 4 + 16, cx.stream), fb = DevMem::alloc((size_t)n + 16, cx.stream);
        cx.m.launches += launch_join_probe_count(k, n, built_->table, 0, (uint32_t*)head->ptr, nullptr, cx.stream);
        cx.m.launches += launch_join_match_bytes((const uint32_t*)head->ptr, n, (uint8_t*)fb->ptr, cx.stream);
        DevColumn ex; ex.type.id = T_BOOL; ex.values = pack_bits(cx, fb->ptr, n);
        ob.cols.push_back(ex);
        outs.push_back(std::move(ob));
      } else {                                         // LeftSemi / LeftAnti with the probe side as the join side (semi_join.rs:243-251)
        DevMemP idx = DevMem::alloc((size_t)n * 4 + 16, cx.stream);
        cx.m.launches += launch_join_probe_select(k, n, built_->table, jt_ == PJ_ANTI ? 1 : 0, (unsigned long long*)cursor->ptr, (uint32_t*)idx->ptr, cx.stream);
        const int64_t total = read_cursor();
        if (total > 0) { DevBatch ob; ob.num_rows = total; ob.cols = gather_probe(cx, in, (const uint32_t*)idx->ptr, total, false); outs.push_back(std::move(ob)); }
      }
    }
    B200Q_CUDA(cudaEventRecord(cx.ev1, cx.stream));
    B200Q_CUDA(cudaStreamSynchronize(cx.stream));
    add_kernel_time(cx, n, true);
    cx.m.fast_launches++;
  }

  void finish(OpContext& cx, std::vector<DevBatch>& outs) override {
    if (!built_) { if (cx.m.input_rows == 0) return; throw ExecError(B200Q_ERR_STATE, "join: no build side attached"); }
    need_built(cx);
    const int64_t nb = built_->cols.rows;
    if (nb == 0 || !map_joined_) return;
    if (!semi_like_ && build_outer_) {                 // unjoined build rows next to NULL probe columns (full_join.rs:322-362)
      DevMemP fl = DevMem::alloc((size_t)nb * 4 + 16, cx.stream), offs;
      cx.m.launches += launch_bytes_to_flags((const uint8_t*)map_joined_->ptr, nb, 1, (int32_t*)fl->ptr, cx.stream);
      const int64_t total = scan(cx, (const int32_t*)fl->ptr, nb, offs);
      if (total > 0) {
        DevMemP idx = DevMem::alloc((size_t)total * 4 + 16, cx.stream);
        cx.m.launches += launch_join_compact_indices((const int32_t*)fl->ptr, (const int32_t*)offs->ptr, nb, (uint32_t*)idx->ptr, cx.stream);
        emit(outs, null_columns(cx, probe_schema(), total), gather_build(cx, (const uint32_t*)idx->ptr, total, false), total);
      }
    } else if (semi_like_ && !probe_is_join_side_) {   // the build side is the join side (semi_join.rs:276-312)
      if (jt_ == PJ_EXISTENCE) {
        DevMemP idn = DevMem::alloc((size_t)nb * 4 + 16, cx.stream), ones = DevMem::alloc((size_t)nb * 4 + 16, cx.stream), offs;
        B200Q_CUDA(cudaMemsetAsync(ones->ptr, 0, (size_t)nb * 4, cx.stream));
        cx.m.launches += launch_bytes_to_flags((const uint8_t*)map_joined_->ptr, nb, 0, (int32_t*)ones->ptr, cx.stream);          // reused below as the exists flags
        DevMemP all = DevMem::alloc((size_t)nb * 4 + 16, cx.stream);
        DevMemP allb = DevMem::alloc((size_t)nb + 16, cx.stream);
        B200Q_CUDA(cudaMemsetAsync(allb->ptr, 1, (size_t)nb, cx.stream));
        cx.m.launches += launch_bytes_to_flags((const uint8_t*)allb->ptr, nb, 0, (int32_t*)all->ptr, cx.stream);
        scan(cx, (const int32_t*)all->ptr, nb, offs);
        cx.m.launches += launch_join_compact_indices((const int32_t*)all->ptr, (const int32_t*)offs->ptr, nb, (uint32_t*)idn->ptr, cx.stream);   // identity indices
        DevBatch ob; ob.num_rows = nb; ob.cols = gather_build(cx, (const uint32_t*)idn->ptr, nb, false);
        DevColumn ex; ex.type.id = T_BOOL; ex.values = pack_bits(cx, map_joined_->ptr, nb);
        ob.cols.push_back(ex);
        outs.push_back(std::move(ob));
      } else {
        DevMemP fl = DevMem::alloc((size_t)nb * 4 + 16, cx.stream), offs;
        cx.m.launches += launch_bytes_to_flags((const uint8_t*)map_joined_->ptr, nb, jt_ == PJ_ANTI ? 1 : 0, (int32_t*)fl->ptr, cx.stream);
        const int64_t total = scan(cx, (const int32_t*)fl->ptr, nb, offs);
        if (total > 0) {
          DevMemP idx = DevMem::alloc((size_t)total * 4 + 16, cx.stream);
          cx.m.launches += launch_join_compact_indices((const int32_t*)fl->ptr, (const int32_t*)offs->ptr, nb, (uint32_t*)idx->ptr, cx.stream);
          DevBatch ob; ob.num_rows = total; ob.cols = gather_build(cx, (const uint32_t*)idx->ptr, total, false);
          outs.push_back(std::move(ob));
        }
      }
    }
    map_joined_.reset();
  }
};

}  // namespace

std::unique_ptr<Stage> make_join_build_stage(OpContext& cx, const SchemaDef& in_schema, const PlanNode& node) { return std::unique_ptr<Stage>(new JoinBuildStage(cx, in_schema, node)); }
std::unique_ptr<Stage> make_join_probe_stage(OpContext& cx, const SchemaDef& in_schema, const PlanNode& node) { return std::unique_ptr<Stage>(new JoinProbeStage(cx, in_schema, node)); }

}  // namespace b200q
