// SortStage: SortExecNode (SURVEY.md §8(f) rank 4).
//
// Reference (datafusion-ext-plans/src/sort_exec.rs): SortExec::new(input, exprs, fetch) :97-112; per-batch sort by the
// arrow-row encoded keys + `take(limit)` :626-678; merge of the sorted blocks + output in batches :680-752, 896-1027;
// plan decode auron-serde/src/from_proto.rs:312-324 (PhysicalSortExprNode{expr, asc, nulls_first}, FetchLimit).
// GPU: the input is collected in HBM (the sort is a pipeline breaker in the reference too); finish() sorts a row
// permutation with the stable radix passes of kernels_sort.cu, least significant key first, and gathers the first
// `fetch` rows of every column.  No spill: an input that does not fit HBM reports UNSUPPORTED (DevMem::alloc) and the
// host keeps its external sorter.
#include <cstring>

#include "kernels_join.cuh"
#include "kernels_sort.cuh"
#include "runtime.h"

namespace b200q {

namespace {

class SortStage : public Stage {
  struct Key { int col; bool desc, nulls_first; };
  std::vector<Key> keys_;
  int64_t fetch_ = -1;
  std::vector<ByteCols> parts_;                                       // owned copies of the pushed batches

 public:
  SortStage(OpContext&, const SchemaDef& in, const PlanNode& node) {
    in_schema = in; out_schema = in;
    if (node.sort_exprs.empty()) throw PlanError(B200Q_ERR_INVALID_PLAN, "SortExec without sort expressions");
    for (auto& se : node.sort_exprs) {
      if (se.expr->kind != E_COLUMN) throw PlanError(B200Q_ERR_UNSUPPORTED, "sort key is a computed expression (project it first)");
      keys_.push_back(Key{se.expr->col_index, !se.asc, se.nulls_first});
    }
    for (auto& f : in.fields)
      if (f.type.id == T_BOOL || f.type.is_varlen() || f.type.id == T_NULL) throw PlanError(B200Q_ERR_UNSUPPORTED, "SortExec over a " + f.type.str() + " column is not on the GPU path");
    fetch_ = node.sort_has_fetch ? (int64_t)node.sort_fetch : -1;
    for (size_t i = 0; i < in.fields.size(); i++) used_input_cols.push_back((int)i);
  }

  void push(OpContext& cx, DevBatch& in, std::vector<DevBatch>&) override {
    if (in.num_rows == 0) return;                                       // sort_exec.rs:627-629
    parts_.push_back(to_byte_cols(cx, in_schema, {&in}));              // the caller's buffers are released when push returns
  }

  void finish(OpContext& cx, std::vector<DevBatch>& outs) override {
    int64_t n = 0;
    for (auto& p : parts_) n += p.rows;
    if (n == 0) return;
    if (n > 0x7FFFFFFFLL) throw ExecError(B200Q_ERR_UNSUPPORTED, "SortExec: more than 2^31-1 rows");
    const size_t ncols = in_schema.fields.size();
    const ByteCols cols = concat(cx, in_schema, std::move(parts_));
    const std::vector<DevMemP> &values = cols.values, &valid = cols.valid;
    // ---- sort a permutation ------------------------------------------------------------------------------------------
    const int64_t ntiles = sort_num_tiles(n);
    DevMemP keyA = DevMem::alloc((size_t)n * 8, cx.stream), keyB = DevMem::alloc((size_t)n * 8, cx.stream);
    DevMemP nulA = DevMem::alloc((size_t)n + 16, cx.stream), nulB = DevMem::alloc((size_t)n + 16, cx.stream);
    DevMemP idxA = DevMem::alloc((size_t)n * 4 + 16, cx.stream), idxB = DevMem::alloc((size_t)n * 4 + 16, cx.stream);
    DevMemP counts = DevMem::alloc((size_t)(256 * ntiles + 1) * 4, cx.stream), offs = DevMem::alloc((size_t)(256 * ntiles + 1) * 4, cx.stream);
    DevMemP sums = DevMem::alloc((size_t)scan_num_blocks(256 * ntiles) * 4 + 16, cx.stream), hist = DevMem::alloc(9 * 256 * 8, cx.stream);
    B200Q_CUDA(cudaEventRecord(cx.ev0, cx.stream));
    cx.m.launches += launch_sort_iota((uint32_t*)idxA->ptr, n, cx.stream);
    std::vector<unsigned long long> h(9 * 256);
    for (size_t ki = keys_.size(); ki-- > 0;) {                         // least significant key first
      const Key& k = keys_[ki];
      const DType& t = in_schema.fields[(size_t)k.col].type;
      const int nwords = t.id == T_DECIMAL128 ? 2 : 1;
      const bool nullable = (bool)valid[(size_t)k.col];
      for (int wd = 0; wd < nwords; wd++) {
        SortKeyCol sk{}; sk.values = values[(size_t)k.col]->ptr; sk.valid_bytes = nullable ? (const uint8_t*)valid[(size_t)k.col]->ptr : nullptr;
        sk.phys = (uint8_t)phys_of(t); sk.descending = k.desc; sk.nulls_first = k.nulls_first; sk.dec_word = (uint8_t)wd;
        const int w = t.id == T_DECIMAL128 ? 8 : t.byte_width();
        sk.mask = w >= 8 ? ~0ull : ((1ull << (8 * w)) - 1);
        const bool last_word = wd == nwords - 1;
        cx.m.launches += launch_sort_normalise(sk, (const uint32_t*)idxA->ptr, n, (unsigned long long*)keyA->ptr, nullable ? (uint8_t*)nulA->ptr : nullptr, cx.stream);
        B200Q_CUDA(cudaMemsetAsync(hist->ptr, 0, 9 * 256 * 8, cx.stream));
        cx.m.launches += launch_sort_digit_hist((const unsigned long long*)keyA->ptr, nullable ? (const uint8_t*)nulA->ptr : nullptr, n, (unsigned long long*)hist->ptr, cx.stream);
        B200Q_CUDA(cudaMemcpyAsync(h.data(), hist->ptr, 9 * 256 * 8, cudaMemcpyDeviceToHost, cx.stream));
        B200Q_CUDA(cudaStreamSynchronize(cx.stream));
        auto varies = [&](int d) { for (int b = 0; b < 256; b++) if (h[(size_t)d * 256 + b] == (unsigned long long)n) return false; return true; };
        for (int d = 0; d < 9; d++) {
          if (d == 8 && (!nullable || !last_word)) break;                // the NULL rank is the most significant digit of the column
          if (!varies(d)) continue;                                      // every row agrees on this digit
          cx.m.launches += launch_sort_pass((const unsigned long long*)keyA->ptr, nullable ? (const uint8_t*)nulA->ptr : nullptr, (const uint32_t*)idxA->ptr, n, d == 8 ? -1 : 8 * d,
                                            (int32_t*)counts->ptr, (int32_t*)offs->ptr, (int32_t*)sums->ptr, (unsigned long long*)keyB->ptr, nullable ? (uint8_t*)nulB->ptr : nullptr,
                                            (uint32_t*)idxB->ptr, cx.stream);
          std::swap(keyA, keyB); std::swap(nulA, nulB); std::swap(idxA, idxB);
        }
      }
    }
    B200Q_CUDA(cudaEventRecord(cx.ev1, cx.stream));
    // ---- gather the first `fetch` rows ----------------------------------------------------------------------------------
    const int64_t m = fetch_ >= 0 ? std::min<int64_t>(fetch_, n) : n;
    if (m > 0) {
      DevBatch ob; ob.num_rows = m;
      for (size_t c = 0; c < ncols; c++) {
        DevColumn o; o.type = in_schema.fields[c].type;
        const int w = o.type.byte_width();
        o.values = DevMem::alloc((size_t)m * w + 16, cx.stream);
        DevMemP ob_valid = valid[c] ? DevMem::alloc((size_t)m + 16, cx.stream) : nullptr;
        cx.m.launches += launch_join_gather(values[c]->ptr, nullptr, 0, valid[c] ? (const uint8_t*)valid[c]->ptr : nullptr, w, (const uint32_t*)idxA->ptr, m, o.values->ptr,
                                            ob_valid ? (uint8_t*)ob_valid->ptr : nullptr, cx.stream);
        if (ob_valid) o.validity = pack_bits(cx, ob_valid->ptr, m);
        ob.cols.push_back(o);
      }
      outs.push_back(std::move(ob));
    }
    B200Q_CUDA(cudaStreamSynchronize(cx.stream));
    add_kernel_time(cx, n, cx.cur_stage == 0);
    cx.m.fast_launches++;
  }
};

}  // namespace

std::unique_ptr<Stage> make_sort_stage(OpContext& cx, const SchemaDef& in_schema, const PlanNode& node) { return std::unique_ptr<Stage>(new SortStage(cx, in_schema, node)); }

}  // namespace b200q
