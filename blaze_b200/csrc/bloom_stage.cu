// AggExec whose aggregates are all BLOOM_FILTER, without grouping keys (agg/bloom_filter.rs AggBloomFilter): Spark's runtime
// bloom filter on its creation side.  One accumulator per aggregate, a device bit array that is None until the first row arrives
// (Partial: partial_update creates it from estimated_num_items / num_bits; merge modes: the first non-None state becomes it).
//   Partial       put_long of every non-NULL value (kernels_bloom.cu)
//   PartialMerge  put_all of every incoming state: equal k and equal size, else INVALID_ARG
//   Final         put_all, then shrink_to_fit and write_to into a Binary column of one row (None -> NULL)
// States travel as the reference's frozen row in the Binary agg-buffer column ([0] for None, else [1] ++ write_to of the
// unshrunk filter, one after another for the aggregates of the node; AccBloomFilterColumn::freeze_to_rows) or, with
// partial_state_columnar = 1, as one nullable Binary column per aggregate holding the write_to bytes.
#include <cstring>

#include "kernels_bloom.cuh"
#include "runtime.h"

namespace b200q {

namespace {

struct BloomHeader { int32_t k = 0; int64_t nwords = 0; };

int32_t be32(const uint8_t* p) { return (int32_t)((uint32_t)p[0] << 24 | (uint32_t)p[1] << 16 | (uint32_t)p[2] << 8 | (uint32_t)p[3]); }

class BloomAggStage : public Stage {
  struct Acc { DevMemP bits; int64_t nwords = 0; int32_t k = 0; };   // bits null: None
  std::vector<AggDef> aggs_;
  std::vector<int> value_cols_;          // Partial: the input column of each aggregate's value
  std::vector<int> state_cols_;          // merge modes: the Binary state column (one for the frozen rows, one per aggregate columnar)
  bool update_ = false, final_ = false, columnar_ = false;
  std::vector<Acc> acc_;

  Acc new_acc(OpContext& cx, int64_t nwords, int32_t k) {
    Acc a; a.nwords = nwords; a.k = k;
    a.bits = DevMem::alloc((size_t)nwords * 8, cx.stream, true);
    return a;
  }

  // the header of the serialized filter at device address p (at most `avail` bytes there), checked as read_from would need it
  static BloomHeader read_header(OpContext& cx, const uint8_t* p, int64_t avail, const std::string& where) {
    auto fault = [&](const std::string& m) { throw ExecError(B200Q_ERR_INVALID_ARG, "BLOOM_FILTER state " + where + ": " + m); };
    if (avail < 12) fault(std::to_string(avail) + " bytes, shorter than the 12-byte header");
    uint8_t h[12];
    B200Q_CUDA(cudaMemcpyAsync(h, p, 12, cudaMemcpyDeviceToHost, cx.stream));
    B200Q_CUDA(cudaStreamSynchronize(cx.stream));
    cx.m.d2h_bytes += 12;
    const int32_t version = be32(h), k = be32(h + 4), words = be32(h + 8);
    if (version != 1) fault("unsupported version " + std::to_string(version) + " (expected 1)");
    if (k <= 0) fault("num_hash_functions " + std::to_string(k) + " is not positive");
    if (words <= 0) fault("num_words " + std::to_string(words) + " is not positive");
    if ((int64_t)words * 64 > 0x7FFFFFFF) fault("num_words " + std::to_string(words) + " makes more than INT32_MAX bits");
    if (12 + 8 * (int64_t)words > avail) fault(std::to_string(avail) + " bytes where num_words " + std::to_string(words) + " needs " + std::to_string(12 + 8 * (int64_t)words));
    return BloomHeader{k, words};
  }

  // put_all of the filter serialized at device address p into accumulator i
  void merge_into(OpContext& cx, size_t i, const uint8_t* p, const BloomHeader& h) {
    Acc& a = acc_[i];
    if (!a.bits) a = new_acc(cx, h.nwords, h.k);
    else if (a.k != h.k || a.nwords != h.nwords)
      throw ExecError(B200Q_ERR_INVALID_ARG, "BLOOM_FILTER " + aggs_[i].field_name + ": merging a filter of k=" + std::to_string(h.k) + ", " +
                      std::to_string(64 * h.nwords) + " bits into one of k=" + std::to_string(a.k) + ", " + std::to_string(64 * a.nwords) +
                      " bits (put_all needs equal k and size)");
    cx.m.launches += launch_bloom_merge(p + 12, (unsigned long long*)a.bits->ptr, h.nwords, cx.stream);
  }

  void merge_batch(OpContext& cx, const DevBatch& in) {
    const int64_t n = in.num_rows;
    for (size_t s = 0; s < state_cols_.size(); s++) {
      const DevColumn& c = in.cols[(size_t)state_cols_[s]];
      std::vector<int32_t> offs((size_t)n + 1);
      B200Q_CUDA(cudaMemcpyAsync(offs.data(), (const int32_t*)c.offsets->ptr + c.offset, (size_t)(n + 1) * 4, cudaMemcpyDeviceToHost, cx.stream));
      std::vector<uint8_t> vb;
      if (c.validity) {
        vb.resize((size_t)((c.offset + n + 7) / 8));
        B200Q_CUDA(cudaMemcpyAsync(vb.data(), c.validity->ptr, vb.size(), cudaMemcpyDeviceToHost, cx.stream));
      }
      B200Q_CUDA(cudaStreamSynchronize(cx.stream));
      cx.m.d2h_bytes += (int64_t)(offs.size() * 4 + vb.size());
      const uint8_t* data = (const uint8_t*)c.values->ptr;
      for (int64_t r = 0; r < n; r++) {
        const uint64_t bi = (uint64_t)(c.offset + r);
        if (c.validity && !((vb[bi >> 3] >> (bi & 7)) & 1)) continue;                  // a NULL state: None
        int64_t pos = offs[(size_t)r];
        const int64_t end = offs[(size_t)r + 1];
        const std::string where = "row " + std::to_string(r);
        if (columnar_) {
          const BloomHeader h = read_header(cx, data + pos, end - pos, where);
          if (12 + 8 * h.nwords != end - pos) throw ExecError(B200Q_ERR_INVALID_ARG, "BLOOM_FILTER state " + where + ": " + std::to_string(end - pos) + " bytes where num_words " + std::to_string(h.nwords) + " needs " + std::to_string(12 + 8 * h.nwords));
          merge_into(cx, s, data + pos, h);
          continue;
        }
        for (size_t i = 0; i < aggs_.size(); i++) {                                      // the frozen rows of the aggregates, in order
          if (pos >= end) throw ExecError(B200Q_ERR_INVALID_ARG, "BLOOM_FILTER state " + where + ": truncated accumulator row");
          uint8_t flag;
          B200Q_CUDA(cudaMemcpyAsync(&flag, data + pos, 1, cudaMemcpyDeviceToHost, cx.stream));
          B200Q_CUDA(cudaStreamSynchronize(cx.stream));
          pos += 1;
          if (flag == 0) continue;
          if (flag != 1) throw ExecError(B200Q_ERR_INVALID_ARG, "BLOOM_FILTER state " + where + ": accumulator flag " + std::to_string(flag) + " (expected 0 or 1)");
          const BloomHeader h = read_header(cx, data + pos, end - pos, where);
          merge_into(cx, i, data + pos, h);
          pos += 12 + 8 * h.nwords;
        }
        if (pos != end) throw ExecError(B200Q_ERR_INVALID_ARG, "BLOOM_FILTER state " + where + ": " + std::to_string(end - pos) + " bytes after the last accumulator");
      }
    }
  }

  // shrink_to_fit (spark_bloom_filter.rs): shrunk = next_pow2(max(1, k * true_count * 2)); fold bit i to i mod shrunk when smaller
  void shrink(OpContext& cx, Acc& a) {
    DevMemP cnt = DevMem::alloc(8, cx.stream, true);
    cx.m.launches += launch_bloom_popcount((const unsigned long long*)a.bits->ptr, a.nwords, (unsigned long long*)cnt->ptr, cx.stream);
    unsigned long long trues = 0;
    B200Q_CUDA(cudaMemcpyAsync(&trues, cnt->ptr, 8, cudaMemcpyDeviceToHost, cx.stream));
    B200Q_CUDA(cudaStreamSynchronize(cx.stream));
    unsigned long long want = std::max<unsigned long long>(1, (unsigned long long)a.k * trues * 2), shrunk = 1;
    while (shrunk < want) shrunk <<= 1;
    if (shrunk >= (unsigned long long)(64 * a.nwords)) return;
    Acc s = new_acc(cx, (int64_t)((shrunk + 63) / 64), a.k);
    cx.m.launches += launch_bloom_fold((const unsigned long long*)a.bits->ptr, a.nwords, (unsigned long long*)s.bits->ptr, (int64_t)shrunk, cx.stream);
    a = s;
  }

  // write_to of `a` at device address dst (12 + 8 * nwords bytes)
  void write_to(OpContext& cx, const Acc& a, uint8_t* dst) {
    uint8_t h[12];
    const int32_t v[3] = {1, a.k, (int32_t)a.nwords};
    for (int f = 0; f < 3; f++) for (int j = 0; j < 4; j++) h[4 * f + j] = (uint8_t)((uint32_t)v[f] >> (24 - 8 * j));
    B200Q_CUDA(cudaMemcpyAsync(dst, h, 12, cudaMemcpyHostToDevice, cx.stream));
    cx.m.launches += launch_bloom_write((const unsigned long long*)a.bits->ptr, a.nwords, dst + 12, cx.stream);
    B200Q_CUDA(cudaStreamSynchronize(cx.stream));                     // `h` lives on this stack frame
  }

  // a one-row Binary column of `bytes` bytes (filled by `fill` at the data address), or NULL
  DevColumn binary_row(OpContext& cx, int64_t bytes, bool null, const std::function<void(uint8_t*)>& fill) {
    DevColumn c; c.type.id = T_BINARY;
    c.values = DevMem::alloc((size_t)std::max<int64_t>(bytes, 1) + 16, cx.stream);
    const int32_t offs[2] = {0, null ? 0 : (int32_t)bytes};
    c.offsets = DevMem::alloc(8, cx.stream);
    B200Q_CUDA(cudaMemcpyAsync(c.offsets->ptr, offs, 8, cudaMemcpyHostToDevice, cx.stream));
    if (null) c.validity = DevMem::alloc(bitmap_bytes(1), cx.stream, true);
    else fill((uint8_t*)c.values->ptr);
    B200Q_CUDA(cudaStreamSynchronize(cx.stream));                     // `offs` lives on this stack frame
    return c;
  }

 public:
  BloomAggStage(OpContext& cx, const SchemaDef& in, const PlanNode& node, const std::vector<int>& value_cols) {
    in_schema = in; aggs_ = node.aggs; value_cols_ = value_cols;
    update_ = node.need_partial_update; final_ = node.need_final_merge;
    columnar_ = cx.conf.partial_state_columnar != 0;
    if (node.need_partial_update && node.need_partial_merge) throw PlanError(B200Q_ERR_UNSUPPORTED, "BLOOM_FILTER in Partial next to PartialMerge mode in one AggExec is not on the hot path");
    if (update_) {
      if (value_cols_.size() != aggs_.size()) throw PlanError(B200Q_ERR_INVALID_PLAN, "BLOOM_FILTER: one value per aggregate");
      for (int c : value_cols_) {
        if (!in.fields[(size_t)c].type.is_integer()) throw PlanError(B200Q_ERR_UNSUPPORTED, "BLOOM_FILTER over a " + in.fields[(size_t)c].type.str() + " value");
        used_input_cols.push_back(c);
      }
    } else if (columnar_) {
      for (auto& a : aggs_) {
        const int c = in.index_of(a.field_name);
        if (c < 0 || in.fields[(size_t)c].type.id != T_BINARY) throw PlanError(B200Q_ERR_INVALID_PLAN, "BLOOM_FILTER " + a.field_name + ": no Binary state column of that name in the input");
        state_cols_.push_back(c);
      }
    } else {
      if (in.fields.empty() || in.fields.back().type.id != T_BINARY) throw PlanError(B200Q_ERR_INVALID_PLAN, "BLOOM_FILTER: the input's last column must be the Binary agg-buffer column");
      state_cols_.push_back((int)in.fields.size() - 1);
    }
    for (int c : state_cols_) used_input_cols.push_back(c);
    std::sort(used_input_cols.begin(), used_input_cols.end());
    used_input_cols.erase(std::unique(used_input_cols.begin(), used_input_cols.end()), used_input_cols.end());
    out_schema = node.schema;
    if (!final_ && columnar_) {
      out_schema.fields.clear();
      DType b; b.id = T_BINARY;
      for (auto& a : aggs_) out_schema.fields.push_back(FieldDef{a.field_name, b, true});
    }
    acc_.resize(aggs_.size());
  }

  void push(OpContext& cx, DevBatch& in, std::vector<DevBatch>&) override {
    const int64_t n = in.num_rows;
    if (n == 0) return;
    B200Q_CUDA(cudaEventRecord(cx.ev0, cx.stream));
    if (update_) {
      for (size_t i = 0; i < aggs_.size(); i++) {
        const AggDef& a = aggs_[i];
        if (!acc_[i].bits) acc_[i] = new_acc(cx, (a.bloom_num_bits + 63) / 64, a.bloom_k);   // partial_update creates the filter
        const DevColumn& c = in.cols[(size_t)value_cols_[i]];
        cx.m.launches += launch_bloom_put(dev_col_of(c), (uint8_t)phys_of(c.type), n, (unsigned long long*)acc_[i].bits->ptr,
                                          (int32_t)(64 * acc_[i].nwords), acc_[i].k, cx.stream);
      }
    } else {
      merge_batch(cx, in);
    }
    B200Q_CUDA(cudaEventRecord(cx.ev1, cx.stream));
    B200Q_CUDA(cudaGetLastError());
    B200Q_CUDA(cudaStreamSynchronize(cx.stream));
    add_kernel_time(cx, n, cx.cur_stage == 0);
  }

  void finish(OpContext& cx, std::vector<DevBatch>& outs) override {
    DevBatch ob; ob.num_rows = 1;                                     // no grouping keys: one row, also without input
    if (final_) {
      for (auto& a : acc_) {
        if (a.bits) shrink(cx, a);
        ob.cols.push_back(binary_row(cx, a.bits ? 12 + 8 * a.nwords : 0, !a.bits, [&](uint8_t* d) { write_to(cx, a, d); }));
      }
    } else if (columnar_) {
      for (auto& a : acc_) ob.cols.push_back(binary_row(cx, a.bits ? 12 + 8 * a.nwords : 0, !a.bits, [&](uint8_t* d) { write_to(cx, a, d); }));
    } else {
      int64_t bytes = 0;
      for (auto& a : acc_) bytes += a.bits ? 13 + 8 * a.nwords : 1;
      ob.cols.push_back(binary_row(cx, bytes, false, [&](uint8_t* d) {
        int64_t pos = 0;
        for (auto& a : acc_) {
          const uint8_t f = a.bits ? 1 : 0;
          B200Q_CUDA(cudaMemcpyAsync(d + pos, &f, 1, cudaMemcpyHostToDevice, cx.stream));
          B200Q_CUDA(cudaStreamSynchronize(cx.stream));
          pos += 1;
          if (a.bits) { write_to(cx, a, d + pos); pos += 12 + 8 * a.nwords; }
        }
      }));
    }
    outs.push_back(std::move(ob));
  }
};

}  // namespace

std::unique_ptr<Stage> make_bloom_agg_stage(OpContext& cx, const SchemaDef& in_schema, const PlanNode& agg, const std::vector<int>& value_cols) {
  return std::unique_ptr<Stage>(new BloomAggStage(cx, in_schema, agg, value_cols));
}

}  // namespace b200q
