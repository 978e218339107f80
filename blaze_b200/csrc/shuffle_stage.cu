// ShuffleWriteStage: the terminal stage of a plan rooted at ShuffleWriterExecNode (SURVEY.md §8(f) rank 1).
//
// Reference behaviour restated (paths relative to the reference's native-engine/datafusion-ext-plans/src/):
//   ShuffleWriterExec::execute            shuffle_writer_exec.rs:109-165   (repartitioner by partitioning kind; empty output stream)
//   SortShuffleRepartitioner              shuffle/sort_repartitioner.rs:121-185 (insert_batch -> BufferedData; shuffle_write: .data + .index)
//   BufferedData::write                   shuffle/buffered_data.rs:123-158 (per partition: batches -> IpcCompressionWriter, finish_current_buf)
//   SingleShuffleRepartitioner            shuffle/single_repartitioner.rs:66-99
//   IpcCompressionWriter                  common/ipc_compression.rs:34-112 (blocks of u32 LE length ‖ LZ4 frame)
// GPU side (kernels_shuffle.cu): every pushed batch ("chunk") is partitioned and encoded into the uncompressed
// batch_serde bytes of each partition in ONE device buffer; the chunks' bytes are brought to the host, and finish()
// frames them per partition into compression blocks (host threads, lz4_frame.cc) and writes the two files exactly as
// the no-spill branch of shuffle_write does.  A partition of the file = the blocks of chunk 0, chunk 1, ... for it —
// the same shape the reference produces when it merges spills (sort_repartitioner.rs:226-246).
// Binary columns (the frozen accumulator rows AggExec(Partial) emits in the reference format) are encoded too: such a chunk sums
// its data bytes first, then cuts records of compute_suggested_batch_size_for_output rows and brings back every record's offset,
// so the compression blocks end on record boundaries (kernels_shuffle.cu, "batches with Binary columns").
// Not on the GPU path (B200Q_ERR_UNSUPPORTED -> the host keeps its CPU operator, INTEGRATION.md §3): range and
// round-robin partitioning (they need the sort operator first, shuffle_writer_exec.rs:133-158), Utf8 / Null / nested columns,
// Binary hash keys, more than 4096 partitions, codec zstd.
#include <algorithm>
#include <atomic>
#include <cstdio>
#include <cstring>
#include <thread>

#include "kernels_shuffle.cuh"
#include "lz4_frame.h"
#include "runtime.h"

namespace b200q {

namespace {

struct ShuffleChunk {
  int64_t rows = 0;
  std::vector<unsigned long long> part_off, part_rows;      // host copies: P + 1 byte offsets, P row counts
  std::vector<unsigned long long> rec_start, rec_off;       // chunks with Binary columns: first record of each partition (P + 1), record offsets (R + 1)
  std::vector<uint8_t> host;                                // encoded bytes (shuffle_output_to_host)
  DevMemP dev;                                              // encoded bytes in HBM (kept when the result stays on the device)
};

class ShuffleWriteStage : public Stage, public ShuffleResult {
  ShufSpec base_{};
  std::vector<int> hash_cols_;
  int P_ = 1;
  bool any_bits_ = false;
  std::vector<int> varlen_cols_;                            // Binary columns, ascending
  std::string data_file_, index_file_;
  std::vector<ShuffleChunk> chunks_;
  std::vector<uint64_t> file_offsets_;
  DevMemP d_small_;                                         // counts | part_off | cursors

 public:
  ShuffleWriteStage(OpContext& cx, const SchemaDef& in, const PlanNode& node) {
    in_schema = in; out_schema = in;                        // ShuffleWriterExec::schema() = input schema (shuffle_writer_exec.rs:76-78); the stream is empty
    P_ = node.shuffle_kind == SHUFFLE_SINGLE ? 1 : (int)node.num_partitions;
    if (node.shuffle_kind == SHUFFLE_ROUND_ROBIN && P_ > 1) throw PlanError(B200Q_ERR_UNSUPPORTED, "round-robin shuffle partitioning sorts its input first (shuffle_writer_exec.rs:133-158): not on the GPU path");
    if (node.shuffle_kind == SHUFFLE_RANGE && P_ > 1) throw PlanError(B200Q_ERR_UNSUPPORTED, "range shuffle partitioning is not on the GPU path");
    if (P_ < 1) throw PlanError(B200Q_ERR_INVALID_PLAN, "shuffle writer with zero output partitions");
    if (P_ > SHUF_MAX_PARTS) throw PlanError(B200Q_ERR_UNSUPPORTED, "more than 4096 shuffle partitions");
    if (in.fields.size() > (size_t)SHUF_MAX_COLS) throw PlanError(B200Q_ERR_UNSUPPORTED, "more than 32 columns in a shuffled batch");
    data_file_ = node.data_file; index_file_ = node.index_file;
    base_.ncols = (int)in.fields.size(); base_.num_partitions = P_;
    base_.batch_size = cx.conf.batch_size > 0 ? cx.conf.batch_size : 10000;
    uint32_t k8 = 0, kw = 0;
    for (size_t i = 0; i < in.fields.size(); i++) {
      const FieldDef& f = in.fields[i];
      const bool binary = f.type.id == T_BINARY;
      if ((f.type.is_varlen() && !binary) || f.type.id == T_NULL) throw PlanError(B200Q_ERR_UNSUPPORTED, "shuffle of a " + f.type.str() + " column is not on the GPU path");
      ShufCol& c = base_.col[i];
      c.width = binary ? 4 : (uint8_t)f.type.byte_width(); c.nullable = f.nullable ? 1 : 0; c.k8 = k8; c.kw = kw;      // Binary: its int32 length planes
      c.varlen = binary ? 1 : 0;
      if (binary) varlen_cols_.push_back((int)i);
      if (c.nullable) k8++;
      if (c.width == 0) k8++; else kw += c.width;
      any_bits_ = any_bits_ || c.nullable || c.width == 0;
      used_input_cols.push_back((int)i);
    }
    base_.tot_k8 = k8; base_.tot_kw = kw;
    if (P_ > 1) {
      if (node.hash_exprs.empty()) throw PlanError(B200Q_ERR_INVALID_PLAN, "hash repartition without expressions");
      if (node.hash_exprs.size() > 8) throw PlanError(B200Q_ERR_UNSUPPORTED, "more than 8 hash partitioning expressions");
      for (auto& e : node.hash_exprs) {
        if (e->kind != E_COLUMN) throw PlanError(B200Q_ERR_UNSUPPORTED, "hash partitioning on a computed expression (project it first)");
        if (e->type.is_varlen()) throw PlanError(B200Q_ERR_UNSUPPORTED, "hash partitioning on a " + e->type.str() + " column (murmur3 over bytes) is not on the GPU path");
        base_.key_col[base_.nkeys] = (int8_t)e->col_index; base_.key_phys[base_.nkeys] = (uint8_t)phys_of(e->type); base_.nkeys++;
      }
    }
    d_small_ = DevMem::alloc((size_t)(3 * P_ + 1) * 8, cx.stream);
  }

  void push(OpContext& cx, DevBatch& in, std::vector<DevBatch>&) override {
    const int64_t step = std::max<int64_t>(1, std::min<int64_t>(cx.conf.max_launch_rows > 0 ? cx.conf.max_launch_rows : (1LL << 27), 1LL << 27));
    for (int64_t r0 = 0; r0 < in.num_rows; r0 += step) encode_chunk(cx, in, r0, std::min(step, in.num_rows - r0));
  }

  void encode_chunk(OpContext& cx, DevBatch& in, int64_t r0, int64_t n) {
    if (!varlen_cols_.empty()) { encode_chunk_varlen(cx, in, r0, n); return; }
    ShufSpec sp = base_;
    for (int i = 0; i < sp.ncols; i++) {
      const DevColumn& dc = in.cols[i]; ShufCol& c = sp.col[i];
      const int64_t off = dc.offset + r0;
      if (off > 0xFFFFFFFFLL) throw ExecError(B200Q_ERR_UNSUPPORTED, "column offset beyond 2^32 rows");
      if (!dc.values) throw ExecError(B200Q_ERR_INVALID_ARG, "shuffle: column without a values buffer");
      c.values = c.width ? (const uint8_t*)dc.values->ptr + (size_t)off * c.width : (const uint8_t*)dc.values->ptr;
      c.validity = dc.validity ? (const uint8_t*)dc.validity->ptr : nullptr;
      c.bit_offset = (uint32_t)off;
      if (dc.validity && !c.nullable) throw ExecError(B200Q_ERR_INVALID_ARG, "shuffle: validity bitmap on a column the schema declares non-nullable");
    }
    unsigned long long* d_counts = (unsigned long long*)d_small_->ptr;
    unsigned long long* d_part_off = d_counts + P_;
    unsigned long long* d_cursors = d_part_off + P_ + 1;
    // every partition adds at most one short record per chunk: an upper bound of the encoded size that needs no host round trip
    const unsigned long long nrec_max = (unsigned long long)n / (unsigned long long)sp.batch_size + (unsigned long long)P_;
    const unsigned long long cap = (unsigned long long)sp.tot_kw * (unsigned long long)n + (unsigned long long)sp.tot_k8 * ((unsigned long long)n / 8 + nrec_max) +
                                   (unsigned long long)(5 + sp.ncols) * nrec_max + 64;
    DevMemP d_out = DevMem::alloc((size_t)cap, cx.stream);
    DevMemP d_pids = P_ > 1 ? DevMem::alloc((size_t)n * 2 + 16, cx.stream) : nullptr;
    B200Q_CUDA(cudaEventRecord(cx.ev0, cx.stream));
    B200Q_CUDA(cudaMemsetAsync(d_counts, 0, (size_t)P_ * 8, cx.stream));
    if (P_ > 1) cx.m.launches += launch_shuffle_pids(sp, n, (uint16_t*)d_pids->ptr, d_counts, cx.stream);
    else { const unsigned long long nn = (unsigned long long)n; B200Q_CUDA(cudaMemcpyAsync(d_counts, &nn, 8, cudaMemcpyHostToDevice, cx.stream)); }
    if (any_bits_) B200Q_CUDA(cudaMemsetAsync(d_out->ptr, 0, (size_t)cap, cx.stream));      // bit regions are OR-ed into
    cx.m.launches += launch_shuffle_layout(sp, d_counts, d_part_off, d_cursors, (uint8_t*)d_out->ptr, cx.stream);
    cx.m.launches += launch_shuffle_encode(sp, P_ > 1 ? (const uint16_t*)d_pids->ptr : nullptr, n, d_counts, d_part_off, d_cursors, (uint8_t*)d_out->ptr, cx.stream);
    cx.m.fast_launches++;
    B200Q_CUDA(cudaEventRecord(cx.ev1, cx.stream));
    ShuffleChunk ch; ch.rows = n; ch.part_off.resize((size_t)P_ + 1); ch.part_rows.resize((size_t)P_);
    B200Q_CUDA(cudaMemcpyAsync(ch.part_rows.data(), d_counts, (size_t)P_ * 8, cudaMemcpyDeviceToHost, cx.stream));
    B200Q_CUDA(cudaMemcpyAsync(ch.part_off.data(), d_part_off, (size_t)(P_ + 1) * 8, cudaMemcpyDeviceToHost, cx.stream));
    B200Q_CUDA(cudaStreamSynchronize(cx.stream));
    add_kernel_time(cx, n, cx.cur_stage == 0);
    const unsigned long long total = ch.part_off[(size_t)P_];
    if (total > cap) throw ExecError(B200Q_ERR_EXECUTION, "internal: encoded shuffle chunk larger than its bound");
    if (cx.conf.shuffle_output_on_device) ch.dev = d_out;
    else {
      ch.host.resize((size_t)total);
      if (total) B200Q_CUDA(cudaMemcpyAsync(ch.host.data(), d_out->ptr, (size_t)total, cudaMemcpyDeviceToHost, cx.stream));
      B200Q_CUDA(cudaStreamSynchronize(cx.stream));
      cx.m.d2h_bytes += (int64_t)total;
    }
    chunks_.push_back(std::move(ch));
  }

  // rows per record of a chunk with Binary columns: compute_suggested_batch_size_for_output (datafusion-ext-commons/src/lib.rs:93-116)
  // over the chunk's Arrow buffer bytes (get_batch_mem_size: offsets, data, values, validity)
  int64_t varlen_batch_size(int64_t n, unsigned long long data_bytes) const {
    unsigned long long mem = data_bytes;
    for (int c = 0; c < base_.ncols; c++) {
      const ShufCol& col = base_.col[c];
      mem += col.varlen ? 4ull * (unsigned long long)(n + 1) : col.width ? (unsigned long long)col.width * (unsigned long long)n : (unsigned long long)(n + 7) / 8;
      mem += (unsigned long long)(n + 7) / 8;
    }
    const unsigned long long per_row = std::max<unsigned long long>(mem, 16) / (unsigned long long)std::max<int64_t>(n, 1);
    const unsigned long long sub = (8ull << 20) / std::max<unsigned long long>(per_row, 16);
    return (int64_t)std::max<unsigned long long>(20, std::min<unsigned long long>(sub, (unsigned long long)base_.batch_size));
  }

  // Binary columns: the record sizes depend on the data.  Pass 1 sums the data bytes (brought back with the partition counts in one
  // round trip); the host then fixes the rows per record, the record count and the buffer size, and the device assigns every row its
  // sorted position once, scans the lengths in that order (64-bit), sizes and places the records and writes them.
  void encode_chunk_varlen(OpContext& cx, DevBatch& in, int64_t r0, int64_t n) {
    ShufSpec sp = base_;
    ShufVarlen vl{};
    vl.n = n; vl.nb = (int)varlen_cols_.size();
    for (int i = 0; i < sp.ncols; i++) {
      const DevColumn& dc = in.cols[i]; ShufCol& c = sp.col[i];
      const int64_t off = dc.offset + r0;
      if (off > 0xFFFFFFFFLL) throw ExecError(B200Q_ERR_UNSUPPORTED, "column offset beyond 2^32 rows");
      if (!dc.values) throw ExecError(B200Q_ERR_INVALID_ARG, "shuffle: column without a values buffer");
      if (dc.validity && !c.nullable) throw ExecError(B200Q_ERR_INVALID_ARG, "shuffle: validity bitmap on a column the schema declares non-nullable");
      c.validity = dc.validity ? (const uint8_t*)dc.validity->ptr : nullptr;
      c.bit_offset = (uint32_t)off;
      if (c.varlen) {
        if (!dc.offsets) throw ExecError(B200Q_ERR_INVALID_ARG, "shuffle: Binary column without an offsets buffer");
        c.values = dc.values->ptr;                                                  // the data base the offsets index
        const int k = (int)(std::find(varlen_cols_.begin(), varlen_cols_.end(), i) - varlen_cols_.begin());
        vl.col[k] = (int8_t)i; vl.offsets[k] = (const int32_t*)dc.offsets->ptr + off;
      } else {
        c.values = c.width ? (const uint8_t*)dc.values->ptr + (size_t)off * c.width : (const uint8_t*)dc.values->ptr;
      }
    }
    const size_t P1 = (size_t)P_ + 1, nb = (size_t)vl.nb;
    unsigned long long* d_counts = (unsigned long long*)d_small_->ptr;
    unsigned long long* d_part_off = d_counts + P_;
    unsigned long long* d_cursors = d_part_off + P_ + 1;
    DevMemP d_meta = DevMem::alloc((2 * P1 + nb + 1) * 8, cx.stream);           // row_start | rec_start | totals | err
    unsigned long long* d_row_start = (unsigned long long*)d_meta->ptr;
    unsigned long long* d_rec_start = d_row_start + P1;
    unsigned long long* d_totals = d_rec_start + P1;
    DevMemP d_pids = P_ > 1 ? DevMem::alloc((size_t)n * 2 + 16, cx.stream) : nullptr;
    B200Q_CUDA(cudaEventRecord(cx.ev0, cx.stream));
    B200Q_CUDA(cudaMemsetAsync(d_counts, 0, (size_t)P_ * 8, cx.stream));
    B200Q_CUDA(cudaMemsetAsync(d_totals, 0, (nb + 1) * 8, cx.stream));
    if (P_ > 1) cx.m.launches += launch_shuffle_pids(sp, n, (uint16_t*)d_pids->ptr, d_counts, cx.stream);
    else { const unsigned long long nn = (unsigned long long)n; B200Q_CUDA(cudaMemcpyAsync(d_counts, &nn, 8, cudaMemcpyHostToDevice, cx.stream)); }
    cx.m.launches += launch_shuffle_varlen_bytes(sp, vl, d_totals, cx.stream);
    ShuffleChunk ch; ch.rows = n; ch.part_off.resize(P1); ch.part_rows.resize((size_t)P_);
    std::vector<unsigned long long> totals(nb);
    B200Q_CUDA(cudaMemcpyAsync(ch.part_rows.data(), d_counts, (size_t)P_ * 8, cudaMemcpyDeviceToHost, cx.stream));
    B200Q_CUDA(cudaMemcpyAsync(totals.data(), d_totals, nb * 8, cudaMemcpyDeviceToHost, cx.stream));
    B200Q_CUDA(cudaStreamSynchronize(cx.stream));
    unsigned long long data_bytes = 0;
    for (unsigned long long t : totals) data_bytes += t;
    const unsigned long long B = (unsigned long long)varlen_batch_size(n, data_bytes);
    std::vector<unsigned long long> row_start(2 * P1);                            // row_start | rec_start, uploaded together
    unsigned long long rows = 0, R = 0;
    for (size_t p = 0; p < (size_t)P_; p++) {
      row_start[p] = rows; row_start[P1 + p] = R;
      rows += ch.part_rows[p]; R += (ch.part_rows[p] + B - 1) / B;
    }
    row_start[(size_t)P_] = rows; row_start[P1 + (size_t)P_] = R;
    if (rows != (unsigned long long)n) throw ExecError(B200Q_ERR_EXECUTION, "internal: shuffle partition counts do not add up to the chunk's rows");
    ch.rec_start.assign(row_start.begin() + (ptrdiff_t)P1, row_start.end());
    const unsigned long long cap = (unsigned long long)sp.tot_kw * (unsigned long long)n + (unsigned long long)sp.tot_k8 * ((unsigned long long)n / 8 + R) +
                                   (unsigned long long)(5 + sp.ncols) * R + data_bytes + 64;
    B200Q_CUDA(cudaMemcpyAsync(d_row_start, row_start.data(), 2 * P1 * 8, cudaMemcpyHostToDevice, cx.stream));
    DevMemP d_out = DevMem::alloc((size_t)cap, cx.stream);
    DevMemP d_perm = P_ > 1 ? DevMem::alloc((size_t)n * 4, cx.stream) : nullptr;
    DevMemP d_lens = DevMem::alloc(nb * (size_t)n * 4, cx.stream);
    DevMemP d_doff = DevMem::alloc(nb * (size_t)(n + 1) * 8, cx.stream);
    DevMemP d_recs = DevMem::alloc((size_t)(2 * R + 1) * 8, cx.stream);           // rec_size | rec_off
    DevMemP d_sums = DevMem::alloc((size_t)shuffle_varlen_scan_blocks(std::max<int64_t>(n, (int64_t)R)) * 8 + 16, cx.stream);
    vl.B = (uint32_t)B; vl.R = (long long)R;
    vl.perm = d_perm ? (uint32_t*)d_perm->ptr : nullptr;
    vl.lens = (uint32_t*)d_lens->ptr; vl.doff = (unsigned long long*)d_doff->ptr;
    vl.row_start = d_row_start; vl.rec_start = d_rec_start;
    vl.rec_size = (unsigned long long*)d_recs->ptr; vl.rec_off = vl.rec_size + R;
    vl.sums = (unsigned long long*)d_sums->ptr; vl.err = (unsigned*)(d_totals + nb);
    if (any_bits_) B200Q_CUDA(cudaMemsetAsync(d_out->ptr, 0, (size_t)cap, cx.stream));      // bit regions are OR-ed into
    cx.m.launches += launch_shuffle_varlen_encode(sp, vl, P_ > 1 ? (const uint16_t*)d_pids->ptr : nullptr, d_counts, d_cursors, d_part_off, (uint8_t*)d_out->ptr, cx.stream);
    cx.m.fast_launches++;
    B200Q_CUDA(cudaGetLastError());
    B200Q_CUDA(cudaEventRecord(cx.ev1, cx.stream));
    ch.rec_off.resize((size_t)R + 1);
    unsigned err = 0;
    B200Q_CUDA(cudaMemcpyAsync(ch.part_off.data(), d_part_off, P1 * 8, cudaMemcpyDeviceToHost, cx.stream));
    B200Q_CUDA(cudaMemcpyAsync(ch.rec_off.data(), vl.rec_off, (size_t)(R + 1) * 8, cudaMemcpyDeviceToHost, cx.stream));
    B200Q_CUDA(cudaMemcpyAsync(&err, vl.err, 4, cudaMemcpyDeviceToHost, cx.stream));
    B200Q_CUDA(cudaStreamSynchronize(cx.stream));
    add_kernel_time(cx, n, cx.cur_stage == 0);
    if (err & 1) throw ExecError(B200Q_ERR_UNSUPPORTED, "one shuffle record would carry more than INT32_MAX (2^31 - 1) bytes of Binary data, "
                                                        "the limit of the reader's 32-bit offsets; push smaller batches or lower batch_size");
    const unsigned long long total = ch.part_off[(size_t)P_];
    if (total > cap) throw ExecError(B200Q_ERR_EXECUTION, "internal: encoded shuffle chunk larger than its bound");
    if (cx.conf.shuffle_output_on_device) ch.dev = d_out;
    else {
      ch.host.resize((size_t)total);
      if (total) B200Q_CUDA(cudaMemcpyAsync(ch.host.data(), d_out->ptr, (size_t)total, cudaMemcpyDeviceToHost, cx.stream));
      B200Q_CUDA(cudaStreamSynchronize(cx.stream));
      cx.m.d2h_bytes += (int64_t)total;
    }
    chunks_.push_back(std::move(ch));
  }

  // ---- finish: frame + write (sort_repartitioner.rs:151-185, buffered_data.rs:123-158) ---------------------------------
  // one compression block = whole records of one (chunk, partition) up to ~4 MiB of payload (ipc_compression.rs:77-83 cuts
  // on 0.9 x 4 MiB of *compressed* bytes; where a block ends is not observable by a reader, :129-165)
  void compress_partition(int p, std::vector<uint8_t>& out) const {
    const unsigned long long B = (unsigned long long)base_.batch_size, F = shuf_record_bytes(base_, B);
    constexpr unsigned long long TARGET = 4ull << 20;
    auto block = [&out](const uint8_t* src, unsigned long long blen) {
      const size_t at = out.size();
      out.resize(at + 4);
      lz4_frame_append(src, (size_t)blen, out);
      const uint32_t framed = (uint32_t)(out.size() - at - 4);
      memcpy(out.data() + at, &framed, 4);
    };
    for (const ShuffleChunk& ch : chunks_) {
      const unsigned long long t = ch.part_rows[(size_t)p];
      if (t == 0) continue;
      if (!ch.rec_off.empty()) {                            // Binary columns: records differ in size, cut at the recorded boundaries
        const unsigned long long g1 = ch.rec_start[(size_t)p + 1];
        for (unsigned long long g = ch.rec_start[(size_t)p]; g < g1;) {
          unsigned long long h = g + 1;                     // a record larger than the target is a block of its own
          while (h < g1 && ch.rec_off[h + 1] - ch.rec_off[g] <= TARGET) h++;
          block(ch.host.data() + ch.rec_off[g], ch.rec_off[h] - ch.rec_off[g]);
          g = h;
        }
        continue;
      }
      const uint8_t* src = ch.host.data() + ch.part_off[(size_t)p];
      const unsigned long long len = ch.part_off[(size_t)p + 1] - ch.part_off[(size_t)p];
      const unsigned long long per_block = std::max<unsigned long long>(1, TARGET / F) * F;     // whole records
      for (unsigned long long pos = 0; pos < len; pos += per_block) block(src + pos, std::min(per_block, len - pos));
    }
  }

  void finish(OpContext& cx, std::vector<DevBatch>&) override {
    if (cx.conf.shuffle_output_on_device || data_file_.empty()) return;
    std::vector<std::vector<uint8_t>> comp((size_t)P_);
    std::atomic<int> next{0};
    const unsigned hw = std::thread::hardware_concurrency();
    const int nthreads = (int)std::max(1u, std::min(std::min(hw ? hw : 4u, 32u), (unsigned)P_));
    auto work = [&] { for (int p = next.fetch_add(1); p < P_; p = next.fetch_add(1)) compress_partition(p, comp[(size_t)p]); };
    std::vector<std::thread> th;
    for (int i = 1; i < nthreads; i++) th.emplace_back(work);
    work();
    for (auto& t : th) t.join();
    FILE* fd = fopen(data_file_.c_str(), "wb");
    if (!fd) throw ExecError(B200Q_ERR_EXECUTION, "shuffle write error: cannot open " + data_file_);
    file_offsets_.assign((size_t)P_ + 1, 0);
    uint64_t pos = 0; bool ok = true;
    for (int p = 0; p < P_; p++) {
      file_offsets_[(size_t)p] = pos;
      if (!comp[(size_t)p].empty()) ok = ok && fwrite(comp[(size_t)p].data(), 1, comp[(size_t)p].size(), fd) == comp[(size_t)p].size();
      pos += comp[(size_t)p].size();
    }
    file_offsets_[(size_t)P_] = pos;
    ok = (fclose(fd) == 0) && ok;
    FILE* fi = fopen(index_file_.c_str(), "wb");
    if (!fi) throw ExecError(B200Q_ERR_EXECUTION, "shuffle write error: cannot open " + index_file_);
    for (uint64_t o : file_offsets_) { const int64_t v = (int64_t)o; ok = ok && fwrite(&v, 8, 1, fi) == 1; }     // little-endian i64 (sort_repartitioner.rs:181-185)
    ok = (fclose(fi) == 0) && ok;
    if (!ok) throw ExecError(B200Q_ERR_EXECUTION, "shuffle write error: short write");
  }

  // ---- ShuffleResult ------------------------------------------------------------------------------------------------
  int64_t chunk_count() const override { return (int64_t)chunks_.size(); }
  void chunk(int64_t i, b200q_shuffle_chunk* out) const override {
    const ShuffleChunk& ch = chunks_.at((size_t)i);
    out->num_partitions = P_; out->rows = ch.rows;
    out->on_device = ch.dev ? 1 : 0;
    out->data = ch.dev ? (const uint8_t*)ch.dev->ptr : ch.host.data();
    out->part_off = (const uint64_t*)ch.part_off.data(); out->part_rows = (const uint64_t*)ch.part_rows.data();
  }
};

}  // namespace

std::unique_ptr<Stage> make_shuffle_write_stage(OpContext& cx, const SchemaDef& in_schema, const PlanNode& node) {
  return std::unique_ptr<Stage>(new ShuffleWriteStage(cx, in_schema, node));
}

}  // namespace b200q
