// IpcReaderExec as the SOURCE of an op: the reduce side of a shuffle reads the `u32 LE length ‖ LZ4 frame` blocks the map side
// wrote (ShuffleWriterExec, shuffle_stage.cu) and decodes their batch_serde records into device batches.
//
// Reference: IpcReaderExec::execute (datafusion-ext-plans/src/ipc_reader_exec.rs:164-272) reads each BlockObject through
// IpcCompressionReader (common/ipc_compression.rs:114-183: the decompressed blocks form one stream, a record may straddle two
// blocks) and read_batch (datafusion-ext-commons/src/io/batch_serde.rs:79-99), then coalesces the batches.  Here:
//   host   the blocks of one push are LZ4-decoded on worker threads into pinned blocks (lz4_frame.cc), the records are walked
//          and every extent checked (ipc_records.cc), the blocks are uploaded back to back on the op's stream;
//   device the records of up to conf.staging_rows rows form one flush: ipc_decode_fixed_kernel un-transposes every fixed-width
//          column (and the Binary length planes), ipc_decode_bits_kernel re-packs validity and Boolean bits, an exclusive scan
//          turns the lengths into offsets and ipc_decode_bytes_kernel copies the row bytes (kernels.cu).
// The pinned blocks go back to the pool once their upload has drained (polled at the next push): the next push's decompression
// overlaps the device work of this one.
#include <algorithm>
#include <atomic>
#include <cstring>
#include <thread>

#include "ipc_records.h"
#include "lz4_frame.h"
#include "runtime.h"

namespace b200q {

namespace {

constexpr int64_t IPC_MAX_FLUSH_BYTES = 1LL << 30;        // decoded stream bytes behind one flush
constexpr int64_t IPC_MAX_DATA_BYTES = 0x7FFFFFFFLL;      // Binary / Utf8 bytes of one output column: int32 offsets

inline size_t align16(size_t n) { return (n + 15) & ~(size_t)15; }

struct PinnedGuard {                                       // the pinned blocks of one push until they are handed to a Release
  std::vector<void*> blocks;
  ~PinnedGuard() { for (void* p : blocks) pinned_free(p); }
};
struct Release { cudaEvent_t ev; std::vector<void*> blocks; };

class IpcSourceImpl : public IpcSource {
  SchemaDef schema_;
  std::vector<DType> types_;
  std::vector<int> used_;
  int64_t max_rows_;
  // records of the flush being accumulated: per record its rows, the device address of its push's stream and its extents
  // (used columns only)
  std::vector<int64_t> rows_;
  std::vector<const uint8_t*> base_;
  std::vector<IpcColExtent> ext_;
  std::vector<int64_t> data_bytes_;                        // per used column: Binary / Utf8 bytes so far
  int64_t total_rows_ = 0, stream_bytes_ = 0;
  std::vector<DevMemP> keep_;                              // the uploaded streams the records point into
  std::vector<Release> releases_;
  cudaEvent_t ev_a_ = nullptr, ev_b_ = nullptr;
  bool timing_pending_ = false;

  void poll_releases(bool wait) {
    for (size_t i = 0; i < releases_.size();) {
      const cudaError_t q = wait ? cudaEventSynchronize(releases_[i].ev) : cudaEventQuery(releases_[i].ev);
      if (q == cudaErrorNotReady) { i++; continue; }
      for (void* p : releases_[i].blocks) pinned_free(p);
      cudaEventDestroy(releases_[i].ev);
      releases_.erase(releases_.begin() + (ptrdiff_t)i);
    }
  }
  void collect_timing(OpContext& cx) {
    if (!timing_pending_) return;
    B200Q_CUDA(cudaEventSynchronize(ev_b_));
    float ms = 0; B200Q_CUDA(cudaEventElapsedTime(&ms, ev_a_, ev_b_)); cx.m.gpu_ms += ms;
    timing_pending_ = false;
  }

 public:
  IpcSourceImpl(OpContext& cx, const SchemaDef& s, const std::vector<int>& used) : schema_(s), used_(used) {
    for (auto& f : s.fields) types_.push_back(f.type);
    max_rows_ = cx.conf.staging_rows > 0 ? cx.conf.staging_rows : (1 << 20);
    data_bytes_.assign(used_.size(), 0);
    B200Q_CUDA(cudaEventCreate(&ev_a_)); B200Q_CUDA(cudaEventCreate(&ev_b_));
  }
  ~IpcSourceImpl() override {
    poll_releases(true);
    if (ev_a_) cudaEventDestroy(ev_a_);
    if (ev_b_) cudaEventDestroy(ev_b_);
  }

  void push(OpContext& cx, const uint8_t* data, size_t len, const std::function<void(DevBatch&)>& emit) override {
    poll_releases(false);
    // ---- framing: u32 LE length ‖ LZ4 frame (ipc_compression.rs:129-165)
    struct Blk { const uint8_t* src; size_t n, at, bound; uint8_t* out = nullptr; size_t len = 0; std::string err; size_t err_off = 0; };
    std::vector<Blk> blks;
    for (size_t pos = 0; pos < len;) {
      if (len - pos < 4) throw ExecError(B200Q_ERR_INVALID_ARG, "push_ipc: truncated block length at byte " + std::to_string(pos) + " of the push");
      uint32_t bl; memcpy(&bl, data + pos, 4);
      if (bl > len - pos - 4) throw ExecError(B200Q_ERR_INVALID_ARG, "push_ipc: the block at byte " + std::to_string(pos) + " of the push declares " + std::to_string(bl) + " bytes, " + std::to_string(len - pos - 4) + " follow");
      const uint8_t* f = data + pos + 4;
      if (bl >= 4 && f[0] == 0x28 && f[1] == 0xB5 && f[2] == 0x2F && f[3] == 0xFD)
        throw ExecError(B200Q_ERR_UNSUPPORTED, "push_ipc: the block at byte " + std::to_string(pos) + " is a zstd frame; only the lz4 codec is on the GPU path");
      Blk b; b.src = f; b.n = bl; b.at = pos + 4;
      try { b.bound = lz4_frame_bound(f, bl); }
      catch (const Lz4FrameError& e) { throw ExecError(B200Q_ERR_INVALID_ARG, std::string("push_ipc: ") + e.what() + " at byte " + std::to_string(b.at + e.offset) + " of the push"); }
      blks.push_back(b);
      pos += 4 + (size_t)bl;
    }
    // ---- decompression into pinned blocks, in parallel
    PinnedGuard guard;
    for (auto& b : blks) {
      b.out = (uint8_t*)pinned_alloc(std::max<size_t>(b.bound, 1));
      if (!b.out) throw ExecError(B200Q_ERR_EXECUTION, "push_ipc: pinned host allocation of " + std::to_string(b.bound) + " bytes failed");
      guard.blocks.push_back(b.out);
    }
    auto work = [&](size_t i) {
      Blk& b = blks[i];
      try { b.len = lz4_frame_decompress(b.src, b.n, b.out, b.bound); }
      catch (const Lz4FrameError& e) { b.err = e.what(); b.err_off = e.offset; }
    };
    const unsigned hw = std::max(1u, std::thread::hardware_concurrency());
    const size_t nthreads = std::min<size_t>({(size_t)hw, (size_t)32, blks.size()});
    if (nthreads <= 1) for (size_t i = 0; i < blks.size(); i++) work(i);
    else {
      std::atomic<size_t> next{0};
      std::vector<std::thread> th;
      for (size_t t = 0; t < nthreads; t++) th.emplace_back([&] { for (size_t i = next++; i < blks.size(); i = next++) work(i); });
      for (auto& t : th) t.join();
    }
    for (auto& b : blks)
      if (!b.err.empty()) throw ExecError(B200Q_ERR_INVALID_ARG, "push_ipc: " + b.err + " at byte " + std::to_string(b.at + b.err_off) + " of the push");
    // ---- record table over the decompressed stream
    std::vector<IpcSegment> segs;
    size_t total = 0;
    for (auto& b : blks) { segs.push_back(IpcSegment{b.out, b.len}); total += b.len; }
    IpcRecordTable tab; tab.ncols = types_.size();
    try { ipc_walk_records(segs, types_, tab); }
    catch (const IpcRecordError& e) {
      size_t k = 0, acc = 0;
      while (k + 1 < blks.size() && acc + blks[k].len <= e.offset) acc += blks[k++].len;
      throw ExecError(B200Q_ERR_INVALID_ARG, std::string("push_ipc: ") + e.what() + " at byte " + std::to_string(e.offset) + " of the decompressed stream (block at byte " +
                                             std::to_string(blks.empty() ? 0 : blks[k].at - 4) + " of the push)");
    }
    for (size_t r = 0; r < tab.count(); r++)
      for (size_t k = 0; k < used_.size(); k++)
        if (tab.ext[r * tab.ncols + (size_t)used_[k]].data_len > IPC_MAX_DATA_BYTES)
          throw ExecError(B200Q_ERR_UNSUPPORTED, "push_ipc: one record carries more than INT32_MAX (2^31 - 1) bytes of " + types_[(size_t)used_[k]].str() +
                                                 " data in column " + schema_.fields[(size_t)used_[k]].name + ", beyond the 32-bit offsets of a device batch");
    // ---- commit: upload, then queue the records
    if (total == 0) return;
    DevMemP d = DevMem::alloc(total + 16, cx.stream);      // the pad is only over-read by masked bit loads
    size_t off = 0;
    for (auto& b : blks) { if (b.len) B200Q_CUDA(cudaMemcpyAsync((uint8_t*)d->ptr + off, b.out, b.len, cudaMemcpyHostToDevice, cx.stream)); off += b.len; }
    cx.m.h2d_bytes += (int64_t)total;
    Release rel; rel.blocks.swap(guard.blocks);
    B200Q_CUDA(cudaEventCreateWithFlags(&rel.ev, cudaEventDisableTiming));
    releases_.push_back(rel);
    B200Q_CUDA(cudaEventRecord(rel.ev, cx.stream));
    const uint8_t* base = (const uint8_t*)d->ptr;
    for (size_t r = 0; r < tab.count(); r++) {
      const int64_t n = tab.rows[r];
      cx.m.input_rows += n; cx.m.input_batches++;
      if (n == 0) continue;
      const int64_t rec_bytes = (r + 1 < tab.count() ? tab.start[r + 1] : (int64_t)total) - tab.start[r];
      const IpcColExtent* e = &tab.ext[r * tab.ncols];
      bool full = total_rows_ + n > max_rows_ || stream_bytes_ + rec_bytes > IPC_MAX_FLUSH_BYTES;
      for (size_t k = 0; k < used_.size(); k++) full = full || data_bytes_[k] + e[used_[k]].data_len > IPC_MAX_DATA_BYTES;
      if (full && !rows_.empty()) flush_pending(cx, emit);
      if (keep_.empty() || keep_.back() != d) keep_.push_back(d);
      rows_.push_back(n); base_.push_back(base);
      for (size_t k = 0; k < used_.size(); k++) { ext_.push_back(e[used_[k]]); data_bytes_[k] += e[used_[k]].data_len; }
      total_rows_ += n; stream_bytes_ += rec_bytes;
    }
    if (total_rows_ >= max_rows_) flush_pending(cx, emit);
  }

  void flush(OpContext& cx, const std::function<void(DevBatch&)>& emit) override {
    flush_pending(cx, emit);
    collect_timing(cx);
  }

 private:
  void flush_pending(OpContext& cx, const std::function<void(DevBatch&)>& emit) {
    const size_t R = rows_.size(), U = used_.size();
    if (R == 0) return;
    collect_timing(cx);
    std::vector<int64_t> rec_row(R + 1, 0);
    for (size_t r = 0; r < R; r++) rec_row[r + 1] = rec_row[r] + rows_[r];
    const int64_t rows = rec_row[R];
    DevBatch b; b.num_rows = rows; b.cols.resize(schema_.fields.size());
    for (size_t i = 0; i < b.cols.size(); i++) b.cols[i].type = types_[i];
    const size_t words = (size_t)((rows + 31) / 32);
    std::vector<IpcFixedJob> jobs; std::vector<IpcTile> tiles; std::vector<IpcCopy> copies;
    struct BitCol { uint32_t* dst; std::vector<const uint8_t*> src; };
    std::vector<BitCol> bits;
    struct Scan { const int32_t* lengths; int32_t* offsets; };
    std::vector<Scan> scans;
    auto add_job = [&](const uint8_t* src, uint8_t* dst, int64_t n, int w) {
      jobs.push_back(IpcFixedJob{src, dst, n, w, 0});
      for (int64_t r0 = 0; r0 < n; r0 += IPC_TILE) tiles.push_back(IpcTile{(int32_t)(jobs.size() - 1), (int32_t)r0});
    };
    for (size_t k = 0; k < U; k++) {
      const int ci = used_[k];
      const DType& t = types_[(size_t)ci];
      DevColumn& col = b.cols[(size_t)ci];
      bool any_null = false;
      for (size_t r = 0; r < R; r++) any_null = any_null || ext_[r * U + k].valid >= 0;
      if (schema_.fields[(size_t)ci].nullable || any_null) {
        col.validity = DevMem::alloc(words * 4 + 16, cx.stream);
        BitCol bc{(uint32_t*)col.validity->ptr, {}};
        for (size_t r = 0; r < R; r++) { const IpcColExtent& e = ext_[r * U + k]; bc.src.push_back(e.valid >= 0 ? base_[r] + e.valid : nullptr); }
        bits.push_back(std::move(bc));
      }
      if (t.id == T_BOOL) {
        col.values = DevMem::alloc(words * 4 + 16, cx.stream);
        BitCol bc{(uint32_t*)col.values->ptr, {}};
        for (size_t r = 0; r < R; r++) bc.src.push_back(base_[r] + ext_[r * U + k].values);
        bits.push_back(std::move(bc));
      } else if (t.is_varlen()) {
        DevMemP lengths = DevMem::alloc((size_t)rows * 4 + 16, cx.stream);
        col.offsets = DevMem::alloc((size_t)(rows + 1) * 4, cx.stream);
        col.values = DevMem::alloc((size_t)data_bytes_[k] + 16, cx.stream);
        keep_.push_back(lengths);
        int64_t at = 0;
        for (size_t r = 0; r < R; r++) {
          const IpcColExtent& e = ext_[r * U + k];
          add_job(base_[r] + e.values, (uint8_t*)lengths->ptr + rec_row[r] * 4, rows_[r], 4);
          for (int64_t p = 0; p < e.data_len; p += IPC_COPY_PIECE)
            copies.push_back(IpcCopy{base_[r] + e.data + p, (uint8_t*)col.values->ptr + at + p, std::min<int64_t>(IPC_COPY_PIECE, e.data_len - p)});
          at += e.data_len;
        }
        scans.push_back(Scan{(const int32_t*)lengths->ptr, (int32_t*)col.offsets->ptr});
      } else {
        const int w = t.byte_width();
        col.values = DevMem::alloc((size_t)rows * (size_t)w + 16, cx.stream);
        for (size_t r = 0; r < R; r++) add_job(base_[r] + ext_[r * U + k].values, (uint8_t*)col.values->ptr + rec_row[r] * w, rows_[r], w);
      }
    }
    // one table upload: rec_row | jobs | tiles | bit columns | their per-record sources | copies
    const size_t o_row = 0, o_jobs = align16(o_row + (R + 1) * 8), o_tiles = align16(o_jobs + jobs.size() * sizeof(IpcFixedJob)),
                 o_bits = align16(o_tiles + tiles.size() * sizeof(IpcTile)), o_src = align16(o_bits + bits.size() * sizeof(IpcBitCol)),
                 o_copies = align16(o_src + bits.size() * R * sizeof(void*)), tbytes = align16(o_copies + copies.size() * sizeof(IpcCopy));
    DevMemP d_tab = DevMem::alloc(tbytes, cx.stream);
    uint8_t* dt = (uint8_t*)d_tab->ptr;
    std::vector<uint8_t> h(tbytes, 0);
    memcpy(h.data() + o_row, rec_row.data(), (R + 1) * 8);
    if (!jobs.empty()) memcpy(h.data() + o_jobs, jobs.data(), jobs.size() * sizeof(IpcFixedJob));
    if (!tiles.empty()) memcpy(h.data() + o_tiles, tiles.data(), tiles.size() * sizeof(IpcTile));
    for (size_t i = 0; i < bits.size(); i++) {
      const IpcBitCol bc{bits[i].dst, (const uint8_t* const*)(dt + o_src + i * R * sizeof(void*))};
      memcpy(h.data() + o_bits + i * sizeof(IpcBitCol), &bc, sizeof(bc));
      memcpy(h.data() + o_src + i * R * sizeof(void*), bits[i].src.data(), R * sizeof(void*));
    }
    if (!copies.empty()) memcpy(h.data() + o_copies, copies.data(), copies.size() * sizeof(IpcCopy));
    // a pageable source: the call returns once `h` has been staged
    B200Q_CUDA(cudaMemcpyAsync(dt, h.data(), tbytes, cudaMemcpyHostToDevice, cx.stream));
    cx.m.h2d_bytes += (int64_t)tbytes;
    B200Q_CUDA(cudaEventRecord(ev_a_, cx.stream));
    cx.m.launches += launch_ipc_decode_fixed((const IpcFixedJob*)(dt + o_jobs), (const IpcTile*)(dt + o_tiles), (int64_t)tiles.size(), cx.stream);
    cx.m.launches += launch_ipc_decode_bits((const IpcBitCol*)(dt + o_bits), (int)bits.size(), (const int64_t*)(dt + o_row), (int64_t)R, rows, cx.stream);
    if (!scans.empty()) {
      DevMemP sums = DevMem::alloc((size_t)scan_num_blocks(rows) * 4 + 16, cx.stream);
      for (auto& s : scans) cx.m.launches += launch_exclusive_scan_i32(s.lengths, s.offsets, rows, (int32_t*)sums->ptr, cx.stream);
    }
    cx.m.launches += launch_ipc_decode_bytes((const IpcCopy*)(dt + o_copies), (int64_t)copies.size(), cx.stream);
    B200Q_CUDA(cudaGetLastError());
    B200Q_CUDA(cudaEventRecord(ev_b_, cx.stream));
    timing_pending_ = true;
    rows_.clear(); base_.clear(); ext_.clear(); keep_.clear();    // stream-ordered frees: the kernels above still read them
    std::fill(data_bytes_.begin(), data_bytes_.end(), 0);
    total_rows_ = 0; stream_bytes_ = 0;
    emit(b);
  }
};

}  // namespace

std::unique_ptr<IpcSource> make_ipc_source(OpContext& cx, const SchemaDef& schema, const std::vector<int>& used_cols) {
  return std::unique_ptr<IpcSource>(new IpcSourceImpl(cx, schema, used_cols));
}

}  // namespace b200q
