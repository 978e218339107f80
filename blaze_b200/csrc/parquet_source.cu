// ParquetScanExec as the SOURCE of an op (SURVEY.md §8(f) rank 3): footer + page framing on the host (parquet_meta.cc),
// column-chunk decode on the GPU (kernels_parquet.cu), row-group pruning from the min / max statistics.
//
// Reference: ParquetExec::execute (datafusion-ext-plans/src/parquet_exec.rs:150-203) builds DataFusion's ParquetOpener over
// the `parquet` crate (row-group pruning by statistics, optional page filtering); bytes arrive through FsProvider
// (:316-396).  Here: every row group inside the split's byte range is one device batch — its projected column chunks
// are read (local files, or the host's reader callback: b200q_set_file_reader, the counterpart of FsProvider), their pages
// decompressed and described as run tables on the host, and expanded on the device; the batch then flows through the
// stages above the scan (FilterExec / AggExec / ...).  A row group is skipped when a pruning predicate `col cmp literal`
// cannot hold for its [min, max] statistics — an optimisation only: Spark keeps the FilterExec above the scan, so the
// rows that leave the pipeline are the same.
#include <fcntl.h>
#include <unistd.h>

#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <condition_variable>
#include <memory>
#include <mutex>
#include <thread>
#include <unordered_map>

#include "kernels_join.cuh"
#include "kernels_parquet.cuh"
#include "parquet_meta.h"
#include "runtime.h"

namespace b200q {

static b200q_file_reader_fn g_reader = nullptr;
static void* g_reader_ctx = nullptr;
void set_file_reader(b200q_file_reader_fn fn, void* ctx) { g_reader = fn; g_reader_ctx = ctx; }

namespace {

struct FileIo {                                   // positional reads: the column chunks of a row group are read by concurrent host threads
  std::string path; int fd = -1; int64_t size = -1; std::mutex mu;
  explicit FileIo(const std::string& p, uint64_t declared_size) : path(p) {
    if (g_reader) { size = (int64_t)declared_size; return; }
    std::string local = p;
    if (local.rfind("file://", 0) == 0) local = local.substr(7); else if (local.rfind("file:", 0) == 0) local = local.substr(5);
    fd = open(local.c_str(), O_RDONLY);
    if (fd < 0) throw ExecError(B200Q_ERR_EXECUTION, "parquet: cannot open " + p + " (register a reader with b200q_set_file_reader for non-local file systems)");
    size = (int64_t)lseek(fd, 0, SEEK_END);
  }
  ~FileIo() { if (fd >= 0) close(fd); }
  void read(int64_t off, size_t len, uint8_t* dst) {
    if (off < 0 || (int64_t)(off + (int64_t)len) > size) throw ExecError(B200Q_ERR_EXECUTION, "parquet: read past the end of " + path);
    if (g_reader) {                                  // the host's callback is not assumed to be re-entrant
      std::lock_guard<std::mutex> l(mu);
      if (g_reader(g_reader_ctx, path.c_str(), off, (int64_t)len, dst) != 0) throw ExecError(B200Q_ERR_EXECUTION, "parquet: the file reader callback failed for " + path);
      return;
    }
    size_t got = 0;
    while (got < len) { const ssize_t r = pread(fd, dst + got, len - got, (off_t)(off + (int64_t)got)); if (r <= 0) throw ExecError(B200Q_ERR_EXECUTION, "parquet: short read from " + path); got += (size_t)r; }
  }
};

// statistics are PLAIN-encoded single values (little-endian) for INT32 / INT64
bool stat_i64(const PqColumnSchema& cs, const std::string& v, long long& out) {
  if (cs.type == PQ_INT32 && v.size() == 4) { int32_t x; memcpy(&x, v.data(), 4); out = x; return true; }
  if (cs.type == PQ_INT64 && v.size() == 8) { long long x; memcpy(&x, v.data(), 8); out = x; return true; }
  return false;
}

// may the predicate hold for some row of a row group whose column `col` lies in [mn, mx]?  Unknown shapes -> true (keep)
bool may_match(const ExprP& e, const std::vector<int>& file_col_of, const PqFileMeta& meta, const PqRowGroup& rg) {
  if (e->kind == E_BINARY && e->op == OP_AND) return may_match(e->children[0], file_col_of, meta, rg) && may_match(e->children[1], file_col_of, meta, rg);
  if (e->kind == E_BINARY && e->op == OP_OR) return may_match(e->children[0], file_col_of, meta, rg) || may_match(e->children[1], file_col_of, meta, rg);
  if (e->kind != E_BINARY || e->op < OP_EQ || e->op > OP_GE) return true;
  ExprP l = e->children[0], r = e->children[1]; int op = e->op;
  if (l->kind == E_LITERAL && r->kind == E_COLUMN) { std::swap(l, r); static const int flip[] = {OP_EQ, OP_NE, OP_GT, OP_GE, OP_LT, OP_LE}; op = flip[op - OP_EQ]; }
  if (l->kind != E_COLUMN || r->kind != E_LITERAL || r->lit_null || !l->type.is_intlike() || !r->type.is_intlike()) return true;
  const int fc = l->col_index >= 0 && (size_t)l->col_index < file_col_of.size() ? file_col_of[(size_t)l->col_index] : -1;
  if (fc < 0) return true;
  const PqStats& st = rg.columns[(size_t)fc].stats;
  long long mn, mx;
  if (!st.has_min || !st.has_max || !stat_i64(meta.columns[(size_t)fc], st.min, mn) || !stat_i64(meta.columns[(size_t)fc], st.max, mx)) return true;
  const long long v = (long long)r->lit_lo;
  switch (op) {
    case OP_EQ: return v >= mn && v <= mx;
    case OP_LT: return mn < v;
    case OP_LE: return mn <= v;
    case OP_GT: return mx > v;
    case OP_GE: return mx >= v;
    default: return true;                                               // NotEq
  }
}

DevMemP upload(OpContext& cx, const void* p, size_t n, size_t pad = 16) {
  DevMemP d = DevMem::alloc(n + pad, cx.stream);       // the pad is only ever over-read by the funnel-shift loads and masked out: no memset
  if (n) B200Q_CUDA(cudaMemcpyAsync(d->ptr, p, n, cudaMemcpyHostToDevice, cx.stream));
  cx.m.h2d_bytes += (int64_t)n;
  return d;
}

// host half of one column chunk (runs on a worker thread): read, frame + decompress the pages, flatten them into one byte buffer and
// two run tables (levels by row, values by stored-value ordinal)
}  // namespace

// Pinned host blocks outlive a scan: pinning pages costs ~1 ms per MB and a long-lived executor runs scan after scan.  Process-wide pool of
// power-of-two blocks, bounded in bytes (B200Q_SCAN_HOST_CACHE_MB, default 2048); blocks above the bound go back to the driver.
struct PinnedPool {
  std::mutex mu; std::unordered_map<void*, size_t> size_of; std::unordered_map<size_t, std::vector<void*>> free_blocks; size_t cached = 0;
  static size_t budget() { static const size_t b = [] { const char* e = getenv("B200Q_SCAN_HOST_CACHE_MB"); return (size_t)(e ? atoll(e) : 2048) << 20; }(); return b; }
  static size_t size_class(size_t n) { size_t c = (size_t)1 << 18; while (c < n) c <<= 1; return c; }
  void* get(size_t n) {
    const size_t c = size_class(n);
    { std::lock_guard<std::mutex> l(mu); auto it = free_blocks.find(c); if (it != free_blocks.end() && !it->second.empty()) { void* p = it->second.back(); it->second.pop_back(); cached -= c; return p; } }
    void* p = nullptr;
    if (cudaMallocHost(&p, c) != cudaSuccess) { (void)cudaGetLastError(); return nullptr; }
    std::lock_guard<std::mutex> l(mu); size_of[p] = c; return p;
  }
  void put(void* p) {
    { std::lock_guard<std::mutex> l(mu); const size_t c = size_of[p]; if (cached + c <= budget()) { cached += c; free_blocks[c].push_back(p); return; } size_of.erase(p); }
    cudaFreeHost(p);
  }
};
PinnedPool& pinned_pool() { static PinnedPool* p = new PinnedPool(); return *p; }            // leaked on purpose: no pinned frees after the driver is gone
void* pinned_alloc(size_t n) { return pinned_pool().get(n); }
void pinned_free(void* p) { pinned_pool().put(p); }

namespace {

// host half of one column chunk: the file bytes, the decompressed page bodies (what the device reads) and the run tables
struct PreparedChunk {
  ByteBuf raw, bytes, dict_bytes; std::vector<PqDevRun> lruns, vruns;
  size_t dict_off = 0, dict_len = 0, runs_off = 0;          // bytes = page bodies ‖ dictionary ‖ level runs ‖ value runs: ONE pinned buffer, one DMA per chunk
                                                            // (every extra stream operation costs ~10 us of engine hand-over, more than a MB of transfer)
  int32_t dict_count = 0; bool has_dict = false, any_null = false;
  std::string error; int error_code = 0;
  PreparedChunk() { for (ByteBuf* b : {&raw, &bytes}) { b->alloc_fn = pinned_alloc; b->free_fn = pinned_free; } }
};

void prepare_chunk(FileIo& io, const PqColumnChunk& cc, const PqColumnSchema& cs, const DType& want, int64_t rows, PreparedChunk& pc) {
  if (cs.arrow.id == T_NULL) throw ExecError(B200Q_ERR_UNSUPPORTED, "parquet: column " + cs.name + " has a physical / logical type outside the GPU path");
  if (cs.arrow != want) throw ExecError(B200Q_ERR_UNSUPPORTED, "parquet: column " + cs.name + " is " + cs.arrow.str() + " in the file, the plan expects " + want.str() + " (schema adaption stays on the host)");
  pc.lruns.clear(); pc.vruns.clear(); pc.has_dict = pc.any_null = false; pc.dict_count = 0; pc.error.clear(); pc.error_code = 0;
  pc.raw.clear();
  io.read(cc.start(), (size_t)cc.total_compressed_size, pc.raw.grow((size_t)cc.total_compressed_size));
  pc.bytes.reserve((size_t)std::max<int64_t>(cc.total_uncompressed_size, cc.total_compressed_size) + (256u << 10));   // page bodies <= the chunk's uncompressed size: no regrowth of the pinned buffer
  std::vector<PqPage> pages = parquet_read_pages(pc.raw.data(), pc.raw.size(), cc, cs, pc.bytes, pc.dict_bytes);
  int64_t row = 0, ord = 0;
  for (auto& pg : pages) if (pg.type != PQ_DICTIONARY_PAGE && !pg.def_runs.empty()) pc.any_null = true;
  for (auto& pg : pages) {
    if (pg.type == PQ_DICTIONARY_PAGE) { pc.has_dict = true; pc.dict_count = pg.num_values; continue; }
    const uint64_t base = pg.base;
    if (pc.any_null) {
      if (pg.def_runs.empty()) pc.lruns.push_back(PqDevRun{(uint32_t)row, (uint32_t)pg.num_values, PQR_RLE, 1, {}, 1});
      uint32_t at = (uint32_t)row;
      for (auto& r : pg.def_runs) { pc.lruns.push_back(PqDevRun{at, r.count, (uint8_t)(r.is_rle ? PQR_RLE : PQR_BITPACKED), 1, {}, r.is_rle ? r.value_or_bit_offset : base * 8 + r.value_or_bit_offset}); at += r.count; }
    }
    if (pg.non_null > 0) {
      if (!pg.idx_runs.empty()) {
        uint32_t at = (uint32_t)ord;
        for (auto& r : pg.idx_runs) { pc.vruns.push_back(PqDevRun{at, r.count, (uint8_t)(r.is_rle ? PQR_RLE : PQR_BITPACKED), (uint8_t)pg.dict_bit_width, {}, r.is_rle ? r.value_or_bit_offset : base * 8 + r.value_or_bit_offset}); at += r.count; }
      } else pc.vruns.push_back(PqDevRun{(uint32_t)ord, (uint32_t)pg.non_null, PQR_PLAIN, 0, {}, base + pg.values_offset});
    }
    row += pg.num_values; ord += pg.non_null;
  }
  auto align16 = [&] { static const uint8_t z[16] = {0}; pc.bytes.append(z, (16 - pc.bytes.size() % 16) % 16); };
  align16(); pc.dict_off = pc.bytes.size(); pc.dict_len = pc.dict_bytes.size(); pc.bytes.append(pc.dict_bytes.data(), pc.dict_bytes.size());
  align16(); pc.runs_off = pc.bytes.size();
  pc.bytes.append((const uint8_t*)pc.lruns.data(), pc.lruns.size() * sizeof(PqDevRun));
  pc.bytes.append((const uint8_t*)pc.vruns.data(), pc.vruns.size() * sizeof(PqDevRun));
  if (row != rows) throw ExecError(B200Q_ERR_EXECUTION, "parquet: column " + cs.name + " holds " + std::to_string(row) + " values, its row group " + std::to_string(rows) + " rows");
}

// device half: upload + expand -> one device column of `rows` rows
double g_dbg_copy_ms = 0, g_dbg_kernel_ms = 0;     // B200Q_PARQUET_TIMING=2: serialised split of the device half (copies / kernels)
DevColumn decode_chunk(OpContext& cx, const PreparedChunk& pc, const PqColumnSchema& cs, const DType& want, int64_t rows, DevMemP d_err) {
  static const bool dbg = getenv("B200Q_PARQUET_TIMING") && atoi(getenv("B200Q_PARQUET_TIMING")) >= 2;
  auto hnow = [] { return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now().time_since_epoch()).count(); };
  double td0 = 0; if (dbg) { cudaStreamSynchronize(cx.stream); td0 = hnow(); }
  const bool any_null = pc.any_null;
  PqDecodeSpec sp{};
  DevMemP d_bytes = upload(cx, pc.bytes.data(), pc.bytes.size());
  const PqDevRun* d_lruns = (const PqDevRun*)((const uint8_t*)d_bytes->ptr + pc.runs_off); const PqDevRun* d_vruns = d_lruns + pc.lruns.size();
  sp.bytes = (const uint8_t*)d_bytes->ptr; sp.value_runs = d_vruns; sp.n_value_runs = (int)pc.vruns.size();
  if (pc.has_dict) { sp.dict = (const uint8_t*)d_bytes->ptr + pc.dict_off; sp.dict_count = pc.dict_count; }
  double td1 = 0; if (dbg) { cudaStreamSynchronize(cx.stream); td1 = hnow(); g_dbg_copy_ms += td1 - td0; }
  int out_w = want.byte_width();
  switch (cs.type) {
    case PQ_BOOLEAN: sp.src_width = 0; sp.out_kind = PQO_BOOL_BYTES; out_w = 1; break;
    case PQ_INT32: sp.src_width = 4; sp.out_kind = want.id == T_INT8 ? PQO_I8 : want.id == T_INT16 ? PQO_I16 : want.id == T_DECIMAL128 ? PQO_DEC_FROM_I32 : PQO_I32; break;
    case PQ_INT64: sp.src_width = 8; sp.out_kind = want.id == T_DECIMAL128 ? PQO_DEC_FROM_I64 : PQO_I64; break;
    case PQ_FLOAT: sp.src_width = 4; sp.out_kind = PQO_I32; break;
    case PQ_DOUBLE: sp.src_width = 8; sp.out_kind = PQO_I64; break;
    default: sp.src_width = cs.type_length; sp.out_kind = PQO_DEC_FROM_FLBA; break;
  }
  if (pc.has_dict && sp.src_width > 0 && (int64_t)pc.dict_len < (int64_t)pc.dict_count * sp.src_width) throw ExecError(B200Q_ERR_EXECUTION, "parquet: dictionary page shorter than its entry count");
  DevColumn col; col.type = want;
  DevMemP d_valid, d_ord;
  if (any_null) {
    d_valid = DevMem::alloc((size_t)rows + 16, cx.stream);
    cx.m.launches += launch_pq_levels((const uint8_t*)d_bytes->ptr, d_lruns, (int)pc.lruns.size(), rows, (uint8_t*)d_valid->ptr, cx.stream);
    DevMemP fl = DevMem::alloc((size_t)rows * 4 + 16, cx.stream), sums = DevMem::alloc((size_t)scan_num_blocks(rows) * 4 + 16, cx.stream);
    d_ord = DevMem::alloc((size_t)(rows + 1) * 4, cx.stream);
    cx.m.launches += launch_bytes_to_flags((const uint8_t*)d_valid->ptr, rows, 0, (int32_t*)fl->ptr, cx.stream);
    cx.m.launches += launch_exclusive_scan_i32((const int32_t*)fl->ptr, (int32_t*)d_ord->ptr, rows, (int32_t*)sums->ptr, cx.stream);
    col.validity = pack_bits(cx, d_valid->ptr, rows);
  }
  DevMemP out = DevMem::alloc((size_t)rows * out_w + 16, cx.stream);
  cx.m.launches += launch_pq_decode(sp, any_null ? (const uint8_t*)d_valid->ptr : nullptr, any_null ? (const int32_t*)d_ord->ptr : nullptr, rows, out->ptr, (int*)d_err->ptr, cx.stream);
  if (cs.type == PQ_BOOLEAN) col.values = pack_bits(cx, out->ptr, rows);
  else col.values = out;
  if (dbg) { cudaStreamSynchronize(cx.stream); g_dbg_kernel_ms += hnow() - td1; }
  return col;
}

}  // namespace

void run_parquet_scan(OpContext& cx, const PlanNode& leaf, const std::function<void(DevBatch&)>& emit) {
  static const bool timing = getenv("B200Q_PARQUET_TIMING") != nullptr;       // where a scan's wall time goes (stderr)
  double t_prep = 0, t_dev = 0, t_sync = 0, t_emit = 0;
  auto now = [] { return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now().time_since_epoch()).count(); };
  const double t_begin = now();
  int64_t remaining = leaf.scan_has_limit ? (int64_t)leaf.scan_limit : -1;
  DevMemP d_err = DevMem::alloc(16, cx.stream, true);
  std::vector<std::unique_ptr<PreparedChunk>> prep;   // the ring of prepared chunks of this scan (their buffers return to the pinned pool with them)
  for (auto& sf : leaf.scan_files) {
    if (remaining == 0) break;
    FileIo io(sf.path, sf.size);
    if (io.size < 12) throw ExecError(B200Q_ERR_EXECUTION, "parquet: " + sf.path + " is too small to be a parquet file");
    uint8_t tail[8]; io.read(io.size - 8, 8, tail);
    if (memcmp(tail + 4, "PAR1", 4) != 0) throw ExecError(B200Q_ERR_EXECUTION, "parquet: " + sf.path + " has no PAR1 footer (encrypted files are not supported)");
    uint32_t flen; memcpy(&flen, tail, 4);
    if ((int64_t)flen + 8 > io.size) throw ExecError(B200Q_ERR_EXECUTION, "parquet: footer length exceeds the file");
    std::vector<uint8_t> footer(flen); io.read(io.size - 8 - flen, flen, footer.data());
    const PqFileMeta meta = parquet_parse_footer(footer.data(), footer.size());
    if (!meta.flat) throw ExecError(B200Q_ERR_UNSUPPORTED, "parquet: nested / repeated columns are not on the GPU path");
    // plan column (by name; exact, then case-insensitive) -> file leaf
    std::vector<int> file_col_of(leaf.scan_file_schema.fields.size(), -1);
    for (size_t i = 0; i < file_col_of.size(); i++) {
      const std::string& want = leaf.scan_file_schema.fields[i].name;
      for (size_t j = 0; j < meta.columns.size() && file_col_of[i] < 0; j++) if (meta.columns[j].name == want) file_col_of[i] = (int)j;
      for (size_t j = 0; j < meta.columns.size() && file_col_of[i] < 0; j++)
        if (meta.columns[j].name.size() == want.size()) { bool eq = true; for (size_t k = 0; k < want.size(); k++) eq = eq && tolower((unsigned char)want[k]) == tolower((unsigned char)meta.columns[j].name[k]); if (eq) file_col_of[i] = (int)j; }
    }
    // the row groups of this split that survive pruning
    std::vector<const PqRowGroup*> todo;
    for (auto& rg : meta.row_groups) {
      if (rg.num_rows == 0 || rg.columns.empty()) continue;
      const int64_t rg_start = rg.columns[0].start();                     // a row group belongs to the split that holds its first byte
      if (sf.has_range && (rg_start < sf.range_start || rg_start >= sf.range_end)) continue;
      bool keep = true;
      for (auto& p : leaf.scan_pruning) keep = keep && may_match(p, file_col_of, meta, rg);
      if (!keep) { cx.m.fast_launches++; continue; }                        // pruned row groups show up in fast_path_launches
      if (rg.num_rows > 0x7FFFFFFFLL) throw ExecError(B200Q_ERR_UNSUPPORTED, "parquet: row group above 2^31-1 rows");
      todo.push_back(&rg);
    }
    // host half (file read, Thrift, Snappy, run tables): a pool of worker threads takes the (row group, projected chunk) tasks in order and
    // fills a ring of row-group slots; device half (upload, expand, stages above) on this thread, in row-group order, while the workers
    // are already preparing the row groups behind it
    const size_t ncol = leaf.scan_projection.size();
    const size_t ntasks = todo.size() * ncol;
    const unsigned hw = std::max(1u, std::thread::hardware_concurrency());
    const size_t nthreads = std::max<size_t>(1, std::min<size_t>({(size_t)hw, (size_t)32, ntasks}));
    const size_t ring = std::min(todo.size(), (nthreads + ncol - 1) / std::max<size_t>(1, ncol) + 3);
    while (prep.size() < ring * ncol) prep.push_back(std::make_unique<PreparedChunk>());
    struct Shared {
      std::mutex mu; std::condition_variable cv_done, cv_free;
      std::vector<int> done; size_t consumed = 0, next = 0; bool stop = false;
    } sh;
    sh.done.assign(todo.size(), 0);
    auto worker = [&] {
      while (true) {
        size_t t;
        { std::unique_lock<std::mutex> l(sh.mu); t = sh.next++; if (t >= ntasks) return;
          sh.cv_free.wait(l, [&] { return sh.stop || t / ncol < sh.consumed + ring; });
          if (sh.stop) return; }
        const size_t rgi = t / ncol, k = t % ncol;
        const int pi = leaf.scan_projection[k], fc = file_col_of[(size_t)pi];
        if (fc >= 0) {
          PreparedChunk* pc = prep[(rgi % ring) * ncol + k].get();
          const PqRowGroup* rg = todo[rgi];
          try { prepare_chunk(io, rg->columns[(size_t)fc], meta.columns[(size_t)fc], leaf.scan_file_schema.fields[(size_t)pi].type, rg->num_rows, *pc); }
          catch (const PlanError& e) { pc->error = e.what(); pc->error_code = e.code; }
          catch (const ExecError& e) { pc->error = e.what(); pc->error_code = e.code; }
          catch (const std::exception& e) { pc->error = e.what(); pc->error_code = B200Q_ERR_EXECUTION; }
        }
        { std::lock_guard<std::mutex> l(sh.mu); sh.done[rgi]++; }
        sh.cv_done.notify_all();
      }
    };
    struct Pool {                                   // joins on every exit path (an error in the device half must not leave workers behind)
      Shared& sh; std::vector<std::thread> th;
      ~Pool() { { std::lock_guard<std::mutex> l(sh.mu); sh.stop = true; } sh.cv_free.notify_all(); for (auto& t : th) t.join(); }
    } pool{sh, {}};
    for (size_t i = 0; i < nthreads && ntasks; i++) pool.th.emplace_back(worker);
    struct Events {                                 // one pair per ring slot: the row group's device work is awaited one row group later
      std::vector<cudaEvent_t> a, b;
      explicit Events(size_t n) : a(n), b(n) { for (size_t i = 0; i < n; i++) { B200Q_CUDA(cudaEventCreate(&a[i])); B200Q_CUDA(cudaEventCreate(&b[i])); } }
      ~Events() { for (auto e : a) cudaEventDestroy(e); for (auto e : b) cudaEventDestroy(e); }
    } ev(ring);
    auto retire = [&](size_t rgi) {                 // row group rgi's uploads and kernels are done: its ring slot goes back to the workers
      const double t = now();
      B200Q_CUDA(cudaEventSynchronize(ev.b[rgi % ring]));
      { float ms = 0; B200Q_CUDA(cudaEventElapsedTime(&ms, ev.a[rgi % ring], ev.b[rgi % ring])); cx.m.gpu_ms += ms; }
      { std::lock_guard<std::mutex> l(sh.mu); sh.consumed = rgi + 1; }
      sh.cv_free.notify_all();
      t_sync += now() - t;
    };
    size_t in_flight = 0, next_retire = 0;
    for (size_t rgi = 0; rgi < todo.size() && remaining != 0; rgi++) {
      const PqRowGroup& rg = *todo[rgi];
      const double t0 = now();
      { std::unique_lock<std::mutex> l(sh.mu); sh.cv_done.wait(l, [&] { return sh.done[rgi] == (int)ncol; }); }
      const double t1 = now(); t_prep += t1 - t0;
      DevBatch b; b.num_rows = rg.num_rows;
      B200Q_CUDA(cudaEventRecord(ev.a[rgi % ring], cx.stream));
      for (size_t k = 0; k < ncol; k++) {
        const int pi = leaf.scan_projection[k];
        const FieldDef& f = leaf.scan_file_schema.fields[(size_t)pi];
        const int fc = file_col_of[(size_t)pi];
        if (fc < 0) {                                                     // column missing in this file (schema evolution): all NULL
          DevColumn c; c.type = f.type;
          c.values = DevMem::alloc(f.type.id == T_BOOL ? bitmap_bytes(rg.num_rows) : (size_t)rg.num_rows * f.type.byte_width() + 16, cx.stream, true);
          c.validity = DevMem::alloc(bitmap_bytes(rg.num_rows), cx.stream, true);
          b.cols.push_back(c);
          continue;
        }
        const PreparedChunk& pc = *prep[(rgi % ring) * ncol + k];
        if (pc.error_code) throw ExecError(pc.error_code, pc.error);
        b.cols.push_back(decode_chunk(cx, pc, meta.columns[(size_t)fc], f.type, rg.num_rows, d_err));
      }
      B200Q_CUDA(cudaEventRecord(ev.b[rgi % ring], cx.stream));
      in_flight = rgi + 1;
      t_dev += now() - t1;
      if (remaining >= 0 && b.num_rows > remaining) b.num_rows = remaining;  // ScanLimit: a prefix of the row group (columns keep their buffers)
      if (remaining >= 0) remaining -= b.num_rows;
      cx.m.input_rows += b.num_rows; cx.m.input_batches++;
      const double t4 = now();
      emit(b);
      t_emit += now() - t4;
      while (next_retire + 1 < in_flight) retire(next_retire++);          // the previous row group: its device work overlapped this one's host side
    }
    while (next_retire < in_flight) retire(next_retire++);
    int err = 0;
    B200Q_CUDA(cudaMemcpyAsync(&err, d_err->ptr, 4, cudaMemcpyDeviceToHost, cx.stream));
    B200Q_CUDA(cudaStreamSynchronize(cx.stream));
    if (err) throw ExecError(B200Q_ERR_EXECUTION, "parquet: dictionary index out of range in " + sf.path);
  }
  if (timing) fprintf(stderr, "parquet scan: %.1f ms = waiting for the host workers %.1f ms + upload + launch %.1f ms + wait for the device %.1f ms + stages above %.1f ms + footer / setup\n",
                      now() - t_begin, t_prep, t_dev, t_sync, t_emit);
  if (timing && g_dbg_copy_ms > 0) { fprintf(stderr, "  device half, serialised: uploads %.1f ms, allocations + kernels %.1f ms\n", g_dbg_copy_ms, g_dbg_kernel_ms); g_dbg_copy_ms = g_dbg_kernel_ms = 0; }
}

}  // namespace b200q
