// Device-side repartitioning (the GPU counterpart of the reference's shuffle between the Partial and the Final
// AggExec, SURVEY.md §8e / §2.4 C1+K7):
//
//   pid[i]   = pmod(murmur3_x86_32(key columns, seed 42), P)          — shuffle/mod.rs:163-188, spark_hash.rs:84-200
//   partition: counting partition of every column into P contiguous regions (one pass for pids + histogram, one
//              pass that ranks the rows inside 4096-row tiles in shared memory and reserves the tile's span of each
//              region with ONE global atomic per (tile, partition), one gather pass per column); the row order inside a
//              partition is not a contract (the reference's radix sort is unstable, rdx_sort.rs:55-73)
//   exchange : one ncclAllGather of the P send counts (so that every rank knows all P x P counts after ONE host
//              synchronisation) and one grouped ncclSend/ncclRecv AllToAllv per column straight into the output columns
//              at their final offsets.  No eager-framework glue, no sort, no per-column host round trip.
//
// NCCL is bound at run time (dlopen of libnccl.so.2, the copy the host process already loaded when there is one): a
// single-GPU deployment needs no NCCL at all.  The communicator is created from an ncclUniqueId the host's own control
// plane distributes (rank 0 calls b200q_exchange_unique_id, everyone b200q_exchange_create).
#include <dlfcn.h>
#include <nccl.h>

#include <algorithm>
#include <cstring>
#include <mutex>
#include <vector>

#include "runtime.h"

namespace b200q {

// ---------------------------------------------------------------------------------------------------
// partition kernels (shared with the shuffle-writer path)
// ---------------------------------------------------------------------------------------------------
constexpr int PT_BLOCK = 256, PT_TILE = 4096, PT_MAX_PARTS = 2048;

// counts[p] += rows of partition p   (pids were written by murmur3_partition_kernel)
__global__ void __launch_bounds__(PT_BLOCK) partition_hist_kernel(const uint32_t* __restrict__ pids, long long n, int P, unsigned long long* counts) {
  __shared__ unsigned s_hist[PT_MAX_PARTS];
  for (int p = threadIdx.x; p < P; p += PT_BLOCK) s_hist[p] = 0;
  __syncthreads();
  for (long long i = blockIdx.x * (long long)PT_BLOCK + threadIdx.x; i < n; i += (long long)gridDim.x * PT_BLOCK) atomicAdd(&s_hist[pids[i]], 1u);
  __syncthreads();
  for (int p = threadIdx.x; p < P; p += PT_BLOCK) if (s_hist[p]) atomicAdd(counts + p, (unsigned long long)s_hist[p]);
}

// offsets[p] = exclusive prefix of counts (P <= PT_MAX_PARTS: one block), cursors[p] = offsets[p]
__global__ void __launch_bounds__(PT_BLOCK) partition_offsets_kernel(const unsigned long long* counts, int P, unsigned long long* offsets /* P + 1 */, unsigned long long* cursors) {
  __shared__ unsigned long long s[PT_MAX_PARTS + 1];
  if (threadIdx.x == 0) { unsigned long long acc = 0; for (int p = 0; p < P; p++) { s[p] = acc; acc += counts[p]; } s[P] = acc; }
  __syncthreads();
  for (int p = threadIdx.x; p <= P; p += PT_BLOCK) { offsets[p] = s[p]; if (p < P) cursors[p] = s[p]; }
}

// dest[i] = position of row i in the partitioned order.  Per 4096-row tile: shared-memory histogram, ONE global
// atomic per non-empty partition to reserve the tile's span of its region, shared-memory ranks inside the span.
__global__ void __launch_bounds__(PT_BLOCK) partition_dest_kernel(const uint32_t* __restrict__ pids, long long n, int P, unsigned long long* cursors, uint32_t* __restrict__ dest) {
  __shared__ unsigned s_cnt[PT_MAX_PARTS];                         // rows of the tile per partition (= the running rank while they are counted)
  __shared__ unsigned long long s_base[PT_MAX_PARTS];              // where the tile's span of each partition starts
  const long long ntiles = (n + PT_TILE - 1) / PT_TILE;
  for (long long tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    for (int p = threadIdx.x; p < P; p += PT_BLOCK) s_cnt[p] = 0;
    __syncthreads();
    const long long t0 = tile * PT_TILE;
    unsigned my_pid[PT_TILE / PT_BLOCK], my_rank[PT_TILE / PT_BLOCK];
#pragma unroll
    for (int r = 0; r < PT_TILE / PT_BLOCK; r++) {
      const long long i = t0 + r * PT_BLOCK + threadIdx.x;
      my_pid[r] = i < n ? pids[i] : 0xFFFFFFFFu;
      if (i < n) my_rank[r] = atomicAdd(&s_cnt[my_pid[r]], 1u);
    }
    __syncthreads();
    for (int p = threadIdx.x; p < P; p += PT_BLOCK) if (s_cnt[p]) s_base[p] = atomicAdd(cursors + p, (unsigned long long)s_cnt[p]);
    __syncthreads();
#pragma unroll
    for (int r = 0; r < PT_TILE / PT_BLOCK; r++) {
      const long long i = t0 + r * PT_BLOCK + threadIdx.x;
      if (i < n) dest[i] = (uint32_t)(s_base[my_pid[r]] + my_rank[r]);
    }
    __syncthreads();
  }
}

// out[dest[i]] = in[i] for one fixed-width column (W bytes per value); validity bits -> one byte per row
template <typename T>
__global__ void __launch_bounds__(PT_BLOCK) scatter_col_kernel(const T* __restrict__ in, const uint32_t* __restrict__ dest, long long n, T* __restrict__ out) {
  for (long long i = blockIdx.x * (long long)PT_BLOCK + threadIdx.x; i < n; i += (long long)gridDim.x * PT_BLOCK) out[dest[i]] = in[i];
}
__global__ void __launch_bounds__(PT_BLOCK) scatter_bits_kernel(const uint8_t* __restrict__ bits, unsigned long long bit_offset, const uint32_t* __restrict__ dest, long long n, uint8_t* __restrict__ out_bytes) {
  for (long long i = blockIdx.x * (long long)PT_BLOCK + threadIdx.x; i < n; i += (long long)gridDim.x * PT_BLOCK) {
    const unsigned long long bi = (unsigned long long)i + bit_offset;
    out_bytes[dest[i]] = (bits[bi >> 3] >> (bi & 7)) & 1;
  }
}

static int pt_grid(int64_t n, int per_block) {
  int dev = 0, sms = 132; cudaGetDevice(&dev); cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  const int64_t want = (n + per_block - 1) / per_block, cap = (int64_t)sms * 8;
  return (int)std::max<int64_t>(1, std::min(want, cap));
}

struct u128 { unsigned long long a, b; };

int launch_partition_plan(const uint32_t* d_pids, int64_t n, int P, unsigned long long* d_counts /*P, zeroed*/, unsigned long long* d_offsets /*P+1*/,
                          unsigned long long* d_cursors /*P*/, uint32_t* d_dest /*n*/, cudaStream_t s) {
  if (P > PT_MAX_PARTS) throw ExecError(B200Q_ERR_UNSUPPORTED, "more than 2048 partitions");
  if (n > 0) partition_hist_kernel<<<pt_grid(n, PT_BLOCK * 8), PT_BLOCK, 0, s>>>(d_pids, n, P, d_counts);
  partition_offsets_kernel<<<1, PT_BLOCK, 0, s>>>(d_counts, P, d_offsets, d_cursors);
  if (n > 0) partition_dest_kernel<<<pt_grid(n, PT_TILE), PT_BLOCK, 0, s>>>(d_pids, n, P, d_cursors, d_dest);
  return n > 0 ? 3 : 1;
}
int launch_scatter_column(const void* in, int width, const uint32_t* d_dest, int64_t n, void* out, cudaStream_t s) {
  if (n <= 0) return 0;
  const int g = pt_grid(n, PT_BLOCK * 4);
  switch (width) {
    case 1: scatter_col_kernel<uint8_t><<<g, PT_BLOCK, 0, s>>>((const uint8_t*)in, d_dest, n, (uint8_t*)out); break;
    case 2: scatter_col_kernel<uint16_t><<<g, PT_BLOCK, 0, s>>>((const uint16_t*)in, d_dest, n, (uint16_t*)out); break;
    case 4: scatter_col_kernel<uint32_t><<<g, PT_BLOCK, 0, s>>>((const uint32_t*)in, d_dest, n, (uint32_t*)out); break;
    case 8: scatter_col_kernel<unsigned long long><<<g, PT_BLOCK, 0, s>>>((const unsigned long long*)in, d_dest, n, (unsigned long long*)out); break;
    case 16: scatter_col_kernel<u128><<<g, PT_BLOCK, 0, s>>>((const u128*)in, d_dest, n, (u128*)out); break;
    default: throw ExecError(B200Q_ERR_UNSUPPORTED, "scatter: unsupported column width");
  }
  return 1;
}
int launch_scatter_bits(const uint8_t* bits, uint64_t bit_offset, const uint32_t* d_dest, int64_t n, uint8_t* out_bytes, cudaStream_t s) {
  if (n <= 0) return 0;
  scatter_bits_kernel<<<pt_grid(n, PT_BLOCK * 4), PT_BLOCK, 0, s>>>(bits, bit_offset, d_dest, n, out_bytes);
  return 1;
}

// ---------------------------------------------------------------------------------------------------
// NCCL, bound at run time
// ---------------------------------------------------------------------------------------------------
struct NcclApi {
  void* h = nullptr;
  ncclResult_t (*GetUniqueId)(ncclUniqueId*) = nullptr;
  ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
  ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
  ncclResult_t (*AllGather)(const void*, void*, size_t, ncclDataType_t, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*Send)(const void*, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*Recv)(void*, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*GroupStart)() = nullptr;
  ncclResult_t (*GroupEnd)() = nullptr;
  const char* (*GetErrorString)(ncclResult_t) = nullptr;
};
static NcclApi& nccl() {
  static NcclApi api; static std::once_flag once;
  std::call_once(once, [] {
#ifdef B200Q_EMULATED_DEVICE                                        /* tools/emu: ranks are threads, NCCL is a host stand-in (test infrastructure) */
    api.h = (void*)&api;
#define B200Q_SYM(f) api.f = nccl##f
#else
    const char* names[] = {"libnccl.so.2", "libnccl.so"};
    for (const char* nm : names) { api.h = dlopen(nm, RTLD_NOW | RTLD_GLOBAL); if (api.h) break; }
    if (!api.h) return;
#define B200Q_SYM(f) *(void**)&api.f = dlsym(api.h, "nccl" #f)
#endif
    B200Q_SYM(GetUniqueId); B200Q_SYM(CommInitRank); B200Q_SYM(CommDestroy); B200Q_SYM(AllGather); B200Q_SYM(Send); B200Q_SYM(Recv);
    B200Q_SYM(GroupStart); B200Q_SYM(GroupEnd); B200Q_SYM(GetErrorString);
#undef B200Q_SYM
  });
  if (!api.h || !api.GetUniqueId || !api.CommInitRank || !api.Send || !api.Recv || !api.GroupStart || !api.GroupEnd || !api.AllGather)
    throw ExecError(B200Q_ERR_UNSUPPORTED, "NCCL (libnccl.so.2) is not available in this process: the multi-GPU exchange cannot run");
  return api;
}
#define B200Q_NCCL(expr)                                                                                                             \
  do {                                                                                                                               \
    ncclResult_t _r = (expr);                                                                                                        \
    if (_r != ncclSuccess) throw CudaError(std::string(#expr) + ": " + (nccl().GetErrorString ? nccl().GetErrorString(_r) : "NCCL error")); \
  } while (0)

}  // namespace b200q

using namespace b200q;

struct b200q_exchange {
  int rank = 0, world = 1, device = 0;
  ncclComm_t comm = nullptr;
  std::shared_ptr<StreamRef> stream_ref;
  cudaStream_t stream = nullptr;
  int64_t launches = 0;
};

extern "C" {

b200q_status b200q_exchange_unique_id(uint8_t* out128) {
  if (!out128) return fail(B200Q_ERR_INVALID_ARG, "out is null");
  return guarded_call([&] {
    static_assert(sizeof(ncclUniqueId) == 128, "ncclUniqueId is 128 bytes");
    ncclUniqueId id; B200Q_NCCL(nccl().GetUniqueId(&id)); memcpy(out128, &id, 128);
  });
}

b200q_status b200q_exchange_create(const uint8_t* unique_id128, int32_t rank, int32_t world, int32_t device, b200q_exchange** out) {
  if (!out || !unique_id128) return fail(B200Q_ERR_INVALID_ARG, "null argument");
  *out = nullptr;
  b200q_exchange* ex = nullptr;
  b200q_status st = guarded_call([&] {
    if (world < 1 || rank < 0 || rank >= world) throw ExecError(B200Q_ERR_INVALID_ARG, "invalid rank / world size");
    if (world > PT_MAX_PARTS) throw ExecError(B200Q_ERR_UNSUPPORTED, "world size above 2048");
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) { cudaGetLastError(); throw ExecError(B200Q_ERR_NO_DEVICE, "no CUDA device is visible: the exchange has no CPU fallback"); }
    if (device < 0 || device >= ndev) throw ExecError(B200Q_ERR_INVALID_ARG, "invalid device ordinal");
    B200Q_CUDA(cudaSetDevice(device));
    ex = new b200q_exchange(); ex->rank = rank; ex->world = world; ex->device = device;
    ex->stream_ref = stream_ref_create(device); ex->stream = ex->stream_ref->s;
    ncclUniqueId id; memcpy(&id, unique_id128, 128);
    B200Q_NCCL(nccl().CommInitRank(&ex->comm, world, id, rank));
  });
  if (st != B200Q_OK) { if (ex) { if (ex->comm && nccl().CommDestroy) nccl().CommDestroy(ex->comm); delete ex; } return st; }
  *out = ex;
  return B200Q_OK;
}

void b200q_exchange_destroy(b200q_exchange* ex) {
  if (!ex) return;
  cudaSetDevice(ex->device);
  if (ex->stream) cudaStreamSynchronize(ex->stream);
  try { if (ex->comm) nccl().CommDestroy(ex->comm); } catch (...) {}
  delete ex;
}

int64_t b200q_exchange_kernel_launches(const b200q_exchange* ex) { return ex ? ex->launches : 0; }

// Repartition the rows of `in` (struct of fixed-width columns in HBM; the first n_key_cols children are the grouping
// keys) over the ranks: rank r receives every row whose pid = pmod(murmur3(keys, 42), world) is r.  `out` gets the
// rows this rank owns, from all ranks (source-rank order), as a device array the caller releases.  `in` is released.
b200q_status b200q_exchange_shuffle(b200q_exchange* ex, const struct ArrowSchema* schema, struct ArrowDeviceArray* in, int32_t n_key_cols, struct ArrowDeviceArray* out) {
  if (!ex || !schema || !in || !out) return fail(B200Q_ERR_INVALID_ARG, "null argument");
  b200q_status st = guarded_call([&] {
    const ArrowArray& a = in->array;
    const int ncols = (int)a.n_children, W = ex->world;
    if (in->device_type != ARROW_DEVICE_CUDA || in->device_id != ex->device) throw ExecError(B200Q_ERR_INVALID_ARG, "exchange: batch is not on this exchange's CUDA device");
    if (schema->n_children != a.n_children || ncols < 1 || ncols > VM_MAX_COLS || n_key_cols < 0 || n_key_cols > ncols) throw ExecError(B200Q_ERR_INVALID_ARG, "exchange: schema / array / key count mismatch");
    B200Q_CUDA(cudaSetDevice(ex->device));
    cudaStream_t s = ex->stream;
    if (in->sync_event) B200Q_CUDA(cudaStreamWaitEvent(s, *(cudaEvent_t*)in->sync_event, 0));
    const int64_t n = a.length;
    if (n > 0xFFFFFFFFLL) throw ExecError(B200Q_ERR_UNSUPPORTED, "exchange: more than 2^32 rows in one batch");
    std::vector<DType> types(ncols); std::vector<bool> nullable(ncols);
    ColTable kt{}; uint8_t kphys[VM_MAX_COLS];
    for (int i = 0; i < ncols; i++) {
      types[i] = type_of_format(schema->children[i]->format);
      if (types[i].is_varlen() || types[i].id == T_BOOL || types[i].id == T_NULL) throw ExecError(B200Q_ERR_UNSUPPORTED, "exchange: only fixed-width columns travel GPU-to-GPU (use partial_state_columnar = 1)");
      const ArrowArray* c = a.children[i];
      nullable[i] = c->n_buffers > 0 && c->buffers[0] && c->null_count != 0;
      if (i < n_key_cols) {
        const int64_t off = c->offset + a.offset;
        kt.col[i].values = (const uint8_t*)c->buffers[1] + (size_t)off * types[i].byte_width();
        kt.col[i].validity = nullable[i] ? (const uint8_t*)c->buffers[0] : nullptr;
        kt.col[i].bit_offset = (uint32_t)off; kphys[i] = phys_of(types[i]);
      }
    }
    // ---- partition plan: pids, counts, destinations
    DevMemP pids = DevMem::alloc((size_t)std::max<int64_t>(n, 1) * 4, s), dest = DevMem::alloc((size_t)std::max<int64_t>(n, 1) * 4, s);
    DevMemP meta = DevMem::alloc((size_t)(3 * W + 1 + W * W) * 8, s, true);       // counts[W] | offsets[W+1] | cursors[W] | all_counts[W*W]
    unsigned long long* d_counts = (unsigned long long*)meta->ptr; unsigned long long* d_offsets = d_counts + W; unsigned long long* d_cursors = d_offsets + W + 1; unsigned long long* d_all = d_cursors + W;
    if (n_key_cols == 0) B200Q_CUDA(cudaMemsetAsync(pids->ptr, 0, (size_t)std::max<int64_t>(n, 1) * 4, s));   // no keys: one global group, owned by rank 0 (hash 42 pmod W would also be a constant)
    else ex->launches += launch_murmur3_partition(kt, kphys, n_key_cols, n, W, (uint32_t*)pids->ptr, s);
    ex->launches += launch_partition_plan((const uint32_t*)pids->ptr, n, W, d_counts, d_offsets, d_cursors, (uint32_t*)dest->ptr, s);
    B200Q_CUDA(cudaGetLastError());
    // ---- every rank learns all W x W counts with one collective and ONE host synchronisation
    B200Q_NCCL(nccl().AllGather(d_counts, d_all, (size_t)W, ncclUint64, ex->comm, s));
    std::vector<unsigned long long> all((size_t)W * W);
    B200Q_CUDA(cudaMemcpyAsync(all.data(), d_all, all.size() * 8, cudaMemcpyDeviceToHost, s));
    // ---- meanwhile: scatter every column into its send buffer (partition-major)
    std::vector<DevMemP> send(ncols), send_valid(ncols);
    for (int i = 0; i < ncols; i++) {
      const ArrowArray* c = a.children[i]; const int w = types[i].byte_width(); const int64_t off = c->offset + a.offset;
      send[i] = DevMem::alloc((size_t)std::max<int64_t>(n, 1) * w, s);
      ex->launches += launch_scatter_column((const uint8_t*)c->buffers[1] + (size_t)off * w, w, (const uint32_t*)dest->ptr, n, send[i]->ptr, s);
      if (nullable[i]) {
        send_valid[i] = DevMem::alloc((size_t)std::max<int64_t>(n, 1), s);
        ex->launches += launch_scatter_bits((const uint8_t*)c->buffers[0], (uint64_t)off, (const uint32_t*)dest->ptr, n, (uint8_t*)send_valid[i]->ptr, s);
      }
    }
    B200Q_CUDA(cudaGetLastError());
    B200Q_CUDA(cudaStreamSynchronize(s));
    // all[src * W + dst] = rows src sends to dst
    std::vector<int64_t> soff(W + 1, 0), roff(W + 1, 0);
    for (int p = 0; p < W; p++) { soff[p + 1] = soff[p] + (int64_t)all[(size_t)ex->rank * W + p]; roff[p + 1] = roff[p] + (int64_t)all[(size_t)p * W + ex->rank]; }
    if (soff[W] != n) throw ExecError(B200Q_ERR_EXECUTION, "exchange: partition counts do not add up");
    const int64_t m = roff[W];
    // any column nullable on ANY rank must travel with validity bytes on EVERY rank: nullability is taken from the schema
    std::vector<bool> sch_nullable(ncols);
    for (int i = 0; i < ncols; i++) sch_nullable[i] = (schema->children[i]->flags & ARROW_FLAG_NULLABLE) != 0;
    DevBatch ob; ob.num_rows = m;
    std::vector<DevMemP> recv_valid(ncols);
    for (int i = 0; i < ncols; i++) {
      DevColumn c; c.type = types[i];
      c.values = DevMem::alloc((size_t)std::max<int64_t>(m, 1) * types[i].byte_width(), s);
      if (sch_nullable[i]) {
        recv_valid[i] = DevMem::alloc((size_t)std::max<int64_t>(m, 1), s);
        c.validity = DevMem::alloc((size_t)((m + 31) / 32) * 4 + 4, s, true);
        if (!send_valid[i]) { send_valid[i] = DevMem::alloc((size_t)std::max<int64_t>(n, 1), s); B200Q_CUDA(cudaMemsetAsync(send_valid[i]->ptr, 1, (size_t)std::max<int64_t>(n, 1), s)); }
      } else if (nullable[i]) throw ExecError(B200Q_ERR_INVALID_ARG, "exchange: column " + std::to_string(i) + " carries NULLs but its schema field is not nullable");
      ob.cols.push_back(c);
    }
    // ---- AllToAllv: one group of sends / receives for all columns
    B200Q_NCCL(nccl().GroupStart());
    for (int i = 0; i < ncols; i++) {
      const size_t w = (size_t)types[i].byte_width();
      for (int p = 0; p < W; p++) {
        const int64_t sc = soff[p + 1] - soff[p], rc = roff[p + 1] - roff[p];
        if (p == ex->rank) {                                          // own partition: a device-to-device copy
          if (sc > 0) B200Q_CUDA(cudaMemcpyAsync((uint8_t*)ob.cols[i].values->ptr + (size_t)roff[p] * w, (const uint8_t*)send[i]->ptr + (size_t)soff[p] * w, (size_t)sc * w, cudaMemcpyDeviceToDevice, s));
          if (sc > 0 && sch_nullable[i]) B200Q_CUDA(cudaMemcpyAsync((uint8_t*)recv_valid[i]->ptr + roff[p], (const uint8_t*)send_valid[i]->ptr + soff[p], (size_t)sc, cudaMemcpyDeviceToDevice, s));
          continue;
        }
        if (sc > 0) B200Q_NCCL(nccl().Send((const uint8_t*)send[i]->ptr + (size_t)soff[p] * w, (size_t)sc * w, ncclUint8, p, ex->comm, s));
        if (rc > 0) B200Q_NCCL(nccl().Recv((uint8_t*)ob.cols[i].values->ptr + (size_t)roff[p] * w, (size_t)rc * w, ncclUint8, p, ex->comm, s));
        if (sch_nullable[i]) {
          if (sc > 0) B200Q_NCCL(nccl().Send((const uint8_t*)send_valid[i]->ptr + soff[p], (size_t)sc, ncclUint8, p, ex->comm, s));
          if (rc > 0) B200Q_NCCL(nccl().Recv((uint8_t*)recv_valid[i]->ptr + roff[p], (size_t)rc, ncclUint8, p, ex->comm, s));
        }
      }
    }
    B200Q_NCCL(nccl().GroupEnd());
    for (int i = 0; i < ncols; i++) if (sch_nullable[i] && m > 0) ex->launches += launch_pack_valid((const uint8_t*)recv_valid[i]->ptr, (uint32_t*)ob.cols[i].validity->ptr, m, s);
    B200Q_CUDA(cudaGetLastError());
    B200Q_CUDA(cudaStreamSynchronize(s));                             // the consumer runs on its own stream: hand over completed buffers
    export_device(ob, ex->device, out);
  });
  if (st != B200Q_OK) { cudaSetDevice(ex->device); cudaStreamSynchronize(ex->stream); }   // nothing may still read the caller's buffers
  if (in->array.release) in->array.release(&in->array);
  return st;
}

}  // extern "C"
