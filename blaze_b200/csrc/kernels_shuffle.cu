// ShuffleWriterExec on the GPU (SURVEY.md §8(f) rank 1): hash partition + `batch_serde` encode of one resident batch.
//
// Replaces, for HashPartitioning / single-partition outputs over fixed-width columns:
//   evaluate_hashes + evaluate_partition_ids     datafusion-ext-plans/src/shuffle/mod.rs:163-188
//   sort_batches_by_partition_id                 datafusion-ext-plans/src/shuffle/buffered_data.rs:284-351
//   PartitionedBatchesIterator + write_batch     buffered_data.rs:219-282, datafusion-ext-commons/src/io/batch_serde.rs:66-77,264-306
// The reference sorts (part_id, batch, row) triples on the host, interleaves the rows into a partition-sorted batch
// (a full copy) and then transposes every column of every sub-batch into byte planes (a second copy).  Here one pass
// computes the partition ids and their histogram, a one-CTA pass lays the output out (every record's size follows from
// the counts alone), and ONE pass moves the data: a CTA ranks a 4096-row tile per partition in shared memory, reserves
// the tile's rows of every partition with one global atomic per (tile, partition), stages each column through shared
// memory in partition order and writes the byte planes of the final wire format directly — rows that are neighbours
// in a partition are neighbours in every plane, so a warp's byte stores fall on one or two 32-byte sectors.
// Traffic: keys once more for the ids (+2 B/row of ids), every column read once, every encoded byte written once.
// The row order inside a partition is not a contract (the reference's radix sort is unstable, rdx_sort.rs:55-73).
#include <cuda_runtime.h>
#include <stdint.h>

#include <algorithm>
#include <cstdlib>

#include "hash.cuh"
#include "kernels_shuffle.cuh"
#include "tma.cuh"

namespace b200q {

namespace {

int sm_count() {
  int dev = 0, sms = 132; cudaGetDevice(&dev); cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  return sms;
}

constexpr int PID_BLOCK = 256;

// Spark murmur3 (seed 42) chained over the key columns, NULL leaves the running hash unchanged (hash/mur.rs:19-87,
// spark_hash.rs:84-200), pmod P (shuffle/mod.rs:178-188); histogram in shared memory, one global atomic per (CTA, partition)
__global__ void __launch_bounds__(PID_BLOCK) shuffle_pids_kernel(const ShufSpec sp, long long n, uint16_t* __restrict__ pids, unsigned long long* counts) {
  __shared__ unsigned s_hist[SHUF_MAX_PARTS];
  const int P = sp.num_partitions;
  for (int p = threadIdx.x; p < P; p += PID_BLOCK) s_hist[p] = 0;
  __syncthreads();
  for (long long i = blockIdx.x * (long long)PID_BLOCK + threadIdx.x; i < n; i += (long long)gridDim.x * PID_BLOCK) {
    uint32_t h = 42;
    for (int c = 0; c < sp.nkeys; c++) {
      const ShufCol& col = sp.col[sp.key_col[c]];
      if (col.validity) { const unsigned long long bi = (unsigned long long)i + col.bit_offset; if (!((col.validity[bi >> 3] >> (bi & 7)) & 1)) continue; }
      uint32_t w[4]; int nw;
      switch (sp.key_phys[c]) {
        case PH_BOOL: { const unsigned long long bi = (unsigned long long)i + col.bit_offset; w[0] = (((const uint8_t*)col.values)[bi >> 3] >> (bi & 7)) & 1; nw = 1; break; }
        case PH_I8: w[0] = (uint32_t)(int32_t)((const int8_t*)col.values)[i]; nw = 1; break;
        case PH_I16: w[0] = (uint32_t)(int32_t)((const int16_t*)col.values)[i]; nw = 1; break;
        case PH_I32: case PH_F32: w[0] = ((const uint32_t*)col.values)[i]; nw = 1; break;
        case PH_I64: case PH_F64: { const unsigned long long v = ((const unsigned long long*)col.values)[i]; w[0] = (uint32_t)v; w[1] = (uint32_t)(v >> 32); nw = 2; break; }
        default: { const unsigned long long a = ((const unsigned long long*)col.values)[2 * i], b = ((const unsigned long long*)col.values)[2 * i + 1];
                   w[0] = (uint32_t)a; w[1] = (uint32_t)(a >> 32); w[2] = (uint32_t)b; w[3] = (uint32_t)(b >> 32); nw = 4; break; }
      }
      uint32_t h1 = h;
      for (int k = 0; k < nw; k++) h1 = mm3_mix_h1(h1, mm3_mix_k1(w[k]));
      h = mm3_fmix(h1, (uint32_t)(4 * nw));
    }
    int32_t m = (int32_t)h % P;                                                      // rem_euclid
    if (m < 0) m += P;
    pids[i] = (uint16_t)m;
    atomicAdd(&s_hist[m], 1u);
  }
  __syncthreads();
  for (int p = threadIdx.x; p < P; p += PID_BLOCK) if (s_hist[p]) atomicAdd(counts + p, (unsigned long long)s_hist[p]);
}

// part_off = exclusive prefix of the partitions' encoded sizes; cursors = 0
__global__ void __launch_bounds__(1024) shuffle_layout_kernel(const ShufSpec sp, const unsigned long long* __restrict__ counts, unsigned long long* part_off, unsigned long long* cursors) {
  __shared__ unsigned long long s[SHUF_MAX_PARTS + 1];
  const int P = sp.num_partitions;
  for (int p = threadIdx.x; p < P; p += 1024) { s[p] = shuf_partition_bytes(sp, counts[p]); cursors[p] = 0; }
  __syncthreads();
  if (threadIdx.x == 0) { unsigned long long acc = 0; for (int p = 0; p < P; p++) { const unsigned long long b = s[p]; s[p] = acc; acc += b; } s[P] = acc; }
  __syncthreads();
  for (int p = threadIdx.x; p <= P; p += 1024) part_off[p] = s[p];
}

__device__ __forceinline__ unsigned long long col_offset(const ShufSpec& sp, int c, unsigned long long m, unsigned long long m8, uint32_t vl) {
  return (unsigned long long)vl + (unsigned long long)c + (unsigned long long)sp.col[c].k8 * m8 + (unsigned long long)sp.col[c].kw * m;
}

// record headers: varint(m) and the per-column `has null buffer` byte (io/mod.rs:60-69, batch_serde.rs:274-284); one CTA per partition
__global__ void __launch_bounds__(128) shuffle_headers_kernel(const ShufSpec sp, const unsigned long long* __restrict__ counts, const unsigned long long* __restrict__ part_off, uint8_t* out) {
  const int p = blockIdx.x;
  const unsigned long long t = counts[p], B = (unsigned long long)sp.batch_size;
  if (t == 0) return;
  const unsigned long long nrec = (t + B - 1) / B, F = shuf_record_bytes(sp, B);
  for (unsigned long long rec = threadIdx.x; rec < nrec; rec += 128) {
    const unsigned long long m = rec == nrec - 1 ? t - rec * B : B, m8 = (m + 7) >> 3;
    uint8_t* base = out + part_off[p] + rec * F;
    unsigned long long v = m; uint32_t vl = 0;
    while (v >= 128) { base[vl++] = (uint8_t)(128 + (v & 127)); v >>= 7; }
    base[vl++] = (uint8_t)v;
    for (int c = 0; c < sp.ncols; c++) base[col_offset(sp, c, m, m8, vl)] = sp.col[c].nullable ? 1 : 0;
  }
}

__device__ __forceinline__ void or_bit(uint8_t* out, unsigned long long byte_off, unsigned bit) {
  const unsigned long long a = (unsigned long long)(uintptr_t)out + byte_off;
  atomicOr((unsigned*)(uintptr_t)(a & ~3ull), 1u << (((unsigned)(a & 3ull) << 3) + bit));
}

constexpr int ENC_NT = 512, ENC_RPT = SHUF_TILE / ENC_NT, SHUF_SMEM_PARTS = 512;

// ---- TMA (cp.async.bulk) staging of the input columns -------------------------------------------------------------------
// One elected thread copies a whole tile of a column (4096 values, contiguous in HBM) into shared memory with ONE bulk copy
// that completes on an mbarrier; two buffers, so the copy of the next column (or of the next tile's first column) is in
// flight while the current one is permuted and written out, and the first copy of a tile overlaps its ranking phase.

// where sorted position `i` of the tile lands: byte offset of its record + its row inside the record; rows of that record
__device__ __forceinline__ unsigned long long dest_of(const ShufSpec& sp, unsigned long long F, unsigned B, unsigned p, unsigned idx, const unsigned long long* counts,
                                                       const unsigned long long* part_off, unsigned& m, unsigned& j) {
  const unsigned t = (unsigned)counts[p], rec = idx / B, nrec = (t + B - 1) / B;
  j = idx - rec * B;
  m = rec == nrec - 1 ? t - rec * B : B;
  return part_off[p] + (unsigned long long)rec * F;
}

template <bool TMA>
__global__ void __launch_bounds__(ENC_NT, 2) shuffle_encode_kernel(const ShufSpec sp, const uint16_t* __restrict__ pids, long long n, const unsigned long long* __restrict__ counts_g,
                                                                   const unsigned long long* __restrict__ part_off_g, unsigned long long* cursors, uint8_t* out) {
#ifdef B200Q_EMULATED_DEVICE                                                 // tools/emu: blocks run one at a time, shared memory is a static array
  static unsigned long long smem_words[(SHUF_TILE * 26 + SHUF_MAX_PARTS * 16) / 8];
  unsigned char* smem = (unsigned char*)smem_words;
#else
  extern __shared__ __align__(16) unsigned char smem[];
#endif
  const int P = sp.num_partitions;
  unsigned long long* s_in = (unsigned long long*)smem;                     // TMA: two input buffers of SHUF_TILE values (input order)
  unsigned long long* s_val = s_in + (TMA ? 2 * SHUF_TILE : 0);             // SHUF_TILE values in partition order
  unsigned long long* s_gbase = s_val + SHUF_TILE;                          // P: index inside the partition of the tile's first row of it
  unsigned* s_cnt = (unsigned*)(s_gbase + P);                               // P: rows of the tile per partition
  unsigned* s_start = s_cnt + P;                                            // P: exclusive prefix of s_cnt
  uint16_t* s_p = (uint16_t*)(s_start + P);                                 // SHUF_TILE: partition of every sorted position
  __shared__ unsigned s_warp[ENC_NT / 32];
  const unsigned B = (unsigned)sp.batch_size, B8 = (B + 7) >> 3;
  const unsigned long long F = shuf_record_bytes(sp, B);
  const uint32_t vlB = shuf_varint_len(B);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const long long ntiles = (n + SHUF_TILE - 1) / SHUF_TILE;
  // rows / byte offset of every partition are looked up once per row and tile: keep them in shared memory when they fit
  __shared__ unsigned long long s_tab[2 * SHUF_SMEM_PARTS];
  if (P <= SHUF_SMEM_PARTS) {
    for (int p = tid; p < P; p += ENC_NT) { s_tab[p] = counts_g[p]; s_tab[SHUF_SMEM_PARTS + p] = part_off_g[p]; }
    __syncthreads();
  }
  const unsigned long long* counts = P <= SHUF_SMEM_PARTS ? s_tab : counts_g;
  const unsigned long long* part_off = P <= SHUF_SMEM_PARTS ? s_tab + SHUF_SMEM_PARTS : part_off_g;
  // TMA load sequence of this CTA: load j = column s_ec[j % ne] of the CTA's (j / ne)-th tile, into buffer j & 1
  __shared__ unsigned long long s_bar[2];                               // 8-byte aligned by type
  __shared__ unsigned char s_ec[SHUF_MAX_COLS];
  __shared__ int s_ne;
  unsigned consumed = 0;
  auto issue = [&](unsigned j) {
    if (!TMA || s_ne == 0) return;
    const long long tl = blockIdx.x + (long long)(j / (unsigned)s_ne) * gridDim.x;
    if (tl >= ntiles || (tl + 1) * SHUF_TILE > n) return;                   // only full tiles are staged by bulk copies
    const int c = s_ec[j % (unsigned)s_ne];
    const unsigned w = sp.col[c].width, bytes = SHUF_TILE * w;
    mbar_expect_tx(&s_bar[j & 1], bytes);
    bulk_g2s(s_in + (size_t)(j & 1) * SHUF_TILE, (const uint8_t*)sp.col[c].values + (size_t)tl * SHUF_TILE * w, bytes, &s_bar[j & 1]);
  };
  if (TMA) {
    if (tid == 0) {
      int ne = 0;
      for (int c = 0; c < sp.ncols; c++) if (sp.col[c].tma) s_ec[ne++] = (unsigned char)c;
      s_ne = ne;
      mbar_init(&s_bar[0], 1); mbar_init(&s_bar[1], 1); mbar_fence_init();
    }
    __syncthreads();
    if (tid == 0) { issue(0); issue(1); }
  }
  for (long long tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const long long t0 = tile * SHUF_TILE;
    const int rows = (int)min((long long)SHUF_TILE, n - t0);
    for (int p = tid; p < P; p += ENC_NT) s_cnt[p] = 0;
    __syncthreads();
    unsigned lpos[ENC_RPT];                                                 // rank inside (tile, partition), then position in the tile's partition order
    {
      unsigned pid[ENC_RPT];
#pragma unroll
      for (int k = 0; k < ENC_RPT; k++) {
        const int i = k * ENC_NT + tid;
        pid[k] = 0; lpos[k] = 0;
        if (i < rows) { pid[k] = pids ? pids[t0 + i] : 0; lpos[k] = atomicAdd(&s_cnt[pid[k]], 1u); }
      }
      __syncthreads();
      {   // exclusive scan of s_cnt, one contiguous span of partitions per thread; reserve the tile's rows of every partition
        const int per = (P + ENC_NT - 1) / ENC_NT, lo = min(P, tid * per), hi = min(P, lo + per);
        unsigned sum = 0;
        for (int p = lo; p < hi; p++) sum += s_cnt[p];
        unsigned inc = sum;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) { const unsigned o = __shfl_up_sync(0xFFFFFFFFu, inc, d); if (lane >= d) inc += o; }
        if (lane == 31) s_warp[warp] = inc;
        __syncthreads();
        unsigned wbase = 0;
        for (int w = 0; w < warp; w++) wbase += s_warp[w];
        unsigned run = wbase + inc - sum;
        for (int p = lo; p < hi; p++) {
          const unsigned c = s_cnt[p];
          s_start[p] = run; run += c;
          if (c) s_gbase[p] = atomicAdd(cursors + p, (unsigned long long)c);
        }
      }
      __syncthreads();
#pragma unroll
      for (int k = 0; k < ENC_RPT; k++) {
        const int i = k * ENC_NT + tid;
        if (i < rows) { lpos[k] += s_start[pid[k]]; s_p[lpos[k]] = (uint16_t)pid[k]; }
      }
    }
    __syncthreads();
    // destination of the sorted positions this thread writes out: record base + row inside the record; bit k of `full`: the
    // record holds batch_size rows (every record but a partition's last one) -> its plane stride and column offsets are constants
    unsigned long long wb[ENC_RPT]; unsigned full = 0;
#pragma unroll
    for (int k = 0; k < ENC_RPT; k++) {
      const int i = k * ENC_NT + tid;
      wb[k] = 0;
      if (i < rows) {
        const unsigned p = s_p[i];
        unsigned m, j;
        wb[k] = dest_of(sp, F, B, p, (unsigned)s_gbase[p] + ((unsigned)i - s_start[p]), counts, part_off, m, j) + j;
        if (m == B) full |= 1u << k;
      }
    }
    for (int c = 0; c < sp.ncols; c++) {
      const unsigned width = sp.col[c].width, nullable = sp.col[c].nullable;
      const void* __restrict__ values = sp.col[c].values;
      const int nh = width == 16 ? 2 : (width ? 1 : 0);
      const int nb = width < 8 ? (int)width : 8;
      // data region of column c inside a full record
      const unsigned long long off_full = (unsigned long long)vlB + (unsigned)c + (unsigned long long)sp.col[c].k8 * B8 + (unsigned long long)sp.col[c].kw * B + 1 + (nullable ? B8 : 0);
      for (int h = 0; h < nh; h++) {
        const bool staged = TMA && sp.col[c].tma && rows == SHUF_TILE;
        if (staged) {                                                       // the column's tile is (being) copied into s_in[consumed & 1]
          mbar_wait(&s_bar[consumed & 1], (consumed >> 1) & 1);
          const unsigned long long* in = s_in + (size_t)(consumed & 1) * SHUF_TILE;
          if (width == 8) {
#pragma unroll
            for (int k = 0; k < ENC_RPT; k++) s_val[lpos[k]] = in[k * ENC_NT + tid];
          } else if (width == 4) {
#pragma unroll
            for (int k = 0; k < ENC_RPT; k++) s_val[lpos[k]] = ((const uint32_t*)in)[k * ENC_NT + tid];
          } else if (width == 2) {
#pragma unroll
            for (int k = 0; k < ENC_RPT; k++) s_val[lpos[k]] = ((const uint16_t*)in)[k * ENC_NT + tid];
          } else {
#pragma unroll
            for (int k = 0; k < ENC_RPT; k++) s_val[lpos[k]] = ((const uint8_t*)in)[k * ENC_NT + tid];
          }
        } else if (width == 8) {
#pragma unroll
          for (int k = 0; k < ENC_RPT; k++) { const int i = k * ENC_NT + tid; if (i < rows) s_val[lpos[k]] = ((const unsigned long long*)values)[t0 + i]; }
        } else if (width == 4) {
#pragma unroll
          for (int k = 0; k < ENC_RPT; k++) { const int i = k * ENC_NT + tid; if (i < rows) s_val[lpos[k]] = ((const uint32_t*)values)[t0 + i]; }
        } else if (width == 16) {
#pragma unroll
          for (int k = 0; k < ENC_RPT; k++) { const int i = k * ENC_NT + tid; if (i < rows) s_val[lpos[k]] = ((const unsigned long long*)values)[2 * (t0 + i) + h]; }
        } else if (width == 2) {
#pragma unroll
          for (int k = 0; k < ENC_RPT; k++) { const int i = k * ENC_NT + tid; if (i < rows) s_val[lpos[k]] = ((const uint16_t*)values)[t0 + i]; }
        } else {
#pragma unroll
          for (int k = 0; k < ENC_RPT; k++) { const int i = k * ENC_NT + tid; if (i < rows) s_val[lpos[k]] = ((const uint8_t*)values)[t0 + i]; }
        }
        __syncthreads();
        if (staged) { if (tid == 0) issue(consumed + 2); consumed++; }     // the buffer just read is free: start the copy two loads ahead
#pragma unroll
        for (int k = 0; k < ENC_RPT; k++) {
          const int i = k * ENC_NT + tid;
          if (i < rows) {
            const unsigned long long v = s_val[i];
            if (full & (1u << k)) {
              uint8_t* a = out + wb[k] + off_full + (unsigned long long)(h * 8) * B;
              if (nb == 8) {
#pragma unroll
                for (int b = 0; b < 8; b++) { *a = (uint8_t)(v >> (8 * b)); a += B; }
              } else if (nb == 4) {
#pragma unroll
                for (int b = 0; b < 4; b++) { *a = (uint8_t)(v >> (8 * b)); a += B; }
              } else {
                for (int b = 0; b < nb; b++) { *a = (uint8_t)(v >> (8 * b)); a += B; }
              }
            } else {                                                        // the short last record of a partition
              const unsigned p = s_p[i];
              unsigned m, j;
              dest_of(sp, F, B, p, (unsigned)s_gbase[p] + ((unsigned)i - s_start[p]), counts, part_off, m, j);
              const unsigned long long m8 = (m + 7) >> 3;
              uint8_t* a = out + wb[k] + col_offset(sp, c, m, m8, shuf_varint_len(m)) + 1 + (nullable ? m8 : 0) + (unsigned long long)(h * 8) * m;
              for (int b = 0; b < nb; b++) a[(size_t)b * m] = (uint8_t)(v >> (8 * b));
            }
          }
        }
        __syncthreads();
      }
      if (nullable || width == 0) {
        // bit regions (validity bitmaps, Boolean values): set bits are OR-ed into the zeroed buffer from the rows' own destinations
        const uint8_t* __restrict__ validity = sp.col[c].validity;
        const unsigned bit_offset = sp.col[c].bit_offset;
#pragma unroll
        for (int k = 0; k < ENC_RPT; k++) {
          const int i = k * ENC_NT + tid;
          if (i < rows) {
            const long long r = t0 + i;
            const unsigned p = s_p[lpos[k]];
            unsigned m, j;
            const unsigned long long rb = dest_of(sp, F, B, p, (unsigned)s_gbase[p] + (lpos[k] - s_start[p]), counts, part_off, m, j);
            const unsigned long long m8 = (m + 7) >> 3;
            const unsigned long long cb = rb + col_offset(sp, c, m, m8, shuf_varint_len(m)) + 1;
            const unsigned long long bi = (unsigned long long)r + bit_offset;
            if (nullable) {
              const bool valid = validity ? ((validity[bi >> 3] >> (bi & 7)) & 1) : true;
              if (valid) or_bit(out, cb + (j >> 3), j & 7);
            }
            if (width == 0 && ((((const uint8_t*)values)[bi >> 3] >> (bi & 7)) & 1)) or_bit(out, cb + (nullable ? m8 : 0) + (j >> 3), j & 7);
          }
        }
      }
    }
    __syncthreads();
  }
}

// ---- batches with Binary columns ----------------------------------------------------------------------------------------------
// Two-pass: the data bytes of the chunk are summed first (the host sizes the buffer and the rows per record from them), then the
// rows get their sorted positions ONCE (perm), and every later pass — lengths, their 64-bit scans, record sizes, headers, planes,
// bytes — reads the same positions, so the order of the length planes and of the data always agree.

__device__ __forceinline__ bool vl_valid(const ShufCol& col, unsigned long long row) {
  if (!col.validity) return true;
  const unsigned long long bi = row + col.bit_offset;
  return (col.validity[bi >> 3] >> (bi & 7)) & 1;
}

__device__ __forceinline__ unsigned long long vl_bytes(const ShufVarlen& vl, int k, unsigned long long q0, unsigned long long m) {
  const unsigned long long* d = vl.doff + (unsigned long long)k * (unsigned long long)(vl.n + 1);
  return d[q0 + m] - d[q0];
}

// largest p with a[p] <= x (a ascending, a[0] <= x < a[P])
__device__ __forceinline__ int vl_find(const unsigned long long* a, int P, unsigned long long x) {
  int lo = 0, hi = P;
  while (hi - lo > 1) { const int mid = (lo + hi) >> 1; if (a[mid] <= x) lo = mid; else hi = mid; }
  return lo;
}

// the record holding sorted position q: its index g, first position q0, rows m, and q's row j inside it
struct VlLoc { unsigned long long g, q0, m, j; };
__device__ __forceinline__ VlLoc vl_locate(const ShufVarlen& vl, const unsigned long long* s_rows, int P, const unsigned long long* counts, unsigned long long q) {
  const int p = vl_find(s_rows, P, q);
  const unsigned long long idx = q - s_rows[p], r = idx / vl.B, t = counts[p];
  VlLoc l;
  l.j = idx - r * vl.B; l.q0 = s_rows[p] + r * vl.B; l.g = vl.rec_start[p] + r;
  l.m = t - r * vl.B < vl.B ? t - r * vl.B : vl.B;
  return l;
}

__global__ void __launch_bounds__(256) shuffle_vl_bytes_kernel(const ShufSpec sp, const ShufVarlen vl, unsigned long long* totals) {
  const unsigned lane = threadIdx.x & 31;
  for (int k = 0; k < vl.nb; k++) {
    const ShufCol& col = sp.col[vl.col[k]];
    const int32_t* __restrict__ off = vl.offsets[k];
    unsigned long long sum = 0;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < vl.n; i += (long long)gridDim.x * blockDim.x)
      if (vl_valid(col, (unsigned long long)i)) sum += (unsigned long long)(off[i + 1] - off[i]);
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, d);
    if (lane == 0 && sum) atomicAdd(totals + k, sum);
  }
}

// sorted positions: a CTA ranks a 4096-row tile per partition in shared memory and reserves the tile's rows of every partition with
// one global atomic per (tile, partition), as shuffle_encode_kernel does; perm[row_start[p] + reserved + rank] = row
constexpr int VR_NT = 512, VR_RPT = SHUF_TILE / VR_NT;
__global__ void __launch_bounds__(VR_NT) shuffle_vl_rank_kernel(const ShufVarlen vl, int P, const uint16_t* __restrict__ pids, unsigned long long* cursors) {
  __shared__ unsigned s_cnt[SHUF_MAX_PARTS], s_base[SHUF_MAX_PARTS];
  const long long ntiles = (vl.n + SHUF_TILE - 1) / SHUF_TILE;
  for (long long tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const long long t0 = tile * SHUF_TILE;
    for (int p = threadIdx.x; p < P; p += VR_NT) s_cnt[p] = 0;
    __syncthreads();
    unsigned pid[VR_RPT], rank[VR_RPT];
#pragma unroll
    for (int k = 0; k < VR_RPT; k++) {
      const long long i = t0 + k * VR_NT + threadIdx.x;
      pid[k] = 0; rank[k] = 0;
      if (i < vl.n) { pid[k] = pids[i]; rank[k] = atomicAdd(&s_cnt[pid[k]], 1u); }
    }
    __syncthreads();
    for (int p = threadIdx.x; p < P; p += VR_NT) {
      const unsigned c = s_cnt[p];
      if (c) s_base[p] = (unsigned)(vl.row_start[p] + atomicAdd(cursors + p, (unsigned long long)c));
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < VR_RPT; k++) {
      const long long i = t0 + k * VR_NT + threadIdx.x;
      if (i < vl.n) vl.perm[s_base[pid[k]] + rank[k]] = (uint32_t)i;
    }
    __syncthreads();
  }
}

// lens[k * n + q] = data bytes of sorted position q in Binary column k (0 for NULL)
__global__ void __launch_bounds__(256) shuffle_vl_lengths_kernel(const ShufSpec sp, const ShufVarlen vl) {
  for (long long q = blockIdx.x * (long long)blockDim.x + threadIdx.x; q < vl.n; q += (long long)gridDim.x * blockDim.x) {
    const unsigned long long row = vl.perm ? vl.perm[q] : (unsigned long long)q;
    for (int k = 0; k < vl.nb; k++) {
      const int32_t* __restrict__ off = vl.offsets[k];
      vl.lens[(unsigned long long)k * vl.n + q] = vl_valid(sp.col[vl.col[k]], row) ? (uint32_t)(off[row + 1] - off[row]) : 0u;
    }
  }
}

// 64-bit exclusive scan (n -> n + 1 entries): block sums, one CTA scans the sums, final pass
constexpr int VS_BLOCK = 256, VS_ITEMS = 8, VS_TILE = VS_BLOCK * VS_ITEMS;

__device__ __forceinline__ unsigned long long vs_block_exclusive(unsigned long long v, unsigned long long* total, unsigned long long* smem /* 9 */) {
  const unsigned lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  unsigned long long incl = v;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) { const unsigned long long t = __shfl_up_sync(0xffffffffu, incl, d); if (lane >= d) incl += t; }
  if (lane == 31) smem[warp] = incl;
  __syncthreads();
  if (warp == 0) {
    const unsigned long long w = lane < VS_BLOCK / 32 ? smem[lane] : 0;
    unsigned long long wi = w;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) { const unsigned long long t = __shfl_up_sync(0xffffffffu, wi, d); if (lane >= d) wi += t; }
    if (lane < VS_BLOCK / 32) smem[lane] = wi - w;
    if (lane == VS_BLOCK / 32 - 1) smem[8] = wi;
  }
  __syncthreads();
  const unsigned long long res = incl - v + smem[warp];
  *total = smem[8];
  __syncthreads();
  return res;
}

template <class T>
__global__ void __launch_bounds__(VS_BLOCK) vl_scan_sums_kernel(const T* __restrict__ in, long long n, unsigned long long* __restrict__ sums) {
  __shared__ unsigned long long smem[9];
  const long long base = blockIdx.x * (long long)VS_TILE;
  unsigned long long s = 0;
  for (int k = 0; k < VS_ITEMS; k++) { const long long i = base + k * VS_BLOCK + threadIdx.x; if (i < n) s += in[i]; }
  unsigned long long total; vs_block_exclusive(s, &total, smem);
  if (threadIdx.x == 0) sums[blockIdx.x] = total;
}
__global__ void __launch_bounds__(VS_BLOCK) vl_scan_carry_kernel(unsigned long long* sums, long long nb) {
  __shared__ unsigned long long smem[9];
  unsigned long long carry = 0;
  for (long long base = 0; base < nb; base += VS_BLOCK) {
    const long long i = base + threadIdx.x;
    const unsigned long long v = i < nb ? sums[i] : 0;
    unsigned long long total; const unsigned long long ex = vs_block_exclusive(v, &total, smem);
    if (i < nb) sums[i] = carry + ex;
    carry += total;
  }
}
template <class T>
__global__ void __launch_bounds__(VS_BLOCK) vl_scan_final_kernel(const T* __restrict__ in, unsigned long long* __restrict__ out, long long n, const unsigned long long* __restrict__ sums) {
  __shared__ unsigned long long smem[9];
  const long long base = blockIdx.x * (long long)VS_TILE + (long long)threadIdx.x * VS_ITEMS;
  unsigned long long v[VS_ITEMS], s = 0;
#pragma unroll
  for (int k = 0; k < VS_ITEMS; k++) { v[k] = base + k < n ? (unsigned long long)in[base + k] : 0; s += v[k]; }
  unsigned long long total; unsigned long long ex = vs_block_exclusive(s, &total, smem) + sums[blockIdx.x];
#pragma unroll
  for (int k = 0; k < VS_ITEMS; k++) { if (base + k < n) out[base + k] = ex; ex += v[k]; }
  if (base <= n - 1 && n - 1 < base + VS_ITEMS) out[n] = ex;                   // the grand total, from the owner of index n - 1
}

template <class T>
int vl_scan(const T* in, unsigned long long* out, int64_t n, unsigned long long* sums, cudaStream_t s) {
  const int64_t nb = (n + VS_TILE - 1) / VS_TILE;
  vl_scan_sums_kernel<T><<<(unsigned)nb, VS_BLOCK, 0, s>>>(in, n, sums);
  vl_scan_carry_kernel<<<1, VS_BLOCK, 0, s>>>(sums, nb);
  vl_scan_final_kernel<T><<<(unsigned)nb, VS_BLOCK, 0, s>>>(in, out, n, sums);
  return 3;
}

// encoded bytes of every record; err bit 0 when the Binary data of one record would exceed INT32_MAX bytes (the reader's 32-bit offsets)
__global__ void __launch_bounds__(256) shuffle_vl_records_kernel(const ShufSpec sp, const ShufVarlen vl, int P, const unsigned long long* __restrict__ counts) {
  for (long long g = blockIdx.x * (long long)blockDim.x + threadIdx.x; g < vl.R; g += (long long)gridDim.x * blockDim.x) {
    const int p = vl_find(vl.rec_start, P, (unsigned long long)g);
    const unsigned long long r = (unsigned long long)g - vl.rec_start[p], t = counts[p];
    const unsigned long long m = t - r * vl.B < vl.B ? t - r * vl.B : vl.B, q0 = vl.row_start[p] + r * vl.B;
    unsigned long long data = 0;
    for (int k = 0; k < vl.nb; k++) data += vl_bytes(vl, k, q0, m);
    vl.rec_size[g] = shuf_record_bytes(sp, m) + data;
    if (data > 0x7FFFFFFFull) atomicOr(vl.err, 1u);
  }
}

// varint(m) + the `has null buffer` byte of every column of every record; part_off[p] = rec_off[rec_start[p]]
__global__ void __launch_bounds__(256) shuffle_vl_headers_kernel(const ShufSpec sp, const ShufVarlen vl, int P, const unsigned long long* __restrict__ counts,
                                                                 unsigned long long* part_off, uint8_t* out) {
  for (long long g = blockIdx.x * (long long)blockDim.x + threadIdx.x; g < vl.R || g <= P; g += (long long)gridDim.x * blockDim.x) {
    if (g <= P) part_off[g] = vl.rec_off[vl.rec_start[g]];
    if (g >= vl.R) continue;
    const int p = vl_find(vl.rec_start, P, (unsigned long long)g);
    const unsigned long long r = (unsigned long long)g - vl.rec_start[p], t = counts[p];
    const unsigned long long m = t - r * vl.B < vl.B ? t - r * vl.B : vl.B, m8 = (m + 7) >> 3, q0 = vl.row_start[p] + r * vl.B;
    uint8_t* base = out + vl.rec_off[g];
    unsigned long long v = m; uint32_t vlen = 0;
    while (v >= 128) { base[vlen++] = (uint8_t)(128 + (v & 127)); v >>= 7; }
    base[vlen++] = (uint8_t)v;
    unsigned long long before = 0; int k = 0;
    for (int c = 0; c < sp.ncols; c++) {
      base[col_offset(sp, c, m, m8, vlen) + before] = sp.col[c].nullable ? 1 : 0;
      if (sp.col[c].varlen) before += vl_bytes(vl, k++, q0, m);
    }
  }
}

// one thread per sorted position: validity and Boolean bits, the byte planes of the fixed-width columns and the length planes.
// Neighbouring positions are neighbouring bytes of every plane; the input rows are gathered through perm.
constexpr int VE_NT = 256;
__global__ void __launch_bounds__(VE_NT) shuffle_vl_encode_kernel(const ShufSpec sp, const ShufVarlen vl, int P, const unsigned long long* __restrict__ counts, uint8_t* out) {
  __shared__ unsigned long long s_rows[SHUF_MAX_PARTS + 1];
  for (int p = threadIdx.x; p <= P; p += VE_NT) s_rows[p] = vl.row_start[p];
  __syncthreads();
  for (long long q = blockIdx.x * (long long)VE_NT + threadIdx.x; q < vl.n; q += (long long)gridDim.x * VE_NT) {
    const VlLoc l = vl_locate(vl, s_rows, P, counts, (unsigned long long)q);
    const unsigned long long row = vl.perm ? vl.perm[q] : (unsigned long long)q, m8 = (l.m + 7) >> 3;
    const uint32_t vlen = shuf_varint_len(l.m);
    const unsigned long long rb = vl.rec_off[l.g];
    unsigned long long before = 0; int k = 0;
    for (int c = 0; c < sp.ncols; c++) {
      const ShufCol& col = sp.col[c];
      unsigned long long a = rb + col_offset(sp, c, l.m, m8, vlen) + before + 1;          // past the `has null buffer` byte
      const bool valid = vl_valid(col, row);
      if (col.nullable) { if (valid) or_bit(out, a + (l.j >> 3), (unsigned)(l.j & 7)); a += m8; }
      if (col.width == 0) {
        const unsigned long long bi = row + col.bit_offset;
        if ((((const uint8_t*)col.values)[bi >> 3] >> (bi & 7)) & 1) or_bit(out, a + (l.j >> 3), (unsigned)(l.j & 7));
        continue;
      }
      uint8_t* d = out + a + l.j;
      if (col.varlen) {
        const int32_t* __restrict__ off = vl.offsets[k];
        const uint32_t len = valid ? (uint32_t)(off[row + 1] - off[row]) : 0u;
#pragma unroll
        for (int b = 0; b < 4; b++) d[(unsigned long long)b * l.m] = (uint8_t)(len >> (8 * b));
        before += vl_bytes(vl, k++, l.q0, l.m);
        continue;
      }
      unsigned long long lo = 0, hi = 0;
      switch (col.width) {
        case 1: lo = ((const uint8_t*)col.values)[row]; break;
        case 2: lo = ((const uint16_t*)col.values)[row]; break;
        case 4: lo = ((const uint32_t*)col.values)[row]; break;
        case 8: lo = ((const unsigned long long*)col.values)[row]; break;
        default: lo = ((const unsigned long long*)col.values)[2 * row]; hi = ((const unsigned long long*)col.values)[2 * row + 1]; break;
      }
      for (int b = 0; b < (int)col.width; b++) d[(unsigned long long)b * l.m] = (uint8_t)((b < 8 ? lo : hi) >> (8 * (b & 7)));
    }
  }
}

struct alignas(16) VlV16 { unsigned long long lo, hi; };

// 16 output bytes from a source `mis` (1..15) bytes past a 16-byte boundary: two aligned loads, each output word a funnel shift
__device__ __forceinline__ VlV16 vl_shifted16(const VlV16* __restrict__ src, int v, unsigned mis) {
  const VlV16 a = src[v], b = src[v + 1];
  const uint32_t w[8] = {(uint32_t)a.lo, (uint32_t)(a.lo >> 32), (uint32_t)a.hi, (uint32_t)(a.hi >> 32),
                         (uint32_t)b.lo, (uint32_t)(b.lo >> 32), (uint32_t)b.hi, (uint32_t)(b.hi >> 32)};
  const unsigned q = mis >> 2, sh = (mis & 3) * 8;
  uint32_t x[5];
#pragma unroll
  for (int i = 0; i < 5; i++) x[i] = q == 0 ? w[i] : q == 1 ? w[i + 1] : q == 2 ? w[i + 2] : w[i + 3];
  uint32_t o[4];
#pragma unroll
  for (int i = 0; i < 4; i++) o[i] = (uint32_t)(((((uint64_t)x[i + 1]) << 32) | x[i]) >> sh);
  VlV16 r; r.lo = o[0] | ((unsigned long long)o[1] << 32); r.hi = o[2] | ((unsigned long long)o[3] << 32);
  return r;
}

// the Binary bytes: one warp per 32 consecutive sorted positions, which it copies one after the other with all 32 lanes, so a long
// value spreads over the warp.  Values of 64 bytes or more go as aligned 16-byte vectors (loads funnel-shifted into place when source
// and destination disagree modulo 16), as varlen_copy_kernel does; heads and tails are byte copies.
__global__ void __launch_bounds__(VE_NT) shuffle_vl_copy_kernel(const ShufSpec sp, const ShufVarlen vl, int P, const unsigned long long* __restrict__ counts, uint8_t* out) {
  __shared__ unsigned long long s_rows[SHUF_MAX_PARTS + 1];
  for (int p = threadIdx.x; p <= P; p += VE_NT) s_rows[p] = vl.row_start[p];
  __syncthreads();
  const unsigned lane = threadIdx.x & 31;
  const long long warps = ((long long)gridDim.x * VE_NT) >> 5;
  for (long long base = ((blockIdx.x * (long long)VE_NT + threadIdx.x) >> 5) * 32; base < vl.n; base += warps * 32) {
    const long long q = base + lane;
    VlLoc l{0, 0, 0, 0};
    unsigned long long row = 0, rb = 0, m8 = 0; uint32_t vlen = 0;
    if (q < vl.n) {
      l = vl_locate(vl, s_rows, P, counts, (unsigned long long)q);
      row = vl.perm ? vl.perm[q] : (unsigned long long)q; rb = vl.rec_off[l.g]; m8 = (l.m + 7) >> 3; vlen = shuf_varint_len(l.m);
    }
    const int cnt = (int)(vl.n - base < 32 ? vl.n - base : 32);
    unsigned long long before = 0;
    for (int k = 0; k < vl.nb; k++) {
      const int c = vl.col[k];
      const ShufCol& col = sp.col[c];
      long long s0 = 0; unsigned long long d0 = 0; int len = 0;
      if (q < vl.n) {
        const unsigned long long* dk = vl.doff + (unsigned long long)k * (unsigned long long)(vl.n + 1);
        s0 = vl.offsets[k][row];
        len = (int)vl.lens[(unsigned long long)k * vl.n + q];
        d0 = rb + col_offset(sp, c, l.m, m8, vlen) + before + 1 + (col.nullable ? m8 : 0) + 4 * l.m + (dk[q] - dk[l.q0]);
        before += vl_bytes(vl, k, l.q0, l.m);
      }
      const uint8_t* data = (const uint8_t*)col.values;
      for (int i = 0; i < cnt; i++) {
        const uint8_t* sp8 = data + __shfl_sync(0xffffffffu, s0, i);
        uint8_t* dp = out + __shfl_sync(0xffffffffu, d0, i);
        const int n = __shfl_sync(0xffffffffu, len, i);
        int done = 0;
        if (n >= 64) {
          const int head = (int)((16 - ((uintptr_t)dp & 15)) & 15);
          if ((int)lane < head) dp[lane] = sp8[lane];
          const int nv = (n - head) >> 4;
          const uint8_t* s = sp8 + head; VlV16* vd = (VlV16*)(dp + head);
          const unsigned mis = (unsigned)((uintptr_t)s & 15);
          if (mis == 0) { const VlV16* vs = (const VlV16*)s; for (int v = (int)lane; v < nv; v += 32) vd[v] = vs[v]; }
          else { const VlV16* vs = (const VlV16*)(s - mis); for (int v = (int)lane; v < nv; v += 32) vd[v] = vl_shifted16(vs, v, mis); }
          done = head + (nv << 4);
        }
        for (int b = done + (int)lane; b < n; b += 32) dp[b] = sp8[b];
      }
    }
  }
}

}  // namespace

int launch_shuffle_pids(const ShufSpec& sp, int64_t n, uint16_t* d_pids, unsigned long long* d_counts, cudaStream_t s) {
  if (n <= 0) return 0;
  const int64_t want = (n + PID_BLOCK * 8 - 1) / (PID_BLOCK * 8);
  const int grid = (int)std::max<int64_t>(1, std::min<int64_t>(want, (int64_t)sm_count() * 8));
  shuffle_pids_kernel<<<grid, PID_BLOCK, 0, s>>>(sp, n, d_pids, d_counts);
  return 1;
}

int launch_shuffle_layout(const ShufSpec& sp, const unsigned long long* d_counts, unsigned long long* d_part_off, unsigned long long* d_cursors, uint8_t* d_out, cudaStream_t s) {
  shuffle_layout_kernel<<<1, 1024, 0, s>>>(sp, d_counts, d_part_off, d_cursors);
  if (!d_out) return 1;
  shuffle_headers_kernel<<<sp.num_partitions, 128, 0, s>>>(sp, d_counts, d_part_off, d_out);
  return 2;
}

int launch_shuffle_encode(const ShufSpec& sp, const uint16_t* d_pids, int64_t n, const unsigned long long* d_counts, const unsigned long long* d_part_off,
                          unsigned long long* d_cursors, uint8_t* d_out, cudaStream_t s) {
  if (n <= 0) return 0;
  ShufSpec spx = sp;
  bool tma = false;
#ifndef B200Q_EMULATED_DEVICE
  // the bulk-copy staging costs 64 KB more shared memory per CTA (a smaller L1 for the write-combining of the byte stores) but takes
  // the column loads off the warps' critical path; on H100 it is the faster form (bench.py M3, 200-way, 2^28 rows: 26.7 ms against
  // 30.4-31.2 ms per step, H100 SXM 80 GB at 700 W), so every column it can take uses it
  for (int c = 0; c < spx.ncols; c++) {                                                     // bulk copies need 16-byte aligned sources
    ShufCol& col = spx.col[c];
    col.tma = (col.width == 1 || col.width == 2 || col.width == 4 || col.width == 8) && ((uintptr_t)col.values & 15) == 0 && n >= SHUF_TILE;
    tma = tma || col.tma;
  }
#endif
  const size_t smem = (size_t)SHUF_TILE * (tma ? 24 : 8) + (size_t)spx.num_partitions * 16 + (size_t)SHUF_TILE * 2;
  const int64_t ntiles = (n + SHUF_TILE - 1) / SHUF_TILE;
  const int grid = (int)std::max<int64_t>(1, std::min<int64_t>(ntiles, (int64_t)sm_count() * 2));
#ifndef B200Q_EMULATED_DEVICE
  cudaFuncSetAttribute(shuffle_encode_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, SHUF_TILE * 10 + SHUF_MAX_PARTS * 16);      // per device: cheap, idempotent
  cudaFuncSetAttribute(shuffle_encode_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, SHUF_TILE * 26 + SHUF_MAX_PARTS * 16);
  if (tma) { shuffle_encode_kernel<true><<<grid, ENC_NT, smem, s>>>(spx, d_pids, n, d_counts, d_part_off, d_cursors, d_out); return 1; }
#endif
  shuffle_encode_kernel<false><<<grid, ENC_NT, smem, s>>>(spx, d_pids, n, d_counts, d_part_off, d_cursors, d_out);
  return 1;
}

int64_t shuffle_varlen_scan_blocks(int64_t n) { return (n + VS_TILE - 1) / VS_TILE; }

static int vl_grid(int64_t items, int per_sm) {
  return (int)std::max<int64_t>(1, std::min<int64_t>((items + 255) / 256, (int64_t)sm_count() * per_sm));
}

int launch_shuffle_varlen_encode(const ShufSpec& sp, const ShufVarlen& vl, const uint16_t* d_pids, const unsigned long long* d_counts,
                                 unsigned long long* d_cursors, unsigned long long* d_part_off, uint8_t* d_out, cudaStream_t s) {
  const int P = sp.num_partitions;
  int launches = 0;
  if (vl.perm) {
    cudaMemsetAsync(d_cursors, 0, (size_t)P * 8, s);
    const int64_t ntiles = (vl.n + SHUF_TILE - 1) / SHUF_TILE;
    const int grid = (int)std::max<int64_t>(1, std::min<int64_t>(ntiles, (int64_t)sm_count() * 2));
    shuffle_vl_rank_kernel<<<grid, VR_NT, 0, s>>>(vl, P, d_pids, d_cursors);
    launches++;
  }
  shuffle_vl_lengths_kernel<<<vl_grid(vl.n, 8), 256, 0, s>>>(sp, vl); launches++;
  for (int k = 0; k < vl.nb; k++) launches += vl_scan(vl.lens + (size_t)k * (size_t)vl.n, vl.doff + (size_t)k * (size_t)(vl.n + 1), vl.n, vl.sums, s);
  shuffle_vl_records_kernel<<<vl_grid(vl.R, 8), 256, 0, s>>>(sp, vl, P, d_counts); launches++;
  launches += vl_scan(vl.rec_size, vl.rec_off, vl.R, vl.sums, s);
  const int hgrid = vl_grid(std::max<int64_t>(vl.R, P + 1), 8);
  shuffle_vl_headers_kernel<<<hgrid, 256, 0, s>>>(sp, vl, P, d_counts, d_part_off, d_out); launches++;
  shuffle_vl_encode_kernel<<<vl_grid(vl.n, 8), VE_NT, 0, s>>>(sp, vl, P, d_counts, d_out); launches++;
  shuffle_vl_copy_kernel<<<vl_grid(vl.n, 8), VE_NT, 0, s>>>(sp, vl, P, d_counts, d_out); launches++;
  return launches;
}

int launch_shuffle_varlen_bytes(const ShufSpec& sp, const ShufVarlen& vl, unsigned long long* d_totals, cudaStream_t s) {
  if (vl.n <= 0 || vl.nb == 0) return 0;
  shuffle_vl_bytes_kernel<<<vl_grid(vl.n, 8), 256, 0, s>>>(sp, vl, d_totals);
  return 1;
}

}  // namespace b200q
