// Microbenchmark (VERDICT round 1, Next #6): can a range-packed radix pre-pass beat the L2 scattered-RED ceiling of M1
// (SUM + COUNT of an int64 value by an int64 key, 1 M dense keys, 2^28 rows) ?
//
//   pass 1  reads {key, value} (16 B/row), range-partitions the rows by key into B buckets (B = a multiple of the SM count) and writes
//           packed tuples {key - bucket base : 13 bits, value - value base : 35 bits} as 6 B/row (a u32 plane + a u16 plane) or 8 B/row
//   pass 2  one CTA per bucket streams its tuples and aggregates into a CTA-private shared-memory table, then stores the bucket's
//           slice of the dense {sum, count} table with plain stores (a key lives in exactly one bucket)
//
// The comparison points are the shipped forms: one RED sector per row into the L2-resident table ("direct") and the stream alone.
// Build: nvcc -O3 -std=c++17 -gencode arch=compute_90a,code=sm_90a -o radix_prepass radix_prepass.cu
#include <cstdio>
#include <cstdint>
#include <cstdlib>
#include <vector>
#include <algorithm>
#include <functional>
#include <cuda_runtime.h>
#define CK(x) do{cudaError_t e=(x); if(e!=cudaSuccess){printf("CUDA %s @%d\n",cudaGetErrorString(e),__LINE__);exit(1);} }while(0)

__device__ __forceinline__ uint64_t mix(uint64_t x){ x^=x>>33; x*=0xff51afd7ed558ccdULL; x^=x>>33; x*=0xc4ceb9fe1a85ec53ULL; x^=x>>33; return x; }
__global__ void gen(int64_t* k, int64_t* v, size_t n, uint64_t card){
  size_t i = blockIdx.x*(size_t)blockDim.x+threadIdx.x, st=(size_t)gridDim.x*blockDim.x;
  for(;i<n;i+=st){ uint64_t h=mix(i*0x9E3779B97F4A7C15ULL+12345); k[i]=(int64_t)(h%card); v[i]=(int64_t)(mix(h)%2000000)-1000000; }
}
__device__ __forceinline__ void red64(unsigned long long* p, unsigned long long v){ asm volatile("red.global.add.u64 [%0], %1;"::"l"(p),"l"(v):"memory"); }
__device__ __forceinline__ void ld256(const int64_t* p, int64_t (&r)[4]){   // two 128-bit loads: the widest on sm_90
  asm volatile("{.reg .b64 pol; createpolicy.fractional.L2::evict_first.b64 pol, 1.0;\n\tld.global.nc.L1::no_allocate.L2::cache_hint.v2.s64 {%0,%1}, [%4], pol;\n\tld.global.nc.L1::no_allocate.L2::cache_hint.v2.s64 {%2,%3}, [%4+16], pol;}":"=l"(r[0]),"=l"(r[1]),"=l"(r[2]),"=l"(r[3]):"l"(p));
}

// ---------------------------------------------------------------- the shipped form: one paired RED per row
__global__ void __launch_bounds__(512) direct_kernel(const int64_t* __restrict__ k, const int64_t* __restrict__ v, size_t n, unsigned long long* tab){
  const size_t nt=(size_t)gridDim.x*blockDim.x; const unsigned lane=threadIdx.x&31;
  for(size_t i=(blockIdx.x*(size_t)blockDim.x+threadIdx.x)*4;i+3<n;i+=nt*4){
    int64_t kk[4],vv[4]; ld256(k+i,kk); ld256(v+i,vv);
    #pragma unroll
    for(int r=0;r<4;r++){
      const uint64_t pk=__shfl_xor_sync(0xffffffffu,(uint64_t)kk[r],1);
      { const uint64_t g=(lane&1)?pk:(uint64_t)kk[r]; red64(tab+2*g+(lane&1),(lane&1)?1ULL:(unsigned long long)vv[r]); }
      { const uint64_t g=(lane&1)?(uint64_t)kk[r]:pk; red64(tab+2*g+((lane&1)^1),(lane&1)?(unsigned long long)vv[r]:1ULL); }
    }
  }
}

// ---------------------------------------------------------------- pass 1: tile-local counting sort by bucket, runs written per (tile, bucket)
// TILE rows per CTA iteration; bucket = (key - kbase) * B >> kbits  (B need not be a power of two); tuples: low 48 bits = local key | (value - vbase) << 13
template<int THREADS, int RPT, int TUPLE>
__global__ void __launch_bounds__(THREADS) partition_kernel(const int64_t* __restrict__ k, const int64_t* __restrict__ v, size_t n, int64_t kbase, int kbits, int64_t vbase, int B,
                                                            unsigned* __restrict__ cursor, size_t cap, uint32_t* __restrict__ lo, uint16_t* __restrict__ hi, uint64_t* __restrict__ t8,
                                                            unsigned* __restrict__ tile_ticket){
  constexpr int TILE = THREADS * RPT;
  extern __shared__ __align__(16) unsigned char smem[];
  uint64_t* s_tup = (uint64_t*)smem;                                  // TILE tuples in bucket order
  unsigned* s_cnt = (unsigned*)(s_tup + TILE);                        // B counts -> exclusive starts
  unsigned* s_dst = s_cnt + B;                                        // B global offsets of the runs (minus the start inside the tile)
  unsigned* s_first = s_dst + B;                                      // first key of every bucket
  uint16_t* s_bkt = (uint16_t*)(s_first + B);                         // TILE bucket ids in bucket order (so the writer knows its run)
  __shared__ unsigned s_warp[THREADS/32]; __shared__ unsigned s_tile;
  const unsigned t = threadIdx.x;
  const size_t ntiles = (n + TILE - 1) / TILE;
  for (int b = t; b < B; b += THREADS) s_first[b] = (unsigned)((((uint64_t)b << kbits) + B - 1) / B);   // ceil(b * 2^kbits / B)
  while (true) {
    if (t == 0) s_tile = atomicAdd(tile_ticket, 1u);
    for (int b = t; b < B; b += THREADS) s_cnt[b] = 0;
    __syncthreads();
    const size_t tile = s_tile;
    if (tile >= ntiles) return;
    const size_t base = tile * (size_t)TILE;
    // rows: thread t owns rows base + (j*THREADS + t)*4 .. +3  (256-bit loads, RPT/4 of them)
    uint64_t tup[RPT]; unsigned br[RPT];                              // br = bucket << 16 | arrival rank inside the tile's bucket
    #pragma unroll
    for (int j = 0; j < RPT/4; j++) {
      const size_t i = base + ((size_t)j*THREADS + t)*4;
      int64_t kk[4], vv[4];
      if (i + 3 < n) { ld256(k+i,kk); ld256(v+i,vv); }
      else { for (int r=0;r<4;r++){ kk[r] = i+r<n ? k[i+r] : kbase; vv[r] = i+r<n ? v[i+r] : vbase; } }
      #pragma unroll
      for (int r = 0; r < 4; r++) {
        const uint64_t dk = (uint64_t)(kk[r] - kbase);
        const unsigned b = (unsigned)((dk * (uint64_t)B) >> kbits);
        tup[j*4+r] = (dk - s_first[b]) | ((uint64_t)(vv[r] - vbase) << 13);                  // local key = key - first key of its bucket
        br[j*4+r] = (i + r < n) ? (b << 16 | atomicAdd(&s_cnt[b], 1u)) : 0xFFFFFFFFu;    // arrival order inside the tile is irrelevant for an aggregate
      }
    }
    __syncthreads();
    // exclusive scan of the B counts (B <= 1024: one value per thread for the first B threads) + global reservations
    {
      unsigned c = t < (unsigned)B ? s_cnt[t] : 0u, x = c;
      #pragma unroll
      for (int o = 1; o < 32; o <<= 1) { unsigned y = __shfl_up_sync(0xffffffffu, x, o); if ((t & 31) >= (unsigned)o) x += y; }
      if ((t & 31) == 31) s_warp[t >> 5] = x;
      __syncthreads();
      if (t < 32) { unsigned w = t < THREADS/32 ? s_warp[t] : 0u, z = w;
        #pragma unroll
        for (int o = 1; o < 32; o <<= 1) { unsigned y = __shfl_up_sync(0xffffffffu, z, o); if (t >= (unsigned)o) z += y; }
        if (t < THREADS/32) s_warp[t] = z - w; }
      __syncthreads();
      const unsigned start = x - c + s_warp[t >> 5];
      if (t < (unsigned)B) { s_cnt[t] = start; s_dst[t] = c ? atomicAdd(&cursor[t], c) - start : 0u; }
    }
    __syncthreads();
    #pragma unroll
    for (int j = 0; j < RPT; j++) if (br[j] != 0xFFFFFFFFu) { const unsigned p = s_cnt[br[j] >> 16] + (br[j] & 0xFFFFu); s_tup[p] = tup[j]; s_bkt[p] = (uint16_t)(br[j] >> 16); }
    __syncthreads();
    const unsigned rows = (unsigned)min((size_t)TILE, n - base);
    for (unsigned p = t; p < rows; p += THREADS) {
      const unsigned b = s_bkt[p]; const uint64_t x = s_tup[p];
      const size_t d = (size_t)b * cap + (size_t)(s_dst[b] + p);
      if (TUPLE == 8) t8[d] = x; else { lo[d] = (uint32_t)x; hi[d] = (uint16_t)(x >> 32); }
    }
    __syncthreads();
  }
}

// ---------------------------------------------------------------- pass 2: one CTA per bucket, shared-memory table
// 64-bit shared-memory atomicAdd is a CAS loop on sm_90a (SASS ATOMS.CAST.SPIN.64); 32-bit ones are native (ATOMS.ADD / ATOMS.POPC.INC). MODE:
//   0  sum: 64-bit CAS loop, count: 32-bit            1  sum: 32-bit add with the old value returned + a carry add into a high word when it wraps, count: 32-bit
//   2  ONE 64-bit CAS loop on {count : 24 | sum : 40} 3  like 1 without the carry (an upper bound: exact only while a key's sum stays below 2^32)
template<int MODE>
__device__ __forceinline__ void upd(unsigned char* smem, unsigned nk, uint64_t x) {
  const unsigned key = (unsigned)x & 8191u; const uint64_t val = x >> 13;
  if (MODE == 0) { atomicAdd((unsigned long long*)smem + key, (unsigned long long)val); atomicAdd((unsigned*)((unsigned long long*)smem + nk) + key, 1u); }
  else if (MODE == 2) { atomicAdd((unsigned long long*)smem + key, (unsigned long long)val + (1ULL << 40)); }
  else {
    unsigned* lo = (unsigned*)smem; unsigned* hi = lo + nk; unsigned* num = hi + nk;
    if (MODE == 1) { const unsigned old = atomicAdd(lo + key, (unsigned)val); if (old + (unsigned)val < old) atomicAdd(hi + key, 1u); }
    else atomicAdd(lo + key, (unsigned)val);
    atomicAdd(num + key, 1u);
  }
}
template<int THREADS, int TUPLE, int MODE>
__global__ void __launch_bounds__(THREADS) bucket_agg_kernel(const unsigned* __restrict__ cursor, size_t cap, const uint32_t* __restrict__ lo, const uint16_t* __restrict__ hi,
                                                             const uint64_t* __restrict__ t8, int kbits, int B, int64_t vbase, unsigned long long* __restrict__ tab){
  extern __shared__ __align__(16) unsigned char smem[];
  const unsigned b = blockIdx.x, t = threadIdx.x;
  const uint64_t first = (((uint64_t)b << kbits) + B - 1) / B, last = (((uint64_t)(b + 1) << kbits) + B - 1) / B;
  const unsigned nk = (unsigned)(last - first);
  for (unsigned i = t; i < nk * 3; i += THREADS) ((unsigned*)smem)[i] = 0;
  __syncthreads();
  const unsigned cnt = cursor[b];
  if (TUPLE == 8) {
    const uint64_t* p = t8 + (size_t)b * cap;
    unsigned i = t * 2;
    for (; i + 1 < cnt; i += THREADS * 2) { ulonglong2 x = *reinterpret_cast<const ulonglong2*>(p + i); upd<MODE>(smem, nk, x.x); upd<MODE>(smem, nk, x.y); }
    if (i < cnt) upd<MODE>(smem, nk, p[i]);
  } else {
    const uint32_t* pl = lo + (size_t)b * cap; const uint16_t* ph = hi + (size_t)b * cap;
    for (unsigned i = t * 4; i + 3 < cnt; i += THREADS * 4) {
      const uint4 l = *reinterpret_cast<const uint4*>(pl + i); const uint2 h = *reinterpret_cast<const uint2*>(ph + i);
      const uint32_t lw[4] = {l.x, l.y, l.z, l.w}; const uint32_t hw[4] = {h.x & 0xFFFFu, h.x >> 16, h.y & 0xFFFFu, h.y >> 16};
      #pragma unroll
      for (int r = 0; r < 4; r++) upd<MODE>(smem, nk, lw[r] | ((uint64_t)hw[r] << 32));
    }
    if (t == 0) for (unsigned j = cnt & ~3u; j < cnt; j++) upd<MODE>(smem, nk, pl[j] | ((uint64_t)ph[j] << 32));
  }
  __syncthreads();
  for (unsigned i = t; i < nk; i += THREADS) {                                      // sum of (v - vbase) -> sum of v
    unsigned long long sum; unsigned c;
    if (MODE == 0) { sum = ((unsigned long long*)smem)[i]; c = ((unsigned*)((unsigned long long*)smem + nk))[i]; }
    else if (MODE == 2) { const unsigned long long w = ((unsigned long long*)smem)[i]; sum = w & ((1ULL << 40) - 1); c = (unsigned)(w >> 40); }
    else { sum = ((unsigned*)smem)[i] | ((unsigned long long)((unsigned*)smem)[nk + i] << 32); c = ((unsigned*)smem)[2 * nk + i]; }
    tab[2 * (first + i)] = sum + (unsigned long long)((long long)c * vbase); tab[2 * (first + i) + 1] = c;
  }
}

// pass 2 alone at its speed of light: the same stream without the atomics
template<int THREADS>
__global__ void __launch_bounds__(THREADS) bucket_stream_kernel(const unsigned* __restrict__ cursor, size_t cap, const uint64_t* __restrict__ t8, unsigned long long* sink){
  const unsigned b = blockIdx.x, t = threadIdx.x; const unsigned cnt = cursor[b]; const uint64_t* p = t8 + (size_t)b * cap; unsigned long long a = 0;
  for (unsigned i = t * 2; i + 1 < cnt; i += THREADS * 2) { ulonglong2 x = *reinterpret_cast<const ulonglong2*>(p + i); a += x.x ^ x.y; }
  if (a == 0x123456789ULL) *sink = a;
}

static float time_ms(cudaStream_t s, int reps, const std::function<void()>& body, const std::function<void()>& before) {
  cudaEvent_t e0, e1; CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1)); std::vector<float> ms;
  for (int r = 0; r < reps + 2; r++) { before(); CK(cudaEventRecord(e0, s)); body(); CK(cudaEventRecord(e1, s)); CK(cudaEventSynchronize(e1)); float m; CK(cudaEventElapsedTime(&m, e0, e1)); if (r >= 2) ms.push_back(m); }
  std::sort(ms.begin(), ms.end()); return ms[ms.size() / 2];
}

int main(int argc, char** argv) {
  const size_t n = argc > 1 ? strtoull(argv[1], 0, 0) : (1ull << 28);
  const uint64_t card = argc > 2 ? strtoull(argv[2], 0, 0) : (1ull << 20);
  int kbits = 0; while ((1ull << kbits) < card) kbits++;
  cudaDeviceProp pr; CK(cudaGetDeviceProperties(&pr, 0)); const int sms = pr.multiProcessorCount;
  printf("device %s, %d SMs; rows %zu, keys %llu (dense range, %d bits), values in [-1e6, 1e6)\n", pr.name, sms, n, (unsigned long long)card, kbits);
  int64_t *k, *v; CK(cudaMalloc(&k, n * 8)); CK(cudaMalloc(&v, n * 8)); gen<<<sms * 8, 256>>>(k, v, n, card); CK(cudaDeviceSynchronize());
  unsigned long long *tab, *tab_ref; CK(cudaMalloc(&tab, card * 16)); CK(cudaMalloc(&tab_ref, card * 16));
  cudaStream_t s; CK(cudaStreamCreate(&s));
  const double hbm = 3350.0;                                            // GB/s: H100 SXM data-sheet HBM3 bandwidth
  // reference result + the shipped form's time
  float ms_direct = time_ms(s, 5, [&]{ direct_kernel<<<sms * 4, 512, 0, s>>>(k, v, n, tab_ref); }, [&]{ CK(cudaMemsetAsync(tab_ref, 0, card * 16, s)); });
  printf("%-58s %7.3f ms  %6.1f Grows/s  frac(16 B/row) %.3f\n", "direct: paired RED into the L2-resident table", ms_direct, n / ms_direct / 1e6, 16.0 * n / ms_direct / 1e6 / hbm);
  std::vector<unsigned long long> ref(card * 2); CK(cudaMemcpy(ref.data(), tab_ref, card * 16, cudaMemcpyDeviceToHost));

  unsigned *cursor, *ticket; CK(cudaMalloc(&cursor, 4096 * 4)); CK(cudaMalloc(&ticket, 4));
  const int64_t vbase = -1000000;
  for (int per_sm = 1; per_sm <= 2; per_sm++) {
    const int B = sms * per_sm;
    const size_t cap = ((size_t)((double)n / B * 1.05) + 4096 + 63) & ~(size_t)63;           // microbench: 5 % slack instead of a count pass
    uint32_t* lo; uint16_t* hi; uint64_t* t8;
    CK(cudaMalloc(&t8, cap * B * 8)); lo = (uint32_t*)t8; CK(cudaMalloc(&hi, cap * B * 2));
    const unsigned nk_max = (unsigned)((card + B - 1) / B + 1);
    if (nk_max > 8192) { printf("B=%d: %u keys per bucket exceed the 13-bit local key\n", B, nk_max); continue; }
    for (int cfg = 0; cfg < 3; cfg++) for (int tuple : {8, 6}) {
      if (getenv("ONLY")) { int oc, ot, op; if (sscanf(getenv("ONLY"), "%d,%d,%d", &oc, &ot, &op) == 3 && (oc != cfg || ot != tuple || op != per_sm)) continue; }
      auto reset = [&]{ CK(cudaMemsetAsync(cursor, 0, 4096 * 4, s)); CK(cudaMemsetAsync(ticket, 0, 4, s)); };
      auto launch_p1 = [&](auto kern, int th, int rpt, int ctas_per_sm) {
        const size_t sm1 = (size_t)th * rpt * 10 + (size_t)B * 12;
        CK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm1));
        kern<<<sms * ctas_per_sm, th, sm1, s>>>(k, v, n, (int64_t)0, kbits, vbase, B, cursor, cap, lo, hi, t8, ticket);
      };
      auto p1 = [&]{
        if (cfg == 0) { if (tuple == 8) launch_p1(partition_kernel<512, 8, 8>, 512, 8, 3); else launch_p1(partition_kernel<512, 8, 6>, 512, 8, 3); }
        if (cfg == 1) { if (tuple == 8) launch_p1(partition_kernel<1024, 8, 8>, 1024, 8, 1); else launch_p1(partition_kernel<1024, 8, 6>, 1024, 8, 1); }
        if (cfg == 2) { if (tuple == 8) launch_p1(partition_kernel<512, 16, 8>, 512, 16, 2); else launch_p1(partition_kernel<512, 16, 6>, 512, 16, 2); }
      };
      const size_t sm2 = (size_t)nk_max * 12 + 16;
      int mode = 0;
      auto launch_p2 = [&](auto kern) { CK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm2)); kern<<<B, 1024, sm2, s>>>(cursor, cap, lo, hi, t8, kbits, B, vbase, tab); };
      auto p2 = [&]{
        if (tuple == 8) { if (mode == 0) launch_p2(bucket_agg_kernel<1024, 8, 0>); if (mode == 1) launch_p2(bucket_agg_kernel<1024, 8, 1>); if (mode == 2) launch_p2(bucket_agg_kernel<1024, 8, 2>); if (mode == 3) launch_p2(bucket_agg_kernel<1024, 8, 3>); }
        else            { if (mode == 0) launch_p2(bucket_agg_kernel<1024, 6, 0>); if (mode == 1) launch_p2(bucket_agg_kernel<1024, 6, 1>); if (mode == 2) launch_p2(bucket_agg_kernel<1024, 6, 2>); if (mode == 3) launch_p2(bucket_agg_kernel<1024, 6, 3>); }
      };
      const float ms1 = time_ms(s, 5, p1, reset);
      CK(cudaGetLastError());
      float ms2m[4];
      for (mode = 0; mode < 4; mode++) { ms2m[mode] = time_ms(s, 5, p2, []{}); CK(cudaGetLastError()); }
      mode = 1;
      const float ms12 = time_ms(s, 5, [&]{ p1(); p2(); }, reset);
      std::vector<unsigned> cur(B); CK(cudaMemcpy(cur.data(), cursor, B * 4, cudaMemcpyDeviceToHost));
      size_t tot = 0; unsigned mx = 0; for (unsigned c : cur) { tot += c; mx = std::max(mx, c); }
      std::vector<unsigned long long> got(card * 2); CK(cudaMemcpy(got.data(), tab, card * 16, cudaMemcpyDeviceToHost));
      size_t bad = 0; for (size_t i = 0; i < card * 2; i++) bad += got[i] != ref[i];
      char name[128];
      snprintf(name, sizeof name, "B=%d, %d-byte tuples, tile %s: pass 1 (partition)", B, tuple, cfg == 0 ? "512x8" : cfg == 1 ? "1024x8" : "512x16");
      printf("%-58s %7.3f ms  %6.1f Grows/s  frac(%d B/row moved) %.3f\n", name, ms1, n / ms1 / 1e6, 16 + tuple, (16.0 + tuple) * n / ms1 / 1e6 / hbm);
      static const char* mname[4] = {"64-bit CAS sum + count", "32-bit sum w/ carry + count", "one packed 64-bit CAS", "32-bit sum, no carry + count"};
      for (int m = 0; m < 4; m++) {
        snprintf(name, sizeof name, "B=%d, %d-byte tuples: pass 2 [%s]", B, tuple, mname[m]);
        printf("%-66s %7.3f ms  %6.1f Grows/s  frac(%d B/row moved) %.3f\n", name, ms2m[m], n / ms2m[m] / 1e6, tuple, (double)tuple * n / ms2m[m] / 1e6 / hbm);
      }
      snprintf(name, sizeof name, "B=%d, %d-byte tuples: both passes (pass 2 = 32-bit w/ carry)", B, tuple);
      printf("%-58s %7.3f ms  %6.1f Grows/s  frac(16 B/row) %.3f   vs direct %.2fx   rows placed %zu (max bucket %u of cap %zu)  mismatching words %zu\n",
             name, ms12, n / ms12 / 1e6, 16.0 * n / ms12 / 1e6 / hbm, ms_direct / ms12, tot, mx, cap, bad);
      if (tuple == 8 && cfg == 0) {
        unsigned long long* sink; CK(cudaMalloc(&sink, 8));
        const float ms3 = time_ms(s, 5, [&]{ bucket_stream_kernel<1024><<<B, 1024, 0, s>>>(cursor, cap, t8, sink); }, []{});
        snprintf(name, sizeof name, "B=%d buckets: pass 2 stream only (no atomics)", B);
        printf("%-58s %7.3f ms  %6.1f Grows/s  frac(8 B/row moved) %.3f\n", name, ms3, n / ms3 / 1e6, 8.0 * n / ms3 / 1e6 / hbm);
        CK(cudaFree(sink));
      }
    }
    CK(cudaFree(t8)); CK(cudaFree(hi));
  }
  return 0;
}
