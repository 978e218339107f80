// Host stand-in for <cuda_runtime.h>: lets the HashAgg kernel SOURCES (copied and asm-translated by
// tools/emu/build_emu.py) compile with g++ and run one OS thread per CUDA thread, so that the kernel LOGIC
// (dispatch forms, lane exchange, shared-memory tables, insert protocol) can be unit-tested without a GPU.
// Test infrastructure only: nothing under blaze_b200/ includes this file; it is no CPU fallback of the product.
#pragma once
#include <math.h>
#include <stdlib.h>
#include <time.h>

#include <atomic>
#include <barrier>
#include <cstdint>
#include <cstring>
#include <memory>
#include <mutex>
#include <thread>
#include <vector>

#define B200Q_EMULATED_DEVICE 1
#define __global__
#define __device__
#define __host__
#define __forceinline__ inline
#define __restrict__
#define __launch_bounds__(...)
#define __shared__ static

struct uint3 { unsigned x, y, z; };
struct dim3 { unsigned x = 1, y = 1, z = 1; };
struct ulonglong2 { unsigned long long x, y; };
typedef void* cudaStream_t;

namespace emu {
struct Warp { std::barrier<> bar{32}; unsigned long long slot[32]; };
struct Block { std::unique_ptr<std::barrier<>> bar; std::vector<std::unique_ptr<Warp>> warps; };
inline thread_local Warp* warp = nullptr;
inline thread_local Block* block = nullptr;
inline thread_local unsigned lane = 0;
}  // namespace emu
inline thread_local uint3 threadIdx, blockIdx;
inline thread_local dim3 blockDim, gridDim;

// ---- block / warp collectives (all callers use full masks in converged code) ----
inline void __syncthreads() { emu::block->bar->arrive_and_wait(); }
inline void __syncwarp(unsigned = 0xffffffffu) { emu::warp->bar.arrive_and_wait(); }
template <class T> inline T emu_exchange(T v, unsigned src) {
  static_assert(sizeof(T) <= 8, "exchange of up to 8 bytes");
  unsigned long long raw = 0; memcpy(&raw, &v, sizeof(T));
  emu::warp->slot[emu::lane] = raw;
  emu::warp->bar.arrive_and_wait();
  raw = emu::warp->slot[src & 31];
  emu::warp->bar.arrive_and_wait();
  T out; memcpy(&out, &raw, sizeof(T)); return out;
}
template <class T> inline T __shfl_sync(unsigned, T v, int src, int width = 32) { return emu_exchange(v, (emu::lane & ~(unsigned)(width - 1)) + ((unsigned)src & (unsigned)(width - 1))); }
template <class T> inline T __shfl_xor_sync(unsigned, T v, int m, int width = 32) { (void)width; return emu_exchange(v, emu::lane ^ (unsigned)m); }
template <class T> inline T __shfl_up_sync(unsigned, T v, unsigned d, int width = 32) { (void)width; return emu_exchange(v, emu::lane >= d ? emu::lane - d : emu::lane); }
inline unsigned __ballot_sync(unsigned, bool p) {
  emu::warp->slot[emu::lane] = p ? 1 : 0;
  emu::warp->bar.arrive_and_wait();
  unsigned m = 0; for (int i = 0; i < 32; i++) m |= (unsigned)(emu::warp->slot[i] & 1) << i;
  emu::warp->bar.arrive_and_wait();
  return m;
}
inline bool __any_sync(unsigned mask, bool p) { return __ballot_sync(mask, p) != 0; }
inline bool __all_sync(unsigned mask, bool p) { return __ballot_sync(mask, p) == 0xffffffffu; }

// ---- scalar intrinsics ----
inline int __popc(unsigned x) { return __builtin_popcount(x); }
inline int __ffs(unsigned x) { return __builtin_ffs((int)x); }
inline unsigned __umulhi(unsigned a, unsigned b) { return (unsigned)(((unsigned long long)a * b) >> 32); }
inline unsigned long long __umul64hi(unsigned long long a, unsigned long long b) { return (unsigned long long)(((unsigned __int128)a * b) >> 64); }
template <class T> inline T __ldg(const T* p) { return *p; }
inline void __nanosleep(unsigned) { std::this_thread::yield(); }
inline void __threadfence() { std::atomic_thread_fence(std::memory_order_seq_cst); }
inline long long clock64() { return 0; }
template <class T> inline T max(T a, T b) { return a > b ? a : b; }
template <class T> inline T min(T a, T b) { return a < b ? a : b; }

inline double __longlong_as_double(long long v) { double d; memcpy(&d, &v, 8); return d; }
inline long long __double_as_longlong(double d) { long long v; memcpy(&v, &d, 8); return v; }
inline float __int_as_float(int v) { float f; memcpy(&f, &v, 4); return f; }
inline double __ull2double_rn(unsigned long long v) { return (double)v; }
inline double __ll2double_rn(long long v) { return (double)v; }
inline float __ll2float_rn(long long v) { return (float)v; }
inline float __double2float_rn(double v) { return (float)v; }
inline long long __double2ll_rn(double v) { return (long long)nearbyint(v); }
inline long long __double2ll_rz(double v) { return v != v ? INT64_MIN /* cvt.rzi.s64.f64 maps NaN to 0x8000000000000000 (what the device conversion returns) */ : v >= 9223372036854775807.0 ? INT64_MAX : v <= -9223372036854775808.0 ? INT64_MIN : (long long)v; }
inline float __fadd_rn(float a, float b) { return a + b; }
inline float __fsub_rn(float a, float b) { return a - b; }
inline float __fmul_rn(float a, float b) { return a * b; }
inline float __fdiv_rn(float a, float b) { return a / b; }
inline double __dadd_rn(double a, double b) { return a + b; }
inline double __dsub_rn(double a, double b) { return a - b; }
inline double __dmul_rn(double a, double b) { return a * b; }
inline double __ddiv_rn(double a, double b) { return a / b; }
inline int __clzll(long long v) { return v == 0 ? 64 : __builtin_clzll((unsigned long long)v); }
inline unsigned __reduce_or_sync(unsigned, unsigned v) { unsigned r = 0; for (int i = 0; i < 32; i++) r |= emu_exchange(v, (unsigned)i); return r; }

// ---- atomics (global and "shared" memory alike) ----
template <class T> inline T atomicAdd(T* p, T v) { return __atomic_fetch_add(p, v, __ATOMIC_RELAXED); }
inline unsigned long long atomicAdd(unsigned long long* p, unsigned long long v) { return __atomic_fetch_add(p, v, __ATOMIC_RELAXED); }
template <class T> inline T atomicOr(T* p, T v) { return __atomic_fetch_or(p, v, __ATOMIC_RELAXED); }
template <class T> inline T atomicExch(T* p, T v) { return __atomic_exchange_n(p, v, __ATOMIC_ACQ_REL); }
template <class T> inline T atomicAnd(T* p, T v) { return __atomic_fetch_and(p, v, __ATOMIC_RELAXED); }
template <class T> inline T atomicCAS(T* p, T cmp, T val) { __atomic_compare_exchange_n(p, &cmp, val, false, __ATOMIC_ACQ_REL, __ATOMIC_ACQUIRE); return cmp; }
template <class T> inline T atomicMax(T* p, T v) { T o = __atomic_load_n(p, __ATOMIC_RELAXED); while (o < v && !__atomic_compare_exchange_n(p, &o, v, false, __ATOMIC_RELAXED, __ATOMIC_RELAXED)) {} return o; }
template <class T> inline T atomicMin(T* p, T v) { T o = __atomic_load_n(p, __ATOMIC_RELAXED); while (o > v && !__atomic_compare_exchange_n(p, &o, v, false, __ATOMIC_RELAXED, __ATOMIC_RELAXED)) {} return o; }

// ---- what tools/emu/build_emu.py maps the inline PTX onto ----
inline unsigned long long emu_ld64(const unsigned long long* p) { return __atomic_load_n(p, __ATOMIC_ACQUIRE); }
inline void emu_st_release32(unsigned* p, unsigned v) { __atomic_store_n(p, v, __ATOMIC_RELEASE); }
inline void emu_st64(unsigned long long* p, unsigned long long v) { __atomic_store_n(p, v, __ATOMIC_RELAXED); }
inline void emu_red_add_u64(unsigned long long* p, unsigned long long v) { __atomic_fetch_add(p, v, __ATOMIC_RELAXED); }
inline void emu_red_add_f64(unsigned long long* p, double v) {
  unsigned long long o = __atomic_load_n(p, __ATOMIC_RELAXED), nw;
  do { double d; memcpy(&d, &o, 8); d += v; memcpy(&nw, &d, 8); } while (!__atomic_compare_exchange_n(p, &o, nw, false, __ATOMIC_RELAXED, __ATOMIC_RELAXED));
}
inline void emu_red_min_s64(unsigned long long* p, long long v) { atomicMin((long long*)p, v); }
inline void emu_red_max_s64(unsigned long long* p, long long v) { atomicMax((long long*)p, v); }
inline unsigned emu_lanemask_lt() { return (1u << emu::lane) - 1u; }

// ---- CUDA runtime API: the "device" is host memory, streams are synchronous ----
typedef int cudaError_t;
typedef struct emu_event_s { double t; }* cudaEvent_t;
typedef void* cudaMemPool_t;
enum { cudaSuccess = 0, cudaErrorMemoryAllocation = 2, cudaErrorNotReady = 600, cudaDevAttrMultiProcessorCount = 16, cudaStreamNonBlocking = 1, cudaEventDisableTiming = 2,
       cudaMemPoolAttrReleaseThreshold = 4 };
enum cudaMemcpyKind { cudaMemcpyHostToHost = 0, cudaMemcpyHostToDevice = 1, cudaMemcpyDeviceToHost = 2, cudaMemcpyDeviceToDevice = 3, cudaMemcpyDefault = 4 };
inline const char* cudaGetErrorString(cudaError_t) { return "emulated device error"; }
inline cudaError_t cudaGetLastError() { return cudaSuccess; }
inline cudaError_t cudaGetDeviceCount(int* n) { *n = 1; return cudaSuccess; }
inline cudaError_t cudaSetDevice(int) { return cudaSuccess; }
inline cudaError_t cudaGetDevice(int* d) { *d = 0; return cudaSuccess; }
inline cudaError_t cudaDeviceGetAttribute(int* v, int, int) { *v = 1; return cudaSuccess; }   // one "SM": small grids
template <class F> inline cudaError_t cudaOccupancyMaxActiveBlocksPerMultiprocessor(int* v, F, int, size_t) { *v = 1; return cudaSuccess; }
inline cudaError_t cudaDeviceGetDefaultMemPool(cudaMemPool_t* p, int) { *p = nullptr; return cudaSuccess; }
inline cudaError_t cudaMemPoolSetAttribute(cudaMemPool_t, int, void*) { return cudaSuccess; }
inline cudaError_t cudaStreamCreateWithFlags(cudaStream_t* s, unsigned) { *s = (cudaStream_t)malloc(8); return cudaSuccess; }
inline cudaError_t cudaStreamDestroy(cudaStream_t s) { free(s); return cudaSuccess; }
inline cudaError_t cudaStreamSynchronize(cudaStream_t) { return cudaSuccess; }
inline cudaError_t cudaStreamWaitEvent(cudaStream_t, cudaEvent_t, unsigned) { return cudaSuccess; }
inline double emu_now_ms() { timespec ts; clock_gettime(CLOCK_MONOTONIC, &ts); return ts.tv_sec * 1e3 + ts.tv_nsec * 1e-6; }
inline cudaError_t cudaEventCreate(cudaEvent_t* e) { *e = new emu_event_s{0}; return cudaSuccess; }
inline cudaError_t cudaEventCreateWithFlags(cudaEvent_t* e, unsigned) { return cudaEventCreate(e); }
inline cudaError_t cudaEventDestroy(cudaEvent_t e) { delete e; return cudaSuccess; }
inline cudaError_t cudaEventRecord(cudaEvent_t e, cudaStream_t) { e->t = emu_now_ms(); return cudaSuccess; }
inline cudaError_t cudaEventSynchronize(cudaEvent_t) { return cudaSuccess; }
inline cudaError_t cudaEventQuery(cudaEvent_t) { return cudaSuccess; }
inline cudaError_t cudaEventElapsedTime(float* ms, cudaEvent_t a, cudaEvent_t b) { *ms = (float)(b->t - a->t); return cudaSuccess; }
inline cudaError_t cudaMallocAsync(void** p, size_t n, cudaStream_t) { *p = malloc(n ? n : 1); return *p ? cudaSuccess : 2; }
inline cudaError_t cudaFreeAsync(void* p, cudaStream_t) { free(p); return cudaSuccess; }
inline cudaError_t cudaFree(void* p) { free(p); return cudaSuccess; }
template <class T> inline cudaError_t cudaMallocHost(T** p, size_t n) { *p = (T*)malloc(n ? n : 1); return *p ? cudaSuccess : 2; }
inline cudaError_t cudaFreeHost(void* p) { free(p); return cudaSuccess; }
inline cudaError_t cudaMemcpyAsync(void* d, const void* s, size_t n, int, cudaStream_t) { if (n) memmove(d, s, n); return cudaSuccess; }
inline cudaError_t cudaMemsetAsync(void* p, int v, size_t n, cudaStream_t) { if (n) memset(p, v, n); return cudaSuccess; }

// ---- launch: one OS thread per CUDA thread, the blocks of the grid one after the other ----
namespace emu {
template <class F> void launch(unsigned grid, unsigned block_threads, F&& kernel_body) {
  for (unsigned b = 0; b < grid; b++) {
    Block blk; blk.bar = std::make_unique<std::barrier<>>((std::ptrdiff_t)block_threads);
    for (unsigned w = 0; w < (block_threads + 31) / 32; w++) blk.warps.push_back(std::make_unique<Warp>());
    std::vector<std::thread> ts;
    for (unsigned t = 0; t < block_threads; t++)
      ts.emplace_back([&, t] {
        threadIdx = {t, 0, 0}; blockIdx = {b, 0, 0}; blockDim.x = block_threads; gridDim.x = grid;
        block = &blk; warp = blk.warps[t / 32].get(); lane = t & 31;
        kernel_body();
      });
    for (auto& th : ts) th.join();
  }
}
struct Launcher {
  unsigned grid, block;
  Launcher(long long g, long long b, long long /*smem*/ = 0, cudaStream_t /*stream*/ = nullptr) : grid((unsigned)g), block((unsigned)b) {}
  // `__shared__` variables are function-local statics here: launches from different host threads (ranks-as-threads tests) are serialised
  template <class F> void run(F&& body) { std::lock_guard<std::mutex> l(launch_mutex()); launch(grid, block, body); }
  static std::mutex& launch_mutex() { static std::mutex m; return m; }
};
}  // namespace emu
