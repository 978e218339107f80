// Microbenchmark 2: cost of the hash-probe load flavour and of the table size (L2 residency across the two dies).
// Build: nvcc -O3 -gencode arch=compute_90a,code=sm_90a -o probes probes.cu
#include <cstdio>
#include <cstdint>
#include <cstdlib>
#include <cuda_runtime.h>
#define CK(x) do{cudaError_t e=(x); if(e!=cudaSuccess){printf("CUDA %s @%d\n",cudaGetErrorString(e),__LINE__);exit(1);} }while(0)
__device__ __forceinline__ uint64_t mix(uint64_t x){ x^=x>>33; x*=0xff51afd7ed558ccdULL; x^=x>>33; x*=0xc4ceb9fe1a85ec53ULL; x^=x>>33; return x; }
__global__ void gen(int64_t* k, size_t n, uint64_t card){ size_t i=blockIdx.x*(size_t)blockDim.x+threadIdx.x, st=(size_t)gridDim.x*blockDim.x; for(;i<n;i+=st) k[i]=(int64_t)(mix(i*0x9E3779B97F4A7C15ULL+12345)%card); }
__global__ void fill(unsigned long long* t, size_t slots){ size_t i=blockIdx.x*(size_t)blockDim.x+threadIdx.x, st=(size_t)gridDim.x*blockDim.x; for(;i<slots;i+=st){ t[4*i]=i|0x8000000000000000ULL; t[4*i+1]=i; } }
// FLAVOUR 0: ld.relaxed.gpu (strong)  1: ld.global.cg  2: ld.global.nc  3: plain ld.global  4: ld.volatile
template<int F> __device__ __forceinline__ ulonglong2 probe(const unsigned long long* p){
  ulonglong2 v;
  if(F==0) asm volatile("ld.relaxed.gpu.global.v2.u64 {%0,%1}, [%2];":"=l"(v.x),"=l"(v.y):"l"(p):"memory");
  else if(F==1) asm volatile("ld.global.cg.v2.u64 {%0,%1}, [%2];":"=l"(v.x),"=l"(v.y):"l"(p):"memory");
  else if(F==2) asm volatile("ld.global.nc.v2.u64 {%0,%1}, [%2];":"=l"(v.x),"=l"(v.y):"l"(p));
  else if(F==3) asm volatile("ld.global.v2.u64 {%0,%1}, [%2];":"=l"(v.x),"=l"(v.y):"l"(p):"memory");
  else asm volatile("ld.volatile.global.v2.u64 {%0,%1}, [%2];":"=l"(v.x),"=l"(v.y):"l"(p):"memory");
  return v;
}
template<int F, int WITH_RED>
__global__ void __launch_bounds__(256) k(const int64_t* __restrict__ keys, size_t n, unsigned long long* t, uint64_t mask, unsigned long long* sink, unsigned long long* t2){
  size_t tid=blockIdx.x*(size_t)blockDim.x+threadIdx.x, nt=(size_t)gridDim.x*blockDim.x; unsigned long long acc=0;
  for(size_t i=tid;i<n;i+=nt*4){
    long long kk[4]; ulonglong2 h[4]; unsigned long long* s[4];
    #pragma unroll
    for(int u=0;u<4;u++){ size_t j=i+u*nt; kk[u]= j<n? __ldg((const long long*)keys+j):0; }
    #pragma unroll
    for(int u=0;u<4;u++){ s[u]=t+4*((uint64_t)kk[u]&mask); h[u]=probe<F>(s[u]); }   // identity "hash": slot = key (table pre-filled), measures the load path only
    #pragma unroll
    for(int u=0;u<4;u++){ acc+=h[u].y; if(WITH_RED==1){ asm volatile("red.global.add.u64 [%0], %1;"::"l"(s[u]+2),"l"(1ULL):"memory"); } if(WITH_RED==2){ asm volatile("red.global.add.u64 [%0], %1;"::"l"(t2+2*((uint64_t)kk[u]&mask)),"l"(1ULL):"memory"); } }
  }
  if(acc==0x1234567) sink[0]=acc;
}
template<int F,int R> float run(const int64_t* keys,size_t n,unsigned long long* t,uint64_t mask,unsigned long long* sink,unsigned long long* t2=nullptr){
  cudaEvent_t a,b; CK(cudaEventCreate(&a)); CK(cudaEventCreate(&b)); float best=1e9;
  for(int it=0;it<3;it++){ CK(cudaEventRecord(a)); k<F,R><<<132*8,256>>>(keys,n,t,mask,sink,t2); CK(cudaEventRecord(b)); CK(cudaEventSynchronize(b)); CK(cudaGetLastError()); float ms; CK(cudaEventElapsedTime(&ms,a,b)); if(it>0&&ms<best)best=ms; }
  return best;
}
int main(){
  size_t n=(size_t)256<<20; int64_t* keys; CK(cudaMalloc(&keys,n*8)); unsigned long long* sink; CK(cudaMalloc(&sink,8));
  const char* names[]={"ld.relaxed.gpu","ld.global.cg","ld.global.nc","ld.global","ld.volatile"};
  for(int lg=18; lg<=23; lg++){
    size_t slots=(size_t)1<<lg; unsigned long long* t; CK(cudaMalloc(&t,slots*32));
    fill<<<132*8,256>>>(t,slots); gen<<<132*8,256>>>(keys,n,slots); CK(cudaDeviceSynchronize());
    float ms[5][2];
    ms[0][0]=run<0,0>(keys,n,t,slots-1,sink); ms[0][1]=run<0,1>(keys,n,t,slots-1,sink);
    ms[1][0]=run<1,0>(keys,n,t,slots-1,sink); ms[1][1]=run<1,1>(keys,n,t,slots-1,sink);
    ms[2][0]=run<2,0>(keys,n,t,slots-1,sink); ms[2][1]=run<2,1>(keys,n,t,slots-1,sink);
    ms[3][0]=run<3,0>(keys,n,t,slots-1,sink); ms[3][1]=run<3,1>(keys,n,t,slots-1,sink);
    ms[4][0]=run<4,0>(keys,n,t,slots-1,sink); ms[4][1]=run<4,1>(keys,n,t,slots-1,sink);
    { unsigned long long* t2; CK(cudaMalloc(&t2,slots*16)); CK(cudaMemset(t2,0,slots*16)); float a=run<0,2>(keys,n,t,slots-1,sink,t2), b=run<3,2>(keys,n,t,slots-1,sink,t2);
      printf("table=%4zu MB keys(32B slots) + %zu MB separate accumulator array: probe(ld.relaxed.gpu)+RED(other array) %.3f ms %.3e rows/s | probe(ld.global)+RED(other array) %.3f ms %.3e rows/s\n",slots*32>>20,slots*16>>20,a,n/(a*1e-3),b,n/(b*1e-3)); CK(cudaFree(t2)); }
    for(int f=0;f<5;f++) printf("table=%4zu MB (%zu slots x 32B)  %-15s probe-only %.3f ms %.3e rows/s | probe+RED(same sector) %.3f ms %.3e rows/s\n",slots*32>>20,slots,names[f],ms[f][0],n/(ms[f][0]*1e-3),ms[f][1],n/(ms[f][1]*1e-3));
    CK(cudaFree(t));
  }
  return 0;
}
