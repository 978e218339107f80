// Microbenchmark: how fast can an H100 do "random RMW into an L2-resident group table" ?
// Decides the HashAgg slot layout (SoA vs AoS, paired lanes, probe + RED).
// Build: nvcc -O3 -gencode arch=compute_90a,code=sm_90a -o atomics atomics.cu
#include <cstdio>
#include <cstdint>
#include <cstdlib>
#include <cuda_runtime.h>
#define CK(x) do{cudaError_t e=(x); if(e!=cudaSuccess){printf("CUDA %s @%d\n",cudaGetErrorString(e),__LINE__);exit(1);} }while(0)

__device__ __forceinline__ uint64_t mix(uint64_t x){ x^=x>>33; x*=0xff51afd7ed558ccdULL; x^=x>>33; x*=0xc4ceb9fe1a85ec53ULL; x^=x>>33; return x; }

__global__ void gen(int64_t* k, int64_t* v, size_t n, uint64_t card){
  size_t i = blockIdx.x*(size_t)blockDim.x+threadIdx.x, st=(size_t)gridDim.x*blockDim.x;
  for(;i<n;i+=st){ uint64_t h=mix(i*0x9E3779B97F4A7C15ULL+12345); k[i]=(int64_t)(h%card); v[i]=(int64_t)(mix(h)%2000000)-1000000; }
}
__device__ __forceinline__ void red64(unsigned long long* p, unsigned long long v){ asm volatile("red.global.add.u64 [%0], %1;"::"l"(p),"l"(v):"memory"); }
__device__ __forceinline__ longlong2 ldnc2(const int64_t* p){ longlong2 r; asm volatile("ld.global.nc.L1::no_allocate.v2.s64 {%0,%1}, [%2];":"=l"(r.x),"=l"(r.y):"l"(p)); return r; }

// mode 0: stream only (sum into register, write 1 value per thread at end)
// mode 1: SoA sum[]/cnt[] direct index, 2 REDs
// mode 2: AoS 16B {sum,cnt} direct index, 2 REDs same sector
// mode 3: AoS 16B, one RED only (sum)
// mode 4: AoS 16B paired lanes (even lane: sum, odd lane: cnt of partner row) -> 2 instr per 2 rows
// mode 5: AoS 32B slot {hdr,key,sum,cnt} hashed; 16B probe load + 2 REDs
// mode 6: AoS 32B slot probe + paired lanes
// mode 7: SoA, atomicAdd with return (ATOMG)
// mode 8: AoS 32B slot probe only (no REDs)
template<int MODE>
__global__ void __launch_bounds__(256) agg(const int64_t* __restrict__ k, const int64_t* __restrict__ v, size_t n,
                    unsigned long long* t0, unsigned long long* t1, uint64_t mask, unsigned long long* sink){
  size_t tid = blockIdx.x*(size_t)blockDim.x+threadIdx.x, nt=(size_t)gridDim.x*blockDim.x;
  unsigned long long acc=0;
  const unsigned lane = threadIdx.x&31;
  // each thread handles 2 consecutive rows per iteration via 16B loads
  for(size_t i=tid*2;i+1<n;i+=nt*2){
    longlong2 kk=ldnc2(k+i), vv=ldnc2(v+i);
    #pragma unroll
    for(int r=0;r<2;r++){
      uint64_t key = r?kk.y:kk.x; unsigned long long val = r?vv.y:vv.x;
      if(MODE==0){ acc+=key^val; }
      else if(MODE==1){ red64(t0+key,val); red64(t1+key,1); }
      else if(MODE==2){ red64(t0+2*key,val); red64(t0+2*key+1,1); }
      else if(MODE==3){ red64(t0+2*key,val); }
      else if(MODE==4){
        // instruction A: even lanes own row; odd lanes help even partner
        uint64_t pk = __shfl_xor_sync(0xffffffffu,key,1); unsigned long long pv=__shfl_xor_sync(0xffffffffu,val,1);
        // step 1: rows of even lanes: even lane -> sum(own), odd lane -> cnt(partner=even's row)
        { uint64_t g = (lane&1)? pk:key; unsigned long long x=(lane&1)?1ULL:val; red64(t0+2*g+(lane&1),x); }
        // step 2: rows of odd lanes: odd lane -> sum(own)... keep adjacency: even lane -> cnt... order within sector irrelevant
        { uint64_t g = (lane&1)? key:pk; unsigned long long x=(lane&1)?val:1ULL; red64(t0+2*g+((lane&1)^1),x); }
        (void)pv;
      }
      else if(MODE==5||MODE==6||MODE==8){
        uint64_t h = mix(key); uint64_t s = h & mask; unsigned tag = (unsigned)(h>>32)|0x80000000u;
        unsigned long long* slot;
        while(true){
          slot = t0 + 4*s;
          ulonglong2 hk; asm volatile("ld.relaxed.gpu.global.v2.u64 {%0,%1}, [%2];":"=l"(hk.x),"=l"(hk.y):"l"(slot));
          unsigned t=(unsigned)hk.x;
          if(t==tag && hk.y==key) break;
          if(t==0){
            unsigned old = atomicCAS((unsigned*)slot,0u,1u);
            if(old==0){ slot[1]=key; __threadfence(); asm volatile("st.release.gpu.global.u32 [%0], %1;"::"l"(slot),"r"(tag):"memory"); break; }
            continue;
          }
          if(t==1) continue;
          s=(s+1)&mask;
        }
        if(MODE==5){ red64(slot+2,val); red64(slot+3,1); }
        else if(MODE==6){
          unsigned long long ps = __shfl_xor_sync(0xffffffffu,(unsigned long long)slot,1);
          unsigned long long* pslot=(unsigned long long*)ps;
          { unsigned long long* g=(lane&1)?pslot:slot; red64(g+2+(lane&1),(lane&1)?1ULL:val); }
          { unsigned long long* g=(lane&1)?slot:pslot; red64(g+2+((lane&1)^1),(lane&1)?val:1ULL); }
        } else acc+=(unsigned long long)slot;
      }
      else if(MODE==7){ acc+=atomicAdd(t0+key,val); acc+=atomicAdd(t1+key,1ULL); }
    }
  }
  if(MODE==0||MODE==7||MODE==8){ if(acc==0x1234567) sink[0]=acc; }
}

template<int MODE> float run(const int64_t*k,const int64_t*v,size_t n,unsigned long long*t0,unsigned long long*t1,size_t tbytes,uint64_t mask,unsigned long long*sink,int grid){
  cudaEvent_t a,b; CK(cudaEventCreate(&a)); CK(cudaEventCreate(&b));
  float best=1e9;
  for(int it=0;it<4;it++){
    if(!(MODE==5||MODE==6||MODE==8) || it==0) { CK(cudaMemset(t0,0,tbytes)); CK(cudaMemset(t1,0,tbytes)); }
    CK(cudaEventRecord(a)); agg<MODE><<<grid,256>>>(k,v,n,t0,t1,mask,sink); CK(cudaEventRecord(b)); CK(cudaEventSynchronize(b)); CK(cudaGetLastError());
    float ms; CK(cudaEventElapsedTime(&ms,a,b)); if(it>0 && ms<best)best=ms;
  }
  return best;
}
int main(int argc,char**argv){
  size_t n = (argc>1)? strtoull(argv[1],0,10) : (size_t)256<<20;
  uint64_t card = (argc>2)? strtoull(argv[2],0,10) : (1u<<20);
  int64_t *k,*v; CK(cudaMalloc(&k,n*8)); CK(cudaMalloc(&v,n*8));
  size_t slots = 1; while(slots < card*2) slots<<=1;          // load <= 0.5
  size_t tbytes = slots*32; unsigned long long *t0,*t1,*sink; CK(cudaMalloc(&t0,tbytes)); CK(cudaMalloc(&t1,tbytes)); CK(cudaMalloc(&sink,8));
  gen<<<132*8,256>>>(k,v,n,card); CK(cudaDeviceSynchronize());
  const char* names[]={"stream-only","SoA 2xRED","AoS16 2xRED","AoS16 1xRED","AoS16 paired","slot32 probe+2RED","slot32 probe+paired","SoA 2xATOM(ret)","slot32 probe only"};
  for(int gm=4; gm<=16; gm*=2){
    int grid=132*gm;
    float ms[9];
    ms[0]=run<0>(k,v,n,t0,t1,tbytes,slots-1,sink,grid); ms[1]=run<1>(k,v,n,t0,t1,tbytes,slots-1,sink,grid);
    ms[2]=run<2>(k,v,n,t0,t1,tbytes,slots-1,sink,grid); ms[3]=run<3>(k,v,n,t0,t1,tbytes,slots-1,sink,grid);
    ms[4]=run<4>(k,v,n,t0,t1,tbytes,slots-1,sink,grid); ms[5]=run<5>(k,v,n,t0,t1,tbytes,slots-1,sink,grid);
    ms[6]=run<6>(k,v,n,t0,t1,tbytes,slots-1,sink,grid); ms[7]=run<7>(k,v,n,t0,t1,tbytes,slots-1,sink,grid);
    ms[8]=run<8>(k,v,n,t0,t1,tbytes,slots-1,sink,grid);
    for(int m=0;m<9;m++) printf("grid=%d x256  %-22s n=%zu card=%llu  %.3f ms  %.3e rows/s  %.1f GB/s(16B/row)\n",grid,names[m],n,(unsigned long long)card,ms[m],n/(ms[m]*1e-3),16.0*n/(ms[m]*1e-3)/1e9);
  }
  return 0;
}
