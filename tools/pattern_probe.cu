// Access-pattern probe: how much HBM copy bandwidth does a persistent one-CTA-per-SM x 1024-thread kernel get when
//   A  the whole grid streams through memory together (grid-stride, 4 rows per thread in flight)
//   B  every WARP walks a private contiguous region (4736 concurrent read streams + 4736 write streams), tiles of 4 rows
//   C  every CTA walks a private contiguous region, its 32 warps taking adjacent 512-byte rows (one stream per SM)
//   D  like B with 64 KiB segments handed out round-robin inside a CTA's range (the layout of walk_kernel)
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o tools/pattern_probe tools/pattern_probe.cu
#include <cuda_runtime.h>
#include <cstdio>
#include <cstdlib>
#include <algorithm>
#include <vector>
#define CK(x) do{cudaError_t e_=(x); if(e_!=cudaSuccess){printf("CUDA error %s at line %d\n", cudaGetErrorString(e_), __LINE__); exit(1);} }while(0)

__host__ __device__ __forceinline__ size_t mn(size_t a, size_t b){ return a<b?a:b; }
__device__ __forceinline__ uint4 ldv(const uint4* p){ uint4 r; asm volatile("ld.global.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x),"=r"(r.y),"=r"(r.z),"=r"(r.w) : "l"(p)); return r; }

template<int T> __global__ void __launch_bounds__(1024,1) kA(const uint4* __restrict__ s, uint4* __restrict__ d, size_t nvec){
  const size_t stride = (size_t)gridDim.x * blockDim.x; size_t i = (size_t)blockIdx.x*blockDim.x + threadIdx.x;
  for(; i + (T-1)*stride < nvec; i += T*stride){ uint4 v[T];
#pragma unroll
    for(int k=0;k<T;k++) v[k]=ldv(s+i+k*stride);
#pragma unroll
    for(int k=0;k<T;k++) d[i+k*stride]=v[k]; }
  for(; i<nvec; i+=stride) d[i]=ldv(s+i);
}
// rows = 512-byte rows; warp-private contiguous region
template<int T> __global__ void __launch_bounds__(1024,1) kB(const uint4* __restrict__ s, uint4* __restrict__ d, size_t nrows){
  const unsigned lane=threadIdx.x&31; const size_t gw=(size_t)blockIdx.x*32+(threadIdx.x>>5), nw=(size_t)gridDim.x*32;
  const size_t per=(nrows+nw-1)/nw, r0=mn(nrows,gw*per), r1=mn(nrows,r0+per);
  size_t r=r0; for(; r+T<=r1; r+=T){ uint4 v[T];
#pragma unroll
    for(int k=0;k<T;k++) v[k]=ldv(s+(r+k)*32+lane);
#pragma unroll
    for(int k=0;k<T;k++) d[(r+k)*32+lane]=v[k]; }
  for(; r<r1; r++) d[r*32+lane]=ldv(s+r*32+lane);
}
// CTA-private contiguous region; warp w takes row step*32*T + k*32 + w
template<int T> __global__ void __launch_bounds__(1024,1) kC(const uint4* __restrict__ s, uint4* __restrict__ d, size_t nrows){
  const unsigned lane=threadIdx.x&31, w=threadIdx.x>>5; const size_t per=(nrows+gridDim.x-1)/gridDim.x, r0=mn(nrows,(size_t)blockIdx.x*per), r1=mn(nrows,r0+per);
  size_t r=r0; for(; r+32*T<=r1; r+=32*T){ uint4 v[T];
#pragma unroll
    for(int k=0;k<T;k++) v[k]=ldv(s+(r+k*32+w)*32+lane);
#pragma unroll
    for(int k=0;k<T;k++) d[(r+k*32+w)*32+lane]=v[k]; }
  for(r+=w; r<r1; r+=32) d[r*32+lane]=ldv(s+r*32+lane);
}
// walk_kernel layout: CTA range contiguous, units of SEGR rows round-robin over the 32 warps
template<int T> __global__ void __launch_bounds__(1024,1) kD(const uint4* __restrict__ s, uint4* __restrict__ d, size_t nrows, unsigned segr){
  const unsigned lane=threadIdx.x&31, w=threadIdx.x>>5; const size_t units=(nrows+segr-1)/segr, per=(units+gridDim.x-1)/gridDim.x, u0=mn(units,(size_t)blockIdx.x*per), u1=mn(units,u0+per);
  for(size_t u=u0+w; u<u1; u+=32){ size_t r=u*segr, r1=mn(nrows,r+segr);
    for(; r+T<=r1; r+=T){ uint4 v[T];
#pragma unroll
      for(int k=0;k<T;k++) v[k]=ldv(s+(r+k)*32+lane);
#pragma unroll
      for(int k=0;k<T;k++) d[(r+k)*32+lane]=v[k]; }
    for(; r<r1; r++) d[r*32+lane]=ldv(s+r*32+lane); }
}
// read-only variants (sum to defeat DCE) of B and C: is the locality effect a read or a write effect?
template<int T> __global__ void __launch_bounds__(1024,1) kBr(const uint4* __restrict__ s, unsigned* out, size_t nrows){
  const unsigned lane=threadIdx.x&31; const size_t gw=(size_t)blockIdx.x*32+(threadIdx.x>>5), nw=(size_t)gridDim.x*32;
  const size_t per=(nrows+nw-1)/nw, r0=mn(nrows,gw*per), r1=mn(nrows,r0+per); unsigned acc=0;
  size_t r=r0; for(; r+T<=r1; r+=T){ uint4 v[T];
#pragma unroll
    for(int k=0;k<T;k++) v[k]=ldv(s+(r+k)*32+lane);
#pragma unroll
    for(int k=0;k<T;k++) acc^=v[k].x^v[k].y^v[k].z^v[k].w; }
  if(acc==0x12345678u) out[0]=acc;
}
template<int T> __global__ void __launch_bounds__(1024,1) kBw(uint4* __restrict__ d, size_t nrows){
  const unsigned lane=threadIdx.x&31; const size_t gw=(size_t)blockIdx.x*32+(threadIdx.x>>5), nw=(size_t)gridDim.x*32;
  const size_t per=(nrows+nw-1)/nw, r0=mn(nrows,gw*per), r1=mn(nrows,r0+per); const uint4 v=make_uint4(lane,1,2,3);
  for(size_t r=r0; r<r1; r++) d[r*32+lane]=v;
}
template<int T> __global__ void __launch_bounds__(1024,1) kCw(uint4* __restrict__ d, size_t nrows){
  const unsigned lane=threadIdx.x&31, w=threadIdx.x>>5; const size_t per=(nrows+gridDim.x-1)/gridDim.x, r0=mn(nrows,(size_t)blockIdx.x*per), r1=mn(nrows,r0+per); const uint4 v=make_uint4(lane,1,2,3);
  for(size_t r=r0+w; r<r1; r+=32) d[r*32+lane]=v;
}

template<typename F> static void timeit(const char* name, double bytes, F launch){
  for(int i=0;i<20;i++) launch(); CK(cudaDeviceSynchronize());
  std::vector<float> ts; cudaEvent_t a,b; CK(cudaEventCreate(&a)); CK(cudaEventCreate(&b));
  for(int i=0;i<20;i++){ CK(cudaEventRecord(a)); launch(); CK(cudaEventRecord(b)); CK(cudaEventSynchronize(b)); float ms; CK(cudaEventElapsedTime(&ms,a,b)); ts.push_back(ms);} 
  std::sort(ts.begin(),ts.end()); printf("%-52s best %7.1f GB/s  median %7.1f GB/s\n", name, bytes/ts[0]/1e6, bytes/ts[10]/1e6); CK(cudaGetLastError());
}
int main(int argc,char**argv){
  const size_t bytes = (argc>1? atof(argv[1]) : 4.0) * (1ull<<30); const size_t nvec=bytes/16, nrows=bytes/512;
  uint4 *s,*d; CK(cudaMalloc(&s,bytes)); CK(cudaMalloc(&d,bytes)); CK(cudaMemset(s,1,bytes)); CK(cudaMemset(d,2,bytes)); unsigned* out; CK(cudaMalloc(&out,4));
  int sm=0; CK(cudaDeviceGetAttribute(&sm,cudaDevAttrMultiProcessorCount,0));
  timeit("cudaMemcpy D2D", 2.0*bytes, [&]{ cudaMemcpyAsync(d,s,bytes,cudaMemcpyDeviceToDevice); });
  timeit("A grid-stride T=4", 2.0*bytes, [&]{ kA<4><<<sm,1024>>>(s,d,nvec); });
  timeit("A grid-stride T=2", 2.0*bytes, [&]{ kA<2><<<sm,1024>>>(s,d,nvec); });
  timeit("B warp-private regions T=4", 2.0*bytes, [&]{ kB<4><<<sm,1024>>>(s,d,nrows); });
  timeit("B warp-private regions T=2", 2.0*bytes, [&]{ kB<2><<<sm,1024>>>(s,d,nrows); });
  timeit("C CTA-private regions, warps on adjacent rows T=4", 2.0*bytes, [&]{ kC<4><<<sm,1024>>>(s,d,nrows); });
  timeit("C CTA-private regions, warps on adjacent rows T=2", 2.0*bytes, [&]{ kC<2><<<sm,1024>>>(s,d,nrows); });
  for(unsigned segr : {8u, 32u, 128u, 512u, 2048u}){ char nm[96]; snprintf(nm,96,"D round-robin %u KiB segments T=4", segr/2); timeit(nm, 2.0*bytes, [&]{ kD<4><<<sm,1024>>>(s,d,nrows,segr); }); }
  timeit("B read-only warp-private T=4", 1.0*bytes, [&]{ kBr<4><<<sm,1024>>>(s,out,nrows); });
  timeit("B write-only warp-private", 1.0*bytes, [&]{ kBw<1><<<sm,1024>>>(d,nrows); });
  timeit("C write-only CTA-private adjacent rows", 1.0*bytes, [&]{ kCw<1><<<sm,1024>>>(d,nrows); });
  return 0;
}
