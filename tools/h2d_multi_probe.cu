// Concurrent pinned-H2D ceiling of this box: how much host->device bandwidth does each GPU get when 1, 2, 4, 8 GPUs copy
// at the same time?  The N>1 bench lands at ~51 GB/s per GPU against 55 GB/s alone; this separates "the platform gives a pair
// of GPUs behind one PCIe switch less than 2 x the solo rate" from "our pipeline loses something when it is not alone".
//   per GPU: one thread bound to the GPU's NUMA node, 4 pinned buffers of 32 MiB allocated from that thread, one stream,
//   cudaMemcpyAsync round-robin for ~1.5 s, CUDA events for the device-side time.
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o tools/h2d_multi_probe tools/h2d_multi_probe.cu
// Run:   tools/h2d_multi_probe            (sweeps the first 1, 2, 4, 8 devices and prints per-GPU GB/s)
#include <cuda_runtime.h>
#include <sched.h>
#include <unistd.h>
#include <atomic>
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <string>
#include <thread>
#include <vector>
#define CK(x) do{cudaError_t e_=(x); if(e_!=cudaSuccess){printf("CUDA error %s at line %d\n", cudaGetErrorString(e_), __LINE__); exit(1);} }while(0)
static double now(){ return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count(); }

static int numa_node_of(int dev){
  char bus[64]={0}; if(cudaDeviceGetPCIBusId(bus,sizeof(bus),dev)!=cudaSuccess) return -1;
  for(char*p=bus;*p;p++) *p=(char)tolower(*p);
  std::ifstream f(std::string("/sys/bus/pci/devices/")+bus+"/numa_node"); int n=-1; if(f) f>>n; return n;
}
static void bind_node(int node){
  if(node<0) return; std::ifstream f("/sys/devices/system/node/node"+std::to_string(node)+"/cpulist"); std::string s; if(!f||!std::getline(f,s)) return;
  cpu_set_t set; CPU_ZERO(&set); size_t p=0;
  while(p<s.size()){ size_t c=s.find(',',p); std::string r=s.substr(p,c==std::string::npos?std::string::npos:c-p); size_t d=r.find('-');
    int a=atoi(r.c_str()), b=d==std::string::npos?a:atoi(r.c_str()+d+1); for(int x=a;x<=b;x++) CPU_SET(x,&set); if(c==std::string::npos) break; p=c+1; }
  sched_setaffinity(0,sizeof(set),&set);
}

int main(int argc,char**argv){
  int ndev=0; CK(cudaGetDeviceCount(&ndev)); const size_t CH=32u<<20; const int NB=4; const double secs = argc>1? atof(argv[1]) : 1.5;
  printf("devices=%d\n", ndev);
  for(int d=0; d<ndev; d++){ char bus[64]={0}; cudaDeviceGetPCIBusId(bus,sizeof(bus),d); printf("dev%d pci=%s numa_node=%d\n", d, bus, numa_node_of(d)); }
  for(int G : {1,2,4,8}){ if(G>ndev) break;
    for(int first=0; first+G<=ndev && first<= (G==1? ndev-1 : 0); first+= (G==1? 1 : ndev)){   // G==1: every device alone
      std::vector<double> gbps(G,0.0); std::atomic<int> ready{0}; std::atomic<bool> go{false}; std::vector<std::thread> ts;
      for(int g=0; g<G; g++) ts.emplace_back([&,g]{ const int dev=first+g; bind_node(numa_node_of(dev)); CK(cudaSetDevice(dev));
        uint8_t* h[NB]; uint8_t* dv; for(int i=0;i<NB;i++){ CK(cudaHostAlloc(&h[i],CH,cudaHostAllocDefault)); memset(h[i],i+1,CH);} CK(cudaMalloc(&dv,CH*NB));
        cudaStream_t st; CK(cudaStreamCreateWithFlags(&st,cudaStreamNonBlocking)); cudaEvent_t a,b; CK(cudaEventCreate(&a)); CK(cudaEventCreate(&b));
        for(int i=0;i<8;i++) CK(cudaMemcpyAsync(dv+(i%NB)*CH,h[i%NB],CH,cudaMemcpyHostToDevice,st)); CK(cudaStreamSynchronize(st));
        ready++; while(!go.load()) sched_yield();
        const double t0=now(); size_t n=0; CK(cudaEventRecord(a,st));
        while(now()-t0<secs){ for(int i=0;i<16;i++){ CK(cudaMemcpyAsync(dv+(n%NB)*CH,h[n%NB],CH,cudaMemcpyHostToDevice,st)); n++; } CK(cudaStreamSynchronize(st)); }
        CK(cudaEventRecord(b,st)); CK(cudaEventSynchronize(b)); float ms; CK(cudaEventElapsedTime(&ms,a,b)); gbps[g]=(double)n*CH/ms/1e6;
        for(int i=0;i<NB;i++) cudaFreeHost(h[i]); cudaFree(dv); });
      while(ready.load()<G) usleep(1000); go=true; for(auto&t:ts) t.join();
      double tot=0; printf("G=%d first=%d :", G, first); for(int g=0; g<G; g++){ printf(" %.1f", gbps[g]); tot+=gbps[g]; } printf("  | total %.1f GB/s, per GPU %.1f\n", tot, tot/G);
    }
  }
  return 0;
}
