// Round-2 box probe for the arena mem tier: what does it cost to pin one big tmpfs arena, and how fast does the copy
// engine read out of it?  (tools/ = measurement scaffolding, not product code.)
//   A  hugepage availability (hugetlb pool, THP for shmem, MFD_HUGETLB)
//   B  populate + cudaHostRegister of a tmpfs arena: one call vs parallel slices; registering an unpopulated mapping
//   C  H2D out of the registered arena: 4 / 32 MiB copies, contiguous and scattered; after mprotect(PROT_READ)
//   D  cudaHostRegisterReadOnly on a PROT_READ mapping (refused in round 1: check again)
#include <cuda_runtime.h>
#include <fcntl.h>
#include <sched.h>
#include <sys/mman.h>
#include <sys/stat.h>
#include <unistd.h>

#include <atomic>
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <functional>
#include <iostream>
#include <string>
#include <thread>
#include <vector>
#ifndef MFD_HUGETLB
#define MFD_HUGETLB 0x0004U
#endif
static double now() { return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count(); }
static std::vector<int> g_cpus;
static void bind_gpu_node() {
    if (g_cpus.empty()) return;
    cpu_set_t s;
    CPU_ZERO(&s);
    for (int c : g_cpus) CPU_SET(c, &s);
    sched_setaffinity(0, sizeof(s), &s);
}
static void cat(const char* p) {
    std::ifstream f(p);
    std::string l;
    printf("--- %s\n", p);
    while (std::getline(f, l)) printf("    %s\n", l.c_str());
}
static void par(int T, size_t n, const std::function<void(size_t, size_t)>& fn) {
    std::vector<std::thread> ts;
    for (int t = 0; t < T; t++) ts.emplace_back([&, t] {
        bind_gpu_node();
        cudaSetDevice(0);
        fn(n * t / T, n * (t + 1) / T);
    });
    for (auto& t : ts) t.join();
}
int main(int argc, char** argv) {
    const size_t GiB = 1ull << 30;
    const size_t N = (argc > 1 ? atoi(argv[1]) : 8) * GiB;
    setvbuf(stdout, nullptr, _IOLBF, 0);
    if (cudaSetDevice(0) != cudaSuccess) { printf("no device\n"); return 1; }
    {  // CPUs of the GPU's NUMA node
        char bus[64] = {0};
        int node = -1;
        cudaDeviceGetPCIBusId(bus, sizeof(bus), 0);
        for (char* p = bus; *p; p++) *p = tolower(*p);
        std::ifstream f(std::string("/sys/bus/pci/devices/") + bus + "/numa_node");
        if (f) f >> node;
        printf("gpu0 pci %s numa_node %d\n", bus, node);
        if (node >= 0) {
            std::ifstream c("/sys/devices/system/node/node" + std::to_string(node) + "/cpulist");
            std::string s;
            std::getline(c, s);
            printf("node cpulist %s\n", s.c_str());
            size_t p = 0;
            while (p < s.size()) {
                size_t c2 = s.find(',', p);
                std::string r = s.substr(p, c2 == std::string::npos ? std::string::npos : c2 - p);
                size_t d = r.find('-');
                int a = atoi(r.c_str()), b = d == std::string::npos ? a : atoi(r.c_str() + d + 1);
                for (int x = a; x <= b; x++) g_cpus.push_back(x);
                if (c2 == std::string::npos) break;
                p = c2 + 1;
            }
        }
    }
    // ---- A
    cat("/sys/kernel/mm/transparent_hugepage/enabled");
    cat("/sys/kernel/mm/transparent_hugepage/shmem_enabled");
    cat("/proc/sys/vm/nr_hugepages");
    cat("/proc/sys/vm/nr_overcommit_hugepages");
    {
        std::ifstream f("/proc/meminfo");
        std::string l;
        while (std::getline(f, l))
            if (l.find("Huge") != std::string::npos || l.find("Shmem") != std::string::npos) printf("    %s\n", l.c_str());
    }
    {
        // uses whatever hugetlb pool the host already has; the probe never changes host settings
        int mfd = memfd_create("hp", MFD_HUGETLB);
        if (mfd < 0) printf("A memfd_create(MFD_HUGETLB): %s\n", strerror(errno));
        else {
            int rc = ftruncate(mfd, GiB);
            void* p = rc == 0 ? mmap(nullptr, GiB, PROT_READ | PROT_WRITE, MAP_SHARED | MAP_POPULATE, mfd, 0) : MAP_FAILED;
            printf("A hugetlb memfd 1 GiB: ftruncate %d mmap %s\n", rc, p == MAP_FAILED ? strerror(errno) : "ok");
            if (p != MAP_FAILED) {
                double t0 = now();
                cudaError_t e = cudaHostRegister(p, GiB, cudaHostRegisterDefault);
                printf("A cudaHostRegister(hugetlb 1 GiB): %s %.1f ms\n", cudaGetErrorString(e), (now() - t0) * 1e3);
                if (e == cudaSuccess) cudaHostUnregister(p);
                munmap(p, GiB);
            }
            close(mfd);
        }
    }
    // ---- B
    uint8_t* dv;
    if (cudaMalloc(&dv, N) != cudaSuccess) { printf("cudaMalloc failed\n"); return 1; }
    auto make = [&](const char* path, bool populate, int T) -> uint8_t* {
        unlink(path);
        int fd = open(path, O_RDWR | O_CREAT, 0644);
        if (ftruncate(fd, N) != 0) { printf("ftruncate: %s\n", strerror(errno)); exit(1); }
        uint8_t* m = (uint8_t*)mmap(nullptr, N, PROT_READ | PROT_WRITE, MAP_SHARED, fd, 0);
        close(fd);
        if (m == MAP_FAILED) { printf("mmap: %s\n", strerror(errno)); exit(1); }
        if (populate) {
            double t0 = now();
            par(T, N, [&](size_t a, size_t b) { for (size_t o = a; o < b; o += 4096) m[o] = (uint8_t)(o >> 12); });
            printf("B populate %zu GiB tmpfs with %d threads: %.2f s (%.1f GB/s)\n", N / GiB, T, now() - t0, N / (now() - t0) / 1e9);
        }
        return m;
    };
    {
        uint8_t* m = make("/dev/shm/arena_probe_a", true, 32);
        double t0 = now();
        cudaError_t e = cudaHostRegister(m, N, cudaHostRegisterDefault);
        printf("B register populated arena, ONE call: %s %.2f s (%.1f GB/s)\n", cudaGetErrorString(e), now() - t0, N / (now() - t0) / 1e9);
        if (e == cudaSuccess) {
            t0 = now();
            cudaHostUnregister(m);
            printf("B unregister: %.2f s\n", now() - t0);
        }
        for (int T : {4, 16, 32}) {
            const size_t S = 256 << 20;  // slice
            std::atomic<size_t> nx{0};
            std::atomic<int> bad{0};
            t0 = now();
            par(T, 1, [&](size_t, size_t) {
                for (;;) {
                    size_t o = nx.fetch_add(S);
                    if (o >= N) break;
                    if (cudaHostRegister(m + o, std::min(S, N - o), cudaHostRegisterDefault) != cudaSuccess) bad++;
                }
            });
            printf("B register populated arena, 256 MiB slices, %2d threads: bad=%d %.2f s (%.1f GB/s)\n", T, bad.load(), now() - t0, N / (now() - t0) / 1e9);
            if (T != 32)
                for (size_t o = 0; o < N; o += S) cudaHostUnregister(m + o);
        }
        // ---- C (registered in 256 MiB slices by the last pass)
        cudaStream_t s;
        cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking);
        auto copy = [&](const char* name, size_t cs, bool scatter) {
            cudaEvent_t a, b;
            cudaEventCreate(&a), cudaEventCreate(&b);
            const size_t nc = N / cs;
            double t0 = now();
            cudaEventRecord(a, s);
            for (size_t i = 0; i < nc; i++) {
                size_t j = scatter ? (i * 2654435761ull) % nc : i;
                if (cudaMemcpyAsync(dv + i * cs, m + j * cs, cs, cudaMemcpyHostToDevice, s) != cudaSuccess) { printf("memcpy failed\n"); break; }
            }
            cudaEventRecord(b, s);
            cudaEventSynchronize(b);
            float ms;
            cudaEventElapsedTime(&ms, a, b);
            printf("C H2D from arena %-28s copy=%3zu MiB: %6.2f GB/s (enqueue+run wall %.3f s)\n", name, cs >> 20, N / ms / 1e6, now() - t0);
        };
        for (int rep = 0; rep < 2; rep++) copy("contiguous", 32 << 20, false);
        copy("contiguous", 4 << 20, false);
        copy("scattered", 4 << 20, true);
        copy("scattered", 32 << 20, true);
        copy("contiguous (crosses slices)", 512 << 20, false);
        int rc = mprotect(m, N, PROT_READ);
        printf("C mprotect(PROT_READ) after registration: %d %s\n", rc, rc ? strerror(errno) : "ok");
        copy("after mprotect(PROT_READ)", 32 << 20, false);
        // content check
        std::vector<uint8_t> h(4096 * 4);
        cudaMemcpy(h.data(), dv + (N / 2), h.size(), cudaMemcpyDeviceToHost);
        printf("C content check: %s\n", h[0] == (uint8_t)((N / 2) >> 12) && h[4096] == (uint8_t)((N / 2 + 4096) >> 12) ? "ok" : "MISMATCH");
        for (size_t o = 0; o < N; o += (256 << 20)) cudaHostUnregister(m + o);
        munmap(m, N);
        unlink("/dev/shm/arena_probe_a");
    }
    {
        uint8_t* m = make("/dev/shm/arena_probe_b", false, 0);
        const size_t S = 256 << 20;
        std::atomic<size_t> nx{0};
        std::atomic<int> bad{0};
        double t0 = now();
        par(16, 1, [&](size_t, size_t) {
            for (;;) {
                size_t o = nx.fetch_add(S);
                if (o >= N) break;
                if (cudaHostRegister(m + o, std::min(S, N - o), cudaHostRegisterDefault) != cudaSuccess) bad++;
            }
        });
        printf("B register UNPOPULATED (sparse) arena, 256 MiB slices, 16 threads: bad=%d %.2f s (%.1f GB/s)\n", bad.load(), now() - t0, N / (now() - t0) / 1e9);
        // pwrite through a second fd lands in the same pages?
        int fd = open("/dev/shm/arena_probe_b", O_RDWR);
        std::vector<uint8_t> blk(1 << 20, 0xAB);
        if (pwrite(fd, blk.data(), blk.size(), 5 << 20) != (ssize_t)blk.size()) printf("pwrite failed\n");
        close(fd);
        std::vector<uint8_t> h(16);
        cudaMemcpy(dv, m + (5 << 20), 1 << 20, cudaMemcpyHostToDevice);
        cudaMemcpy(h.data(), dv, 16, cudaMemcpyDeviceToHost);
        printf("B pwrite-after-register visible to DMA: %s\n", h[0] == 0xAB && h[15] == 0xAB ? "yes" : "NO");
        for (size_t o = 0; o < N; o += S) cudaHostUnregister(m + o);
        munmap(m, N);
        // ---- D
        fd = open("/dev/shm/arena_probe_b", O_RDONLY);
        void* r = mmap(nullptr, GiB, PROT_READ, MAP_SHARED, fd, 0);
        close(fd);
        cudaError_t e = cudaHostRegister(r, GiB, cudaHostRegisterReadOnly);
        printf("D cudaHostRegisterReadOnly on PROT_READ mapping: %s\n", cudaGetErrorString(e));
        cudaGetLastError();
        if (e == cudaSuccess) cudaHostUnregister(r);
        e = cudaHostRegister(r, GiB, cudaHostRegisterDefault);
        printf("D cudaHostRegisterDefault on PROT_READ mapping: %s\n", cudaGetErrorString(e));
        cudaGetLastError();
        if (e == cudaSuccess) cudaHostUnregister(r);
        munmap(r, GiB);
        unlink("/dev/shm/arena_probe_b");
    }
    return 0;
}
