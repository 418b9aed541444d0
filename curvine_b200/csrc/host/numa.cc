#include "numa.h"

#include <cuda_runtime.h>
#include <ctype.h>
#include <sched.h>
#include <stdlib.h>

#include <fstream>
#include <string>

namespace cv {

int gpu_numa_node(int device) {
    char bus[64] = {0};
    if (cudaDeviceGetPCIBusId(bus, sizeof(bus), device) != cudaSuccess) {
        cudaGetLastError();  // an unknown node is not an error: leave nothing for the next CUDA call to report
        return -1;
    }
    for (char* p = bus; *p; p++) *p = static_cast<char>(tolower(*p));
    int node = -1;
    std::ifstream f(std::string("/sys/bus/pci/devices/") + bus + "/numa_node");
    if (f) f >> node;
    return node;
}

std::vector<int> node_cpus(int node) {
    std::vector<int> cpus;
    if (node < 0) return cpus;
    std::ifstream f("/sys/devices/system/node/node" + std::to_string(node) + "/cpulist");
    std::string line;
    if (!f || !std::getline(f, line)) return cpus;
    for (const char* p = line.c_str();;) {
        char* e = nullptr;
        const long a = strtol(p, &e, 10);
        if (e == p) break;
        long b = a;
        if (*e == '-') b = strtol(e + 1, &e, 10);
        for (long x = a; x <= b; x++) cpus.push_back(static_cast<int>(x));
        if (*e != ',') break;
        p = e + 1;
    }
    return cpus;
}

void bind_cpus(const std::vector<int>& cpus) {
    if (cpus.empty()) return;
    cpu_set_t set;
    CPU_ZERO(&set);
    for (int c : cpus) CPU_SET(c, &set);
    sched_setaffinity(0, sizeof(set), &set);
}

}  // namespace cv
