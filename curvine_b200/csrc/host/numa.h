// Placement next to a GPU: the NUMA node a CUDA device hangs off, the CPUs of a node, and pinning a thread to them.  Used by the
// device reader (fetch threads, pinned ring), the worker's mem arena (first touch) and the synthetic-file writer (shard blocks).
// Plain types only, so worker-side code includes it without CUDA.
#pragma once
#include <vector>

namespace cv {

// NUMA node of the PCIe root `device` hangs off, from sysfs; -1 when unknown.
int gpu_numa_node(int device);

// CPUs of NUMA node `node` (its cpulist: ids and a-b ranges, in order); empty when node < 0 or the list cannot be read.
std::vector<int> node_cpus(int node);

// Pin the calling thread to `cpus` (no-op when empty).
void bind_cpus(const std::vector<int>& cpus);

}  // namespace cv
