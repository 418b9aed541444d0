// TEST INFRASTRUCTURE ONLY (see cuda_runtime.h in this directory): the runtime calls of the kernel launchers that the
// host-memory stand-in of tests/mock_cuda does not have.
#include <stdlib.h>

#include "cuda_runtime.h"

extern "C" {
cudaError_t cudaDeviceGetAttribute(int* value, enum cudaDeviceAttr attr, int) {
    if (attr != cudaDevAttrMultiProcessorCount) return cudaErrorInvalidValue;
    const char* e = getenv("CV_SIMT_EMU_SMS");  // persistent kernels launch one CTA per SM: 132 on the H100 SXM
    *value = e ? atoi(e) : 132;
    return cudaSuccess;
}
cudaError_t cudaMemPoolCreate(cudaMemPool_t* pool, const struct cudaMemPoolProps*) {
    *pool = reinterpret_cast<cudaMemPool_t>(malloc(1));
    return cudaSuccess;
}
cudaError_t cudaMemPoolSetAttribute(cudaMemPool_t, enum cudaMemPoolAttr, void*) { return cudaSuccess; }
cudaError_t cudaMallocFromPoolAsync(void** p, size_t n, cudaMemPool_t, cudaStream_t st) { return mock_cudaMallocAsync(p, n, st); }
cudaError_t cudaEventCreate(cudaEvent_t* ev) { return cudaEventCreateWithFlags(ev, 0); }
cudaError_t cudaEventElapsedTime(float* ms, cudaEvent_t, cudaEvent_t) {
    *ms = 1.0f;  // nothing is timed here; callers only need a positive number
    return cudaSuccess;
}
cudaError_t cudaDeviceEnablePeerAccess(int peer, unsigned) { return peer >= 0 && peer < 8 ? cudaSuccess : cudaErrorInvalidDevice; }
}
