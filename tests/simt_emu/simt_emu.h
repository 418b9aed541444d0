// TEST INFRASTRUCTURE ONLY -- a SIMT execution shim that lets g++ compile csrc/kernels.cu (the product's kernel source, unmodified
// apart from the mechanical launch/asm rewrite of tests/simt_emu/build.py) and run its __global__ functions on host cores, so the
// kernels' ALGORITHM is checked against the oracle by the CPU suite too (the GPU suite checks the compiled sm_90a code on an H100).
//
// Execution model: one fiber per CUDA thread, one thread block at a time per host worker thread, blocks of a grid spread over the
// workers.  A fiber runs until it reaches a collective (__syncthreads, __syncwarp, a *_sync warp intrinsic) or returns; collectives
// complete when every live (not yet returned) participant has arrived, exactly the rule the hardware applies.  Code that is
// correctly synchronised computes what it computes on the GPU; a missing barrier shows up as a wrong result or as the deadlock
// report of the scheduler, not as a timing-dependent flake.  Nothing here is timed, shipped or reachable from curvine_b200/.
#pragma once
#include <stddef.h>
#include <stdint.h>
#include <string.h>

#include <tuple>
#include <type_traits>
#include <utility>

#define CVK_SIMT_EMU 1
#define __global__
#define __device__
#define __host__
#define __forceinline__ inline __attribute__((always_inline))
#define __launch_bounds__(...)
#define __align__(n) alignas(n)
#define __shared__ static thread_local  // one block at a time per host thread: per-thread statics are per-block storage

struct uint3 {
    unsigned x, y, z;
};
struct dim3 {
    unsigned x, y, z;
    dim3(unsigned x_ = 1, unsigned y_ = 1, unsigned z_ = 1) : x(x_), y(y_), z(z_) {}
};
struct alignas(16) uint4 {
    uint32_t x, y, z, w;
};
static inline uint4 make_uint4(uint32_t x, uint32_t y, uint32_t z, uint32_t w) { return uint4{x, y, z, w}; }

namespace cv_emu {

struct ThreadCtx {
    uint3 tid, bid;
    dim3 bdim, gdim;
};
// the calling fiber's indices; `const`: a fiber only ever sees its own context, so the compiler may keep the pointer
const ThreadCtx* cur() __attribute__((const));
char* dyn_smem() __attribute__((const));  // this host thread's dynamic shared memory (227 KB)

void sync_block();
void sync_warp(uint32_t mask);
// every participating lane deposits v; returns the value lane `src` deposited (its own when src does not take part)
uint64_t warp_exchange(uint32_t mask, uint64_t v, uint32_t src);
uint32_t warp_ballot(uint32_t mask, bool pred);

typedef void (*Thunk)(void* kernel, void* args);
// runs the grid in stream order (at once on the NULL stream and in the runtime stand-in's default synchronous mode), then frees args
void launch(void* stream, dim3 grid, dim3 block, size_t smem_bytes, Thunk thunk, void* kernel, void* args, void (*free_args)(void*));

struct LaunchCfg {
    dim3 g, b;
    size_t smem;
    void* stream;
    template <class... P, class... A>
    void operator()(void (*k)(P...), A&&... a) const {
        typedef std::tuple<std::decay_t<P>...> Args;
        Args* args = new Args(static_cast<std::decay_t<P>>(std::forward<A>(a))...);  // by value, like a launch's parameter buffer
        struct T {
            static void run(void* kernel, void* t) { std::apply(reinterpret_cast<void (*)(P...)>(kernel), *static_cast<Args*>(t)); }
            static void drop(void* t) { delete static_cast<Args*>(t); }
        };
        launch(stream, g, b, smem, &T::run, reinterpret_cast<void*>(k), args, &T::drop);
    }
};
template <class S>
inline LaunchCfg cfg(dim3 g, dim3 b, size_t smem, S stream) {
    return LaunchCfg{g, b, smem, (void*)stream};
}

// ---- the PTX the kernels use (build.py turns every asm statement into one of these)
//
// 16-byte vector LOADS follow the rule the kernels rely on: a source range is read in whole 16-byte ALIGNED granules, so up to 15
// bytes in front of / behind the range are read too -- never outside the granules that hold the range (hence never across a page
// or an allocation granule).  Under AddressSanitizer that rule is what is checked: a granule with at least one addressable byte
// is fine, a granule that lies entirely outside every allocation is reported.  Stores get no such slack.
#if defined(__SANITIZE_ADDRESS__)
extern "C" int __asan_address_is_poisoned(void const volatile* addr);
void asan_report_load16(const void* p);  // an ordinary instrumented 16-byte read: produces the standard report
__attribute__((no_sanitize("address"))) inline void granule_load(uint32_t v[4], const void* p) {
    bool any = false;
    for (int i = 0; i < 16; i++) any |= !__asan_address_is_poisoned(static_cast<const char*>(p) + i);
    if (!any) asan_report_load16(p);
    typedef uint32_t __attribute__((may_alias)) word;
    const word* q = static_cast<const word*>(__builtin_assume_aligned(p, 16));
    v[0] = q[0], v[1] = q[1], v[2] = q[2], v[3] = q[3];
}
#else
inline void granule_load(uint32_t v[4], const void* p) { memcpy(v, __builtin_assume_aligned(p, 16), 16); }
#endif
inline void ptx_ld_v4(uint32_t& a, uint32_t& b, uint32_t& c, uint32_t& d, const void* p) {
    uint32_t v[4];
    granule_load(v, p);
    a = v[0], b = v[1], c = v[2], d = v[3];
}
inline void ptx_st_v4(void* p, uint32_t a, uint32_t b, uint32_t c, uint32_t d) {
    const uint32_t v[4] = {a, b, c, d};
    memcpy(__builtin_assume_aligned(p, 16), v, 16);
}
inline void ptx_lds_v4(uint32_t& a, uint32_t& b, uint32_t& c, uint32_t& d, uint32_t addr) { ptx_ld_v4(a, b, c, d, dyn_smem() + addr); }
inline void ptx_lds_u32(uint32_t& v, uint32_t addr) { memcpy(&v, dyn_smem() + addr, 4); }
inline void ptx_cp_async16(uint32_t smem_addr, const void* g) {  // lands at once
    uint32_t v[4];
    granule_load(v, g);
    memcpy(dyn_smem() + smem_addr, v, 16);
}
inline void ptx_cp_async_commit() {}
inline void ptx_cp_async_wait(int) {}

}  // namespace cv_emu

#define threadIdx (cv_emu::cur()->tid)
#define blockIdx (cv_emu::cur()->bid)
#define blockDim (cv_emu::cur()->bdim)
#define gridDim (cv_emu::cur()->gdim)

static inline void __syncthreads() { cv_emu::sync_block(); }
static inline void __syncwarp(uint32_t mask = 0xffffffffu) { cv_emu::sync_warp(mask); }
static inline uint32_t cv_emu_lane() { return threadIdx.x & 31u; }

template <class T>
static inline T __shfl_sync(uint32_t mask, T v, int src) {
    static_assert(sizeof(T) <= 8, "shuffle of at most 8 bytes");
    uint64_t raw = 0;
    memcpy(&raw, &v, sizeof(T));
    raw = cv_emu::warp_exchange(mask, raw, static_cast<uint32_t>(src) & 31u);
    T out;
    memcpy(&out, &raw, sizeof(T));
    return out;
}
template <class T>
static inline T __shfl_up_sync(uint32_t mask, T v, unsigned d) {
    const uint32_t lane = cv_emu_lane();
    return __shfl_sync(mask, v, lane >= d ? int(lane - d) : int(lane));
}
template <class T>
static inline T __shfl_down_sync(uint32_t mask, T v, unsigned d) {
    const uint32_t lane = cv_emu_lane();
    return __shfl_sync(mask, v, lane + d < 32 ? int(lane + d) : int(lane));
}
template <class T>
static inline T __shfl_xor_sync(uint32_t mask, T v, int x) {
    return __shfl_sync(mask, v, int(cv_emu_lane() ^ uint32_t(x)));
}
static inline uint32_t __ballot_sync(uint32_t mask, bool pred) { return cv_emu::warp_ballot(mask, pred); }
static inline int __popc(uint32_t v) { return __builtin_popcount(v); }

template <class T>
static inline T __ldg(const T* p) {
    return *p;
}
// funnel shift right: low 32 bits of (hi:lo) >> (s & 31)
static inline uint32_t __funnelshift_r(uint32_t lo, uint32_t hi, uint32_t s) {
    return static_cast<uint32_t>(((uint64_t(hi) << 32) | lo) >> (s & 31u));
}
// PRMT, default mode: result byte i = byte (sel nibble i & 7) of {y:x}; nibble bit 3 replicates that byte's sign bit
static inline uint32_t __byte_perm(uint32_t x, uint32_t y, uint32_t s) {
    const uint64_t src = (uint64_t(y) << 32) | x;
    uint32_t r = 0;
    for (int i = 0; i < 4; i++) {
        const uint32_t n = (s >> (4 * i)) & 0xfu;
        uint32_t b = static_cast<uint32_t>(src >> (8 * (n & 7u))) & 0xffu;
        if (n & 8u) b = (b & 0x80u) ? 0xffu : 0u;
        r |= b << (8 * i);
    }
    return r;
}
static inline size_t __cvta_generic_to_shared(const void* p) { return static_cast<size_t>(static_cast<const char*>(p) - cv_emu::dyn_smem()); }

template <class T, class V>
static inline T atomicAdd(T* p, V v) {
    return __atomic_fetch_add(p, static_cast<T>(v), __ATOMIC_RELAXED);
}
template <class T>
static inline T min(T a, T b) {
    return b < a ? b : a;
}
template <class T>
static inline T max(T a, T b) {
    return a < b ? b : a;
}
