// TEST INFRASTRUCTURE ONLY (see simt_emu.h): the fiber scheduler behind the SIMT shim.
#include "simt_emu.h"

#include <stdio.h>
#include <stdlib.h>
#include <sys/mman.h>

#include <atomic>
#include <condition_variable>
#include <mutex>
#include <thread>
#include <vector>

#if !defined(__x86_64__)
#error "the fiber switch below is written for x86-64 (the build container and the GPU boxes)"
#endif

// void cv_emu_switch(void** save_sp, void* load_sp): callee-saved registers on the old stack, swap stacks, pop, return
extern "C" void cv_emu_switch(void** save_sp, void* load_sp);
extern "C" void mock_cuda_set_last_error(int e);  // tests/mock_cuda/mock_cuda.cc
extern "C" void mock_cuda_enqueue(void* stream, void (*fn)(void*), void* arg);  // runs fn(arg) in stream order
asm(R"(
.text
.globl cv_emu_switch
.type cv_emu_switch,@function
cv_emu_switch:
    pushq %rbp
    pushq %rbx
    pushq %r12
    pushq %r13
    pushq %r14
    pushq %r15
    movq %rsp, (%rdi)
    movq %rsi, %rsp
    popq %r15
    popq %r14
    popq %r13
    popq %r12
    popq %rbx
    popq %rbp
    ret
.size cv_emu_switch,.-cv_emu_switch
)");

// AddressSanitizer has to be told about every stack switch (it tracks the bounds of the running stack)
#if defined(__SANITIZE_ADDRESS__)
#include <sanitizer/common_interface_defs.h>
#define CV_ASAN_START(save, bottom, size) __sanitizer_start_switch_fiber(save, bottom, size)
#define CV_ASAN_FINISH(save, bottom_old, size_old) __sanitizer_finish_switch_fiber(save, bottom_old, size_old)
#else
#define CV_ASAN_START(save, bottom, size) ((void)0)
#define CV_ASAN_FINISH(save, bottom_old, size_old) ((void)0)
#endif

// ThreadSanitizer build (build.py "thread": this file itself stays uninstrumented, the kernel source is instrumented): every CUDA
// thread is a TSan fiber, switches establish NO ordering, and the only happens-before edges are the ones the programming model
// gives -- block start/end, __syncthreads, warp collectives, atomics.  Two threads of a block (or two blocks) that touch the same
// shared or global location without one of those in between are reported as a data race: a race check of the kernel source.
#if defined(CV_EMU_TSAN)
extern "C" {
void* __tsan_get_current_fiber(void);
void* __tsan_create_fiber(unsigned flags);
void __tsan_switch_to_fiber(void* fiber, unsigned flags);
void __tsan_set_fiber_name(void* fiber, const char* name);
void __tsan_acquire(void* addr);
void __tsan_release(void* addr);
}
#define CV_TSAN_SWITCH(fiber) __tsan_switch_to_fiber(fiber, 1u /* no_sync */)
#define CV_TSAN_ACQUIRE(p) __tsan_acquire(p)
#define CV_TSAN_RELEASE(p) __tsan_release(p)
#else
#define CV_TSAN_SWITCH(fiber) ((void)0)
#define CV_TSAN_ACQUIRE(p) ((void)0)
#define CV_TSAN_RELEASE(p) ((void)0)
#endif

namespace cv_emu {
namespace {

constexpr size_t kStackBytes = 64 << 10;
constexpr size_t kDynSmemBytes = 232448;  // 227 KB, the per-CTA maximum on sm_90
constexpr unsigned kMaxThreads = 1024;

enum State : uint8_t { kRunnable, kWaitWarp, kWaitBlock, kDone };

struct Fiber {
    void* sp = nullptr;
    void* asan_fake = nullptr;
    void* tsan = nullptr;  // TSan context of this fiber slot (kept across blocks: its stack is reused too)
    uint32_t bar_gen, warp_gen;  // collectives this fiber has been through: consecutive ones use different sync objects
    ThreadCtx ctx;
    State state;
    uint8_t lane, parity;
    uint16_t warp;
};
struct Warp {
    uint32_t live, arrived, wait_mask;
    uint32_t part[3];  // lanes that took part in the last collective that used data slot 0 / 1 (2: plain __syncwarp)
    uint32_t wait_slot;
    uint64_t slot[2][32];
    char hb[2];  // happens-before objects of the warp's collectives (TSan build)
};
struct Job {
    dim3 grid, block;
    size_t smem;
    Thunk thunk;
    void *kernel, *args;
    std::atomic<uint64_t> next{0};
    uint64_t n_blocks = 0;
    char hb_launch = 0;  // happens-before object: what the launching host thread did before the launch (TSan build)
};

struct Worker {
    Fiber fibers[kMaxThreads];
    Warp warps[kMaxThreads / 32];
    char* stacks = nullptr;
    char* smem = nullptr;
    void* sched_sp = nullptr;
    void* sched_tsan = nullptr;
    char hb_end[2] = {0, 0}, hb_bar[2] = {0, 0};  // happens-before objects: end of the even/odd blocks of this worker / __syncthreads (TSan build)
    uint64_t block_seq = 0;
    const void* sched_bottom = nullptr;  // the scheduler's own stack, as ASan reported it at the first switch
    size_t sched_size = 0;
    Fiber* running = nullptr;
    const Job* job = nullptr;
    unsigned n_threads = 0, live = 0, bar_arrived = 0;

    Worker() {
        stacks = static_cast<char*>(mmap(nullptr, kStackBytes * kMaxThreads, PROT_READ | PROT_WRITE, MAP_PRIVATE | MAP_ANONYMOUS | MAP_NORESERVE, -1, 0));
        if (stacks == MAP_FAILED || posix_memalign(reinterpret_cast<void**>(&smem), 1024, kDynSmemBytes) != 0) {
            fprintf(stderr, "simt_emu: cannot allocate fiber stacks\n");
            abort();
        }
        memset(smem, 0, kDynSmemBytes);
#if defined(CV_EMU_TSAN)
        // The runtime tells at most 256 concurrently live contexts apart (its shadow stores an 8-bit slot id; beyond that slots are
        // recycled and races between recycled contexts go unseen).  So: every LANE of the first two warps is a context of its own
        // (races inside a warp -- a missing __syncwarp -- show there; the code is the same in every warp), the other warps are one
        // context each (races between warps -- a missing __syncthreads -- show everywhere): 94 contexts per worker.  Created here, at
        // worker start: a context inherits its creator's ordering, which must not yet include any other worker's blocks.
        for (unsigned i = 0; i < kMaxThreads; i++) fibers[i].tsan = (i < 64 || (i & 31) == 0) ? __tsan_create_fiber(0) : fibers[i & ~31u].tsan;
#endif
    }
    ~Worker() {
        munmap(stacks, kStackBytes * kMaxThreads);
        free(smem);
    }
};

thread_local Worker* t_worker = nullptr;

void yield(Worker* w, Fiber* f) {
    CV_ASAN_START(&f->asan_fake, w->sched_bottom, w->sched_size);
    CV_TSAN_SWITCH(w->sched_tsan);
    cv_emu_switch(&f->sp, w->sched_sp);
    CV_ASAN_FINISH(f->asan_fake, nullptr, nullptr);
}

void release_warp(Worker* w, Warp& W, unsigned warp_index) {
    uint32_t m = W.arrived;
    W.part[W.wait_slot] = m;
    W.arrived = 0;
    while (m) {
        const int l = __builtin_ctz(m);
        m &= m - 1;
        Fiber& g = w->fibers[warp_index * 32 + l];
        if (g.state == kWaitWarp) g.state = kRunnable;
    }
}
void release_block(Worker* w) {
    w->bar_arrived = 0;
    for (unsigned i = 0; i < w->n_threads; i++)
        if (w->fibers[i].state == kWaitBlock) w->fibers[i].state = kRunnable;
}

[[noreturn]] void fiber_exit(Worker* w, Fiber* f) {
    f->state = kDone;
    w->live--;
    Warp& W = w->warps[f->warp];
    W.live &= ~(1u << f->lane);
    // a thread that has returned no longer takes part in collectives: its exit may complete one
    if (W.arrived && (W.arrived & W.wait_mask & W.live) == (W.wait_mask & W.live)) release_warp(w, W, f->warp);
    if (w->bar_arrived && w->bar_arrived == w->live) release_block(w);
    CV_TSAN_RELEASE(&w->hb_end[w->block_seq & 1]);
    CV_ASAN_START(nullptr, w->sched_bottom, w->sched_size);  // nullptr: this stack's frames are gone for good
    CV_TSAN_SWITCH(w->sched_tsan);
    cv_emu_switch(&f->sp, w->sched_sp);
    abort();
}

void fiber_main() {
    Worker* w = t_worker;
    Fiber* f = w->running;
    CV_ASAN_FINISH(nullptr, &w->sched_bottom, &w->sched_size);
    // ordered after the launch and after the previous block of this worker (whose stacks and shared memory this block reuses) --
    // NOT after whatever the worker thread itself synchronised with (the pool's mutex would order whole workers one after the other)
    CV_TSAN_ACQUIRE(const_cast<char*>(&w->job->hb_launch));
    CV_TSAN_ACQUIRE(&w->hb_end[(w->block_seq + 1) & 1]);  // the object the PREVIOUS block's threads released at their exits
    w->job->thunk(w->job->kernel, w->job->args);
    fiber_exit(w, f);
}

void run_block(Worker* w, const Job& job, uint64_t b) {
    const unsigned n = job.block.x * job.block.y * job.block.z;
    w->job = &job, w->n_threads = n, w->live = n, w->bar_arrived = 0;
    const unsigned n_warps = (n + 31) / 32;
    for (unsigned i = 0; i < n_warps; i++) {
        Warp& W = w->warps[i];
        const unsigned in_warp = n - i * 32 >= 32 ? 32 : n - i * 32;
        W.live = in_warp == 32 ? 0xffffffffu : ((1u << in_warp) - 1u);
        W.arrived = 0, W.wait_mask = 0, W.wait_slot = 2;
    }
    for (unsigned i = 0; i < n; i++) {
        Fiber& f = w->fibers[i];
        f.ctx.tid = uint3{i % job.block.x, (i / job.block.x) % job.block.y, i / (job.block.x * job.block.y)};
        f.ctx.bid = uint3{static_cast<unsigned>(b % job.grid.x), static_cast<unsigned>((b / job.grid.x) % job.grid.y),
                          static_cast<unsigned>(b / (uint64_t(job.grid.x) * job.grid.y))};
        f.ctx.bdim = job.block, f.ctx.gdim = job.grid;
        f.asan_fake = nullptr;
        f.bar_gen = f.warp_gen = 0;
        f.state = kRunnable, f.lane = i & 31, f.warp = static_cast<uint16_t>(i >> 5), f.parity = 0;
        // fresh stack: [top-8] fake return address of fiber_main, [top-16] fiber_main, six zeroed callee-saved registers below
        void** top = reinterpret_cast<void**>(w->stacks + kStackBytes * (i + 1));
        top[-1] = nullptr;
        top[-2] = reinterpret_cast<void*>(&fiber_main);
        for (int k = 3; k <= 8; k++) top[-k] = nullptr;
        f.sp = top - 8;
    }
#if defined(CV_EMU_TSAN)
    if (!w->sched_tsan) w->sched_tsan = __tsan_get_current_fiber();
#endif
    while (w->live) {
        bool progressed = false;
        for (unsigned i = 0; i < n; i++) {
            Fiber& f = w->fibers[i];
            if (f.state != kRunnable) continue;
            progressed = true;
            w->running = &f;
            void* fake = nullptr;
            CV_ASAN_START(&fake, w->stacks + kStackBytes * i, kStackBytes);
            CV_TSAN_SWITCH(f.tsan);
            cv_emu_switch(&w->sched_sp, f.sp);
            CV_ASAN_FINISH(fake, nullptr, nullptr);
            (void)fake;
        }
        if (!progressed) {
            unsigned ww = 0, wb = 0;
            for (unsigned i = 0; i < n; i++) ww += w->fibers[i].state == kWaitWarp, wb += w->fibers[i].state == kWaitBlock;
            fprintf(stderr, "simt_emu: deadlock in block %llu: %u threads live, %u wait at a warp collective, %u at __syncthreads "
                            "(a collective some live participant never reaches)\n", (unsigned long long)b, w->live, ww, wb);
            abort();
        }
    }
    CV_TSAN_ACQUIRE(&w->hb_end[w->block_seq & 1]);  // everything the block's threads did is ordered before whatever follows the launch
    w->block_seq++;
    w->running = nullptr;
}

// ---- worker pool: the blocks of one grid at a time
struct Pool {
    std::mutex mu, launch_mu;
    std::condition_variable cv, done_cv;
    std::vector<std::thread> threads;
    Job* job = nullptr;
    uint64_t generation = 0;
    unsigned busy = 0;
    bool stop = false;

    Pool() {
        unsigned n = std::thread::hardware_concurrency();
        if (const char* e = getenv("CV_SIMT_EMU_THREADS")) n = static_cast<unsigned>(atoi(e));
        if (n < 1) n = 1;
        if (n > 16) n = 16;
        for (unsigned i = 0; i < n; i++) threads.emplace_back([this, i] { loop(i); });
    }
    ~Pool() {
        {
            std::lock_guard<std::mutex> lk(mu);
            stop = true;
        }
        cv.notify_all();
        for (auto& t : threads) t.join();
    }
    void loop(unsigned index) {
        Worker* w = new Worker;
        t_worker = w;
        uint64_t seen = 0;
        (void)index;
        for (;;) {
            Job* j;
            {
                std::unique_lock<std::mutex> lk(mu);
                cv.wait(lk, [&] { return stop || (job && generation != seen); });
                if (stop) break;
                seen = generation, j = job, busy++;
            }
#if defined(CV_EMU_TSAN)
            // race check: blocks of one worker are ordered one after the other (they reuse its stacks and shared memory), so neighbouring
            // blocks always go to DIFFERENT workers -- a race between two blocks is then visible whichever runs first
            for (uint64_t b = index; b < j->n_blocks; b += threads.size()) run_block(w, *j, b);
            j->next.fetch_add(1, std::memory_order_relaxed);  // counts workers here
#else
            for (;;) {
                const uint64_t b = j->next.fetch_add(1, std::memory_order_relaxed);
                if (b >= j->n_blocks) break;
                run_block(w, *j, b);
            }
#endif
            {
                std::lock_guard<std::mutex> lk(mu);
                busy--;
            }
            done_cv.notify_all();
        }
        delete w;
    }
    void run(Job& j) {
        std::lock_guard<std::mutex> one(launch_mu);  // host threads launch concurrently (verifier, readers): one grid at a time
        CV_TSAN_RELEASE(&j.hb_launch);
        {
            std::lock_guard<std::mutex> lk(mu);
            job = &j, generation++;
        }
        cv.notify_all();
        std::unique_lock<std::mutex> lk(mu);
        // every block index has been handed out and every worker that took one is back (busy-- follows its last block)
#if defined(CV_EMU_TSAN)
        done_cv.wait(lk, [&] { return busy == 0 && j.next.load(std::memory_order_relaxed) >= threads.size(); });  // every worker has done its share
#else
        done_cv.wait(lk, [&] { return busy == 0 && j.next.load(std::memory_order_relaxed) >= j.n_blocks; });
#endif
        job = nullptr;
    }
};
Pool& pool() {
    static Pool* p = new Pool;  // never destroyed: worker threads must not be joined from a static destructor at exit
    return *p;
}

inline Worker* me() { return t_worker; }

}  // namespace

#if defined(__SANITIZE_ADDRESS__)
void asan_report_load16(const void* p) {
    volatile uint8_t sink = 0;
    for (int i = 0; i < 16; i++) sink ^= static_cast<const volatile uint8_t*>(p)[i];
    (void)sink;
}
#endif

const ThreadCtx* cur() { return &t_worker->running->ctx; }
char* dyn_smem() { return t_worker->smem; }

void sync_block() {
    Worker* w = me();
    Fiber* f = w->running;
    char* hb = &w->hb_bar[f->bar_gen++ & 1];
    CV_TSAN_RELEASE(hb);
    w->bar_arrived++;
    if (w->bar_arrived == w->live) {
        release_block(w);
    } else {
        f->state = kWaitBlock;
        yield(w, f);
    }
    CV_TSAN_ACQUIRE(hb);
}

static void sync_warp_slot(uint32_t mask, uint32_t slot);
void sync_warp(uint32_t mask) { sync_warp_slot(mask, 2); }

static void sync_warp_slot(uint32_t mask, uint32_t slot) {
    Worker* w = me();
    Fiber* f = w->running;
    Warp& W = w->warps[f->warp];
    if (W.arrived && W.wait_mask != mask) {
        fprintf(stderr, "simt_emu: lanes of one warp wait at collectives with different masks (%08x vs %08x): not modelled\n", W.wait_mask, mask);
        abort();
    }
    char* hb = &W.hb[f->warp_gen++ & 1];
    CV_TSAN_RELEASE(hb);
    W.wait_mask = mask, W.wait_slot = slot;
    W.arrived |= 1u << f->lane;
    const uint32_t need = mask & W.live;
    if ((W.arrived & need) == need) {
        release_warp(w, W, f->warp);
    } else {
        f->state = kWaitWarp;
        yield(w, f);
    }
    CV_TSAN_ACQUIRE(hb);
}

uint64_t warp_exchange(uint32_t mask, uint64_t v, uint32_t src) {
    Worker* w = me();
    Fiber* f = w->running;
    Warp& W = w->warps[f->warp];
    // two slot sets, used alternately: a lane can only reach its next-but-one exchange after every lane has read this one
    const unsigned p = f->parity;
    f->parity ^= 1;
    W.slot[p][f->lane] = v;
    sync_warp_slot(mask, p);
    return (W.part[p] >> src) & 1u ? W.slot[p][src] : v;  // a lane that has returned (or is not named) deposits nothing
}

uint32_t warp_ballot(uint32_t mask, bool pred) {
    Worker* w = me();
    Fiber* f = w->running;
    Warp& W = w->warps[f->warp];
    const unsigned p = f->parity;
    f->parity ^= 1;
    W.slot[p][f->lane] = pred ? 1 : 0;
    sync_warp_slot(mask, p);
    uint32_t r = 0;
    for (uint32_t m = W.part[p]; m; m &= m - 1) {
        const int l = __builtin_ctz(m);
        if (W.slot[p][l]) r |= 1u << l;
    }
    return r;
}

namespace {
struct Launch {
    dim3 grid, block;
    size_t smem;
    Thunk thunk;
    void *kernel, *args;
    void (*free_args)(void*);
};
void run_launch(void* p) {
    Launch* l = static_cast<Launch*>(p);
    Job j;
    j.grid = l->grid, j.block = l->block, j.smem = l->smem, j.thunk = l->thunk, j.kernel = l->kernel, j.args = l->args;
    j.n_blocks = uint64_t(l->grid.x) * l->grid.y * l->grid.z;
    pool().run(j);
    l->free_args(l->args);
    delete l;
}
}  // namespace

void launch(void* stream, dim3 grid, dim3 block, size_t smem_bytes, Thunk thunk, void* kernel, void* args, void (*free_args)(void*)) {
    const uint64_t n_threads = uint64_t(block.x) * block.y * block.z;
    const uint64_t n_blocks = uint64_t(grid.x) * grid.y * grid.z;
    if (n_threads == 0 || n_threads > kMaxThreads || smem_bytes > kDynSmemBytes || n_blocks == 0 || grid.x > 0x7fffffffu || grid.y > 65535u || grid.z > 65535u) {
        mock_cuda_set_last_error(9);  // cudaErrorInvalidConfiguration, reported by the launcher's cudaGetLastError like on the device
        free_args(args);
        return;
    }
    mock_cuda_enqueue(stream, &run_launch, new Launch{grid, block, smem_bytes, thunk, kernel, args, free_args});
}

}  // namespace cv_emu
