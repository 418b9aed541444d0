// Host memory the copy engine reads from directly: the registered-mapping cache of block files, its background registrar, and the
// mem-arena segments pinned once per context.  Used by the device reader (gpu_reader.cu).
#pragma once
#include <cuda_runtime.h>
#include <errno.h>
#include <fcntl.h>
#include <sys/mman.h>
#include <sys/stat.h>
#include <unistd.h>

#include <atomic>
#include <condition_variable>
#include <deque>
#include <list>
#include <memory>
#include <mutex>
#include <set>
#include <thread>
#include <unordered_map>
#include <vector>

#include "common.h"
#include "numa.h"

namespace cv {

inline size_t page_up(size_t bytes) { return (bytes + 4095) & ~size_t(4095); }

// ------------------------------------------------------------------ registered mem-tier mappings (zero-copy ingest)
//
// A mem-tier block file lives in tmpfs page-cache pages.  Instead of pread()ing it into a pinned slot (one CPU copy
// per byte), map the block files of one copy group back to back into a reserved VA range, cudaHostRegister the range
// once, and let the copy engine DMA straight out of the page cache.  Mappings are cached (LRU by bytes, never more than
// `register_cache` bytes registered through the cache) and revalidated by (inode, size, mtime) on every use; block files
// are write-once in Curvine.
// Admission is scan-resistant: a new mapping only displaces mappings that nobody is using AND that have not been used for
// `register_min_age` (default 5 s); otherwise the newcomer is not cached (its group keeps going through the pinned ring).
// With plain LRU a sequential re-read of a file larger than the cache finds every group evicted just before it gets there
// -- 0 hits while paying registration every pass; with this rule the first cache-full of groups stays registered and a
// cyclic scan hits cache/working-set of the time, while a working set that moved away ages out after register_min_age.
struct RegMapping {
    std::string key;
    uint8_t* base = nullptr;
    size_t bytes = 0;     // registered extent (page-rounded)
    std::vector<uint64_t> stamps;  // inode, size, mtime_ns per member file
    bool registered = false;
    double last_used = 0;  // now_sec() of the last find() hit or the insertion (under RegCache's lock)
    ~RegMapping() {
        if (registered) cudaHostUnregister(base);
        if (base) munmap(base, bytes);
    }
};

class RegCache {
   public:
    size_t capacity = 0;   // bytes; 0 disables caching (mappings live for one call)
    double min_age_sec = 5.0;  // a mapping used more recently than this is not displaced by a newcomer
    std::shared_ptr<RegMapping> find(const std::string& key, const std::vector<uint64_t>& stamps) {
        std::shared_ptr<RegMapping> stale;  // destroyed (unregistered, unmapped) outside the lock
        std::lock_guard<std::mutex> lk(mu_);
        auto it = map_.find(key);
        if (it == map_.end()) return nullptr;
        if (it->second->second->stamps != stamps) {  // file replaced: drop the stale mapping
            stale = it->second->second;
            bytes_ -= stale->bytes;
            lru_.erase(it->second);
            map_.erase(it);
            return nullptr;
        }
        lru_.splice(lru_.begin(), lru_, it->second);
        it->second->second->last_used = now_sec();
        hits++;
        return it->second->second;
    }
    // -> true when the mapping was admitted.  A rejected mapping stays valid for the caller's own use and goes away with it.
    bool insert(const std::shared_ptr<RegMapping>& m) {
        std::vector<std::shared_ptr<RegMapping>> evicted;  // destroyed outside the lock
        std::lock_guard<std::mutex> lk(mu_);
        if (capacity == 0 || m->bytes > capacity) return false;
        auto dup = map_.find(m->key);
        if (dup != map_.end()) {  // same group registered twice (two contexts' worth of threads raced): the newer one wins
            bytes_ -= dup->second->second->bytes;
            evicted.push_back(dup->second->second);
            lru_.erase(dup->second);
            map_.erase(dup);
        }
        const double now = now_sec();
        // make room from the cold end; stop at the first entry that is in use or still young
        while (bytes_ + m->bytes > capacity && !lru_.empty()) {
            auto& back = lru_.back();
            if (back.second.use_count() > 1 || now - back.second->last_used < min_age_sec) break;
            bytes_ -= back.second->bytes;
            evicted.push_back(back.second);
            map_.erase(back.first);
            lru_.pop_back();
        }
        if (bytes_ + m->bytes > capacity) {
            rejected++;
            return false;
        }
        m->last_used = now;
        lru_.emplace_front(m->key, m);
        map_[m->key] = lru_.begin();
        bytes_ += m->bytes;
        return true;
    }
    // would insert() admit a mapping of `bytes` right now?  (asked BEFORE paying for mmap + cudaHostRegister)
    bool can_admit(size_t bytes) {
        std::lock_guard<std::mutex> lk(mu_);
        if (capacity == 0 || bytes > capacity) return false;
        size_t room = capacity - std::min(capacity, bytes_);
        const double now = now_sec();
        for (auto it = lru_.rbegin(); room < bytes && it != lru_.rend(); ++it) {
            if (it->second.use_count() > 1 || now - it->second->last_used < min_age_sec) break;
            room += it->second->bytes;
        }
        return room >= bytes;
    }
    void clear() {
        std::lock_guard<std::mutex> lk(mu_);
        map_.clear();
        lru_.clear();
        bytes_ = 0;
    }
    size_t bytes() {
        std::lock_guard<std::mutex> lk(mu_);
        return bytes_;
    }
    std::atomic<uint64_t> hits{0}, misses{0}, rejected{0};

   private:
    std::mutex mu_;
    std::list<std::pair<std::string, std::shared_ptr<RegMapping>>> lru_;
    std::unordered_map<std::string, std::list<std::pair<std::string, std::shared_ptr<RegMapping>>>::iterator> map_;
    size_t bytes_ = 0;
};

// Map `paths` (lens[i] bytes each; all but the last a multiple of the page size) contiguously and register the range.
Err map_and_register(const std::vector<std::string>& paths, const std::vector<int64_t>& lens, std::shared_ptr<RegMapping>* out,
                     std::vector<uint64_t>* stamps_out);
bool stat_stamps(const std::vector<std::string>& paths, std::vector<uint64_t>* stamps);  // false when a path cannot be stat'ed

// Background registration: a cache miss does not stall the read.  The foreground moves the group through the pinned
// ring right away (cold pass at ring speed) while a few registrar threads mmap + cudaHostRegister the same files so that
// the NEXT pass over them is zero-copy.  cudaHostRegister pins 4 KiB pages at a few GB/s per thread and
// serialises with copy enqueues inside the driver, so by default (`register_when_idle`) the registrar threads yield to
// reads in flight: `hold` counts them, and a registrar only starts a new group while it is zero (or while a caller is
// blocked in drain()).
class Registrar {
   public:
    struct Job {
        std::string key;
        std::vector<std::string> paths;
        std::vector<int64_t> lens;
    };
    void start(int threads, int device, RegCache* cache, std::vector<int> cpus, const std::atomic<int>* hold) {
        device_ = device, cache_ = cache, cpus_ = std::move(cpus), hold_ = hold;
        for (int t = 0; t < threads; t++) threads_.emplace_back([this] { loop(); });
    }
    void submit(Job j) {
        std::lock_guard<std::mutex> lk(mu_);
        if (stop_ || unsupported.load() || !pending_keys_.insert(j.key).second) return;
        q_.push_back(std::move(j));
        cv_.notify_one();
    }
    void stop() {
        {
            std::lock_guard<std::mutex> lk(mu_);
            stop_ = true;
            q_.clear();
            cv_.notify_all();
        }
        for (auto& t : threads_) t.join();
        threads_.clear();
    }
    void drain() {  // wait until the queue is empty and no registration is in flight
        std::unique_lock<std::mutex> lk(mu_);
        draining_++;
        idle_cv_.wait(lk, [&] { return (q_.empty() && busy_ == 0) || stop_; });
        draining_--;
    }
    size_t backlog() {
        std::lock_guard<std::mutex> lk(mu_);
        return q_.size() + static_cast<size_t>(busy_);
    }
    std::atomic<bool> unsupported{false};
    std::atomic<uint64_t> registered{0};

   private:
    void loop() {
        bind_cpus(cpus_);
        cudaSetDevice(device_);
        for (;;) {
            Job j;
            {
                std::unique_lock<std::mutex> lk(mu_);
                cv_.wait(lk, [&] { return stop_ || !q_.empty(); });
                if (stop_) return;
                if (hold_ && hold_->load(std::memory_order_acquire) > 0 && draining_ == 0) {  // a read is in flight: stay out of its way
                    lk.unlock();
                    usleep(300);
                    continue;
                }
                j = std::move(q_.front());
                q_.pop_front();
                busy_++;
            }
            std::shared_ptr<RegMapping> m;
            std::vector<uint64_t> stamps;
            size_t job_bytes = 0;
            for (int64_t l : j.lens) job_bytes += page_up(static_cast<size_t>(l));
            Err e = cache_->can_admit(job_bytes) ? map_and_register(j.paths, j.lens, &m, &stamps) : Err(kCommon, "registration cache is full");
            if (!e) {
                m->key = j.key;
                if (cache_->insert(m)) registered++;
            } else if (e.kind == kUnsupported) {
                unsupported.store(true);
            }
            std::lock_guard<std::mutex> lk(mu_);
            pending_keys_.erase(j.key);
            busy_--;
            if (q_.empty() && busy_ == 0) idle_cv_.notify_all();
        }
    }
    int device_ = 0;
    RegCache* cache_ = nullptr;
    std::vector<int> cpus_;
    std::vector<std::thread> threads_;
    std::mutex mu_;
    std::condition_variable cv_, idle_cv_;
    std::deque<Job> q_;
    std::set<std::string> pending_keys_;
    int busy_ = 0, draining_ = 0;
    bool stop_ = false;
    const std::atomic<int>* hold_ = nullptr;
};

// ------------------------------------------------------------------ mem-arena segments (pinned once, off the read path)
//
// An arena-backed worker (arena.h) keeps every mem-tier block as an extent of a few large tmpfs segment files.  A segment is
// mapped and cudaHostRegister'ed ONCE per context -- in the background from the first device read on for the dirs named in
// `[b200] arena_preregister`, on demand for any other segment an Open names -- and stays pinned until the context closes.
// From then on every block in it, whatever file it belongs to and whenever it was written, is DMA'd straight out of the
// segment: no per-file or per-block client state, so the first read of a file runs at the same rate as a re-read.
// Registration is sliced (`arena_register_slice`) so that all registrar threads pin one segment together.
struct ArenaSeg {
    std::string path;
    uint8_t* base = nullptr;
    size_t bytes = 0, slice = 0;
    uint64_t ino = 0;
    std::vector<uint8_t> slice_registered;
    std::mutex mu;
    std::condition_variable cv;
    size_t slices_left = 0;
    bool done = false;
    Err err;
    ~ArenaSeg() {
        if (base) mprotect(base, bytes, PROT_READ | PROT_WRITE);
        for (size_t i = 0; i < slice_registered.size(); i++)
            if (slice_registered[i]) cudaHostUnregister(base + i * slice);
        if (base) munmap(base, bytes);
    }
};

class ArenaSegs {
   public:
    std::atomic<uint64_t> dma_jobs{0}, dma_bytes{0};  // block jobs / bytes moved straight out of a pinned segment
    std::atomic<bool> unsupported{false};             // cudaHostRegister refuses these mappings: arena blocks go through the ring
    double register_sec = 0;                          // wall time from the first slice queued to the last one pinned (under mu_)

    void start(int threads, int device, std::vector<int> cpus, size_t slice) {
        device_ = device, cpus_ = std::move(cpus), slice_ = std::max<size_t>(slice, 2 << 20) & ~size_t(4095);
        for (int t = 0; t < std::max(1, threads); t++) threads_.emplace_back([this] { loop(); });
    }
    void stop() {
        {
            std::lock_guard<std::mutex> lk(mu_);
            stop_ = true;
            q_.clear();
            cv_.notify_all();
        }
        for (auto& t : threads_) t.join();
        threads_.clear();
        std::lock_guard<std::mutex> lk(mu_);
        segs_.clear();
        retired_.clear();
    }
    // Every seg_* file under <data_dir>/<cluster_id>/arena is queued for mapping + pinning.  Returns immediately.
    void preregister_dir(const std::string& arena_dir) {
        for (int k = 0;; k++) {
            const std::string p = str_printf("%s/seg_%04d", arena_dir.c_str(), k);
            struct stat st;
            if (stat(p.c_str(), &st) != 0) break;
            std::shared_ptr<ArenaSeg> seg;
            begin(p, &seg);
        }
    }
    // The pinned mapping of segment `path` (blocks until it is fully registered; starts the registration if nobody has).
    Err get(const std::string& path, std::shared_ptr<ArenaSeg>* out) {
        std::shared_ptr<ArenaSeg> seg;
        CV_RETURN_IF_ERR(begin(path, &seg));
        std::unique_lock<std::mutex> lk(seg->mu);
        seg->cv.wait(lk, [&] { return seg->done; });
        if (seg->err) return seg->err;
        *out = std::move(seg);
        return Err::ok();
    }
    void drain() {  // wait until everything queued so far is pinned
        std::vector<std::shared_ptr<ArenaSeg>> all;
        {
            std::lock_guard<std::mutex> lk(mu_);
            for (auto& kv : segs_) all.push_back(kv.second);
        }
        for (auto& seg : all) {
            std::unique_lock<std::mutex> lk(seg->mu);
            seg->cv.wait(lk, [&] { return seg->done; });
        }
    }
    void stats(uint64_t* n_segs, uint64_t* bytes, double* sec) {
        std::lock_guard<std::mutex> lk(mu_);
        *n_segs = segs_.size(), *bytes = 0, *sec = register_sec;
        for (auto& kv : segs_) *bytes += kv.second->err ? 0 : kv.second->bytes;
    }

   private:
    Err begin(const std::string& path, std::shared_ptr<ArenaSeg>* out) {
        struct stat st;
        if (stat(path.c_str(), &st) != 0) return Err::io(str_printf("arena segment %s: %s", path.c_str(), strerror(errno)));
        std::lock_guard<std::mutex> lk(mu_);
        auto it = segs_.find(path);
        if (it != segs_.end() && it->second->ino == static_cast<uint64_t>(st.st_ino) && it->second->bytes == static_cast<size_t>(st.st_size)) {
            *out = it->second;
            return Err::ok();
        }
        if (it != segs_.end()) retired_.push_back(it->second);  // the file was replaced (worker restarted on a fresh dir): copies may still be in flight
        if (unsupported.load()) return Err(kUnsupported, "cudaHostRegister of arena segments is not supported here");
        std::shared_ptr<ArenaSeg> seg(new ArenaSeg());
        seg->path = path, seg->bytes = static_cast<size_t>(st.st_size), seg->ino = static_cast<uint64_t>(st.st_ino), seg->slice = slice_;
        // cudaHostRegister needs a writable shared mapping (cudaHostRegisterReadOnly is refused on this platform); the mapping is
        // write-protected again as soon as it is pinned
        const int fd = ::open(path.c_str(), O_RDWR | O_CLOEXEC);
        if (fd < 0) return Err(kUnsupported, str_printf("open %s read-write: %s", path.c_str(), strerror(errno)));
        void* m = mmap(nullptr, seg->bytes, PROT_READ | PROT_WRITE, MAP_SHARED, fd, 0);
        ::close(fd);
        if (m == MAP_FAILED) return Err::io(str_printf("mmap %s: %s", path.c_str(), strerror(errno)));
        seg->base = static_cast<uint8_t*>(m);
        const size_t n = (seg->bytes + slice_ - 1) / slice_;
        seg->slice_registered.assign(n, 0);
        seg->slices_left = n;
        if (busy_ == 0 && q_.empty()) t_first_ = now_sec();
        for (size_t i = 0; i < n; i++) q_.emplace_back(seg, i);
        segs_[path] = seg;
        cv_.notify_all();
        *out = std::move(seg);
        return Err::ok();
    }
    void loop() {
        bind_cpus(cpus_);
        cudaSetDevice(device_);
        for (;;) {
            std::pair<std::shared_ptr<ArenaSeg>, size_t> job;
            {
                std::unique_lock<std::mutex> lk(mu_);
                cv_.wait(lk, [&] { return stop_ || !q_.empty(); });
                if (stop_) return;
                job = std::move(q_.front());
                q_.pop_front();
                busy_++;
            }
            ArenaSeg& seg = *job.first;
            const size_t off = job.second * seg.slice, len = std::min(seg.slice, seg.bytes - off);
#ifdef MADV_POPULATE_WRITE
            // map the slice's (already allocated) tmpfs pages in bulk first: the page-by-page faults cudaHostRegister would
            // otherwise take on a fresh mapping are what made pinning 3x slower than on the mapping that created the pages
            madvise(seg.base + off, len, MADV_POPULATE_WRITE);
#endif
            const cudaError_t ce = cudaHostRegister(seg.base + off, len, cudaHostRegisterDefault);
            if (ce != cudaSuccess) cudaGetLastError();
            bool last = false;
            {
                std::lock_guard<std::mutex> lk(seg.mu);
                if (ce == cudaSuccess) seg.slice_registered[job.second] = 1;
                else if (!seg.err) seg.err = Err(kUnsupported, str_printf("cudaHostRegister(%s + %zu, %zu): %s", seg.path.c_str(), off, len, cudaGetErrorString(ce)));
                last = --seg.slices_left == 0;
                if (last) {
                    if (!seg.err) mprotect(seg.base, seg.bytes, PROT_READ);  // pinned pages stay DMA-able; nothing in this process can scribble on them
                    else unsupported.store(true);
                    seg.done = true;
                    seg.cv.notify_all();
                }
            }
            std::lock_guard<std::mutex> lk(mu_);
            busy_--;
            if (busy_ == 0 && q_.empty()) register_sec += now_sec() - t_first_;
        }
    }
    int device_ = 0;
    size_t slice_ = 256 << 20;
    std::vector<int> cpus_;
    std::vector<std::thread> threads_;
    std::mutex mu_;
    std::condition_variable cv_;
    std::deque<std::pair<std::shared_ptr<ArenaSeg>, size_t>> q_;
    std::unordered_map<std::string, std::shared_ptr<ArenaSeg>> segs_;
    std::vector<std::shared_ptr<ArenaSeg>> retired_;
    int busy_ = 0;
    double t_first_ = 0;
    bool stop_ = false;
};

}  // namespace cv
