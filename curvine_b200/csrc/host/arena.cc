#include "arena.h"

#include <errno.h>
#include <fcntl.h>
#include <stdlib.h>
#include <sys/mman.h>
#include <sys/stat.h>
#include <unistd.h>

#include <atomic>
#include <thread>

#include "numa.h"

namespace cv {

MemArena::~MemArena() {
    for (auto& s : segs_) {
        if (s.base) munmap(s.base, static_cast<size_t>(seg_bytes_));
        if (s.fd >= 0) ::close(s.fd);
    }
}

std::string MemArena::seg_path(int32_t seg) const { return str_printf("%s/seg_%04d", dir_.c_str(), seg); }

std::string MemArena::encode_descriptor(const ArenaExtent& e, int64_t len) {
    return str_printf("%s %d %lld %lld\n", kMagic, e.seg, (long long)e.off, (long long)len);
}

bool MemArena::decode_descriptor(const std::string& text, ArenaExtent* e, int64_t* len) {
    char magic[16] = {0};
    int seg = 0;
    long long off = 0, l = 0;
    if (sscanf(text.c_str(), "%15s %d %lld %lld", magic, &seg, &off, &l) != 4 || strcmp(magic, kMagic) != 0) return false;
    if (seg < 0 || off < 0 || l < 0 || off % kGranule) return false;
    e->seg = seg, e->off = off, e->cap = (l + kGranule - 1) / kGranule * kGranule;
    *len = l;
    return true;
}

Err MemArena::init(const std::string& dir, int64_t capacity, int64_t seg_bytes, const std::vector<int>& cpus) {
    dir_ = dir, capacity_ = capacity, cpus_ = cpus;
    seg_bytes_ = std::max<int64_t>(kGranule, seg_bytes / kGranule * kGranule);
    if (mkdir(dir_.c_str(), 0755) != 0 && errno != EEXIST) return Err::io(str_printf("mkdir %s: %s", dir_.c_str(), strerror(errno)));
    // segments left by a previous worker run are taken over as they are (their blocks come back through the descriptors)
    size_t existing = 0;
    for (;; existing++) {
        struct stat st;
        if (stat(seg_path(static_cast<int32_t>(existing)).c_str(), &st) != 0) break;
        if (st.st_size != seg_bytes_) return Err::common(str_printf("arena segment %s has %lld bytes, [worker] arena_segment says %lld", seg_path(static_cast<int32_t>(existing)).c_str(), (long long)st.st_size, (long long)seg_bytes_));
    }
    const size_t want = capacity > 0 ? static_cast<size_t>((capacity + seg_bytes_ - 1) / seg_bytes_) : 1;
    return add_segments(std::max(existing, want));
}

// Creates (or re-opens) segments [segs_.size(), n): ftruncate, map shared, first-touch every page from threads bound to
// the arena's CPUs so the pages land on that NUMA node.  Called with mu_ held or before the arena is shared.
Err MemArena::add_segments(size_t n) {
    const size_t first = segs_.size();
    if (n <= first) return Err::ok();
    const double t0 = now_sec();
    segs_.resize(n);
    std::vector<uint8_t> fresh(n, 0);
    for (size_t s = first; s < n; s++) {
        const std::string p = seg_path(static_cast<int32_t>(s));
        struct stat st;
        fresh[s] = stat(p.c_str(), &st) != 0;
        const int fd = ::open(p.c_str(), O_RDWR | O_CREAT | O_CLOEXEC, 0644);
        if (fd < 0) return Err::io(str_printf("open %s: %s", p.c_str(), strerror(errno)));
        if (fresh[s] && ftruncate(fd, seg_bytes_) != 0) {
            const int e = errno;
            ::close(fd);
            return Err::io(str_printf("ftruncate %s: %s", p.c_str(), strerror(e)));
        }
        void* m = mmap(nullptr, static_cast<size_t>(seg_bytes_), PROT_READ | PROT_WRITE, MAP_SHARED, fd, 0);
        if (m == MAP_FAILED) {
            ::close(fd);
            return Err::io(str_printf("mmap %s: %s", p.c_str(), strerror(errno)));
        }
        segs_[s].base = static_cast<uint8_t*>(m), segs_[s].fd = fd;
    }
    // populate: slices of 64 MiB handed to a few threads
    const int64_t slice = 64ll << 20;
    std::vector<std::pair<size_t, int64_t>> work;
    for (size_t s = first; s < n; s++)
        if (fresh[s])
            for (int64_t o = 0; o < seg_bytes_; o += slice) work.emplace_back(s, o);
    std::atomic<size_t> next{0};
    const size_t T = std::min<size_t>(work.size(), cpus_.empty() ? 16 : std::min<size_t>(32, cpus_.size()));
    std::vector<std::thread> ts;
    for (size_t t = 0; t < T; t++)
        ts.emplace_back([&] {
            bind_cpus(cpus_);
            for (;;) {
                const size_t i = next.fetch_add(1);
                if (i >= work.size()) break;
                volatile uint8_t* p = segs_[work[i].first].base + work[i].second;
                const int64_t end = std::min(slice, seg_bytes_ - work[i].second);
                for (int64_t o = 0; o < end; o += kGranule) p[o] = 0;
            }
        });
    for (auto& t : ts) t.join();
    populate_sec += now_sec() - t0;
    return Err::ok();
}

int64_t MemArena::used_bytes() const {
    std::lock_guard<std::mutex> lk(mu_);
    return used_;
}

Err MemArena::alloc(int64_t bytes, ArenaExtent* out) {
    const int64_t need = std::max<int64_t>(kGranule, (bytes + kGranule - 1) / kGranule * kGranule);
    if (need > seg_bytes_) return Err::common(str_printf("block of %lld bytes does not fit an arena segment of %lld bytes", (long long)bytes, (long long)seg_bytes_));
    std::lock_guard<std::mutex> lk(mu_);
    drain_quarantine_locked(false);
    for (;;) {
        // bump first: a sequential writer gets back-to-back extents (one DMA moves a whole copy group)
        const int64_t total = static_cast<int64_t>(segs_.size()) * seg_bytes_;
        int64_t room_in_seg = seg_bytes_ - bump_ % seg_bytes_;
        if (bump_ < total && room_in_seg < need) {  // the tail of this segment is too small: it goes on the free list
            free_[bump_] = room_in_seg;
            bump_ += room_in_seg;
            room_in_seg = seg_bytes_;
        }
        if (bump_ + need <= total) {
            out->seg = static_cast<int32_t>(bump_ / seg_bytes_), out->off = bump_ % seg_bytes_, out->cap = need;
            bump_ += need;
            used_ += need;
            return Err::ok();
        }
        for (auto it = free_.begin(); it != free_.end(); ++it)  // first fit
            if (it->second >= need) {
                const int64_t at = it->first, len = it->second;
                free_.erase(it);
                if (len > need) free_[at + need] = len - need;
                out->seg = static_cast<int32_t>(at / seg_bytes_), out->off = at % seg_bytes_, out->cap = need;
                used_ += need;
                return Err::ok();
            }
        if (drain_quarantine_locked(true)) continue;  // space freed moments ago becomes usable once its quarantine is over
        if (capacity_ > 0) return Err(kDiskOutOfSpace, str_printf("mem arena %s is full (%lld of %lld bytes in use)", dir_.c_str(), (long long)used_, (long long)total));
        CV_RETURN_IF_ERR(add_segments(segs_.size() + 1));  // unbounded arena: one more segment
    }
}

void MemArena::free(const ArenaExtent& e) {
    if (e.seg < 0 || e.cap <= 0) return;
    std::lock_guard<std::mutex> lk(mu_);
    if (reuse_delay_ms <= 0) release_locked(e);
    else quarantine_.emplace_back(now_sec() + static_cast<double>(reuse_delay_ms) / 1000.0, e);
}

void MemArena::release_now(const ArenaExtent& e) {
    if (e.seg < 0 || e.cap <= 0) return;
    std::lock_guard<std::mutex> lk(mu_);
    release_locked(e);
}

// -> true when at least one extent left quarantine.  wait_one: sleep until the oldest one is due (caller is out of space).
bool MemArena::drain_quarantine_locked(bool wait_one) {
    bool any = false;
    while (!quarantine_.empty()) {
        const double due = quarantine_.front().first, now = now_sec();
        if (due > now) {
            if (!wait_one || any) break;
            usleep(static_cast<useconds_t>((due - now) * 1e6) + 100);
        }
        release_locked(quarantine_.front().second);
        quarantine_.pop_front();
        any = true;
    }
    return any;
}

void MemArena::release_locked(const ArenaExtent& e) {
    int64_t at = static_cast<int64_t>(e.seg) * seg_bytes_ + e.off, len = e.cap;
    used_ -= len;
    auto nx = free_.lower_bound(at);
    if (nx != free_.end() && at + len == nx->first && nx->first / seg_bytes_ == at / seg_bytes_) {  // merge right (same segment)
        len += nx->second;
        nx = free_.erase(nx);
    }
    if (nx != free_.begin()) {
        auto pv = std::prev(nx);
        if (pv->first + pv->second == at && pv->first / seg_bytes_ == at / seg_bytes_) {  // merge left
            pv->second += len;
            return;
        }
    }
    free_[at] = len;
}

void MemArena::shrink(ArenaExtent* e, int64_t used) {
    const int64_t keep = std::max<int64_t>(kGranule, (used + kGranule - 1) / kGranule * kGranule);
    if (keep >= e->cap) return;
    ArenaExtent tail;
    tail.seg = e->seg, tail.off = e->off + keep, tail.cap = e->cap - keep;
    e->cap = keep;
    std::lock_guard<std::mutex> lk(mu_);
    release_locked(tail);  // never-committed bytes: nobody can be reading them, no quarantine
}

Err MemArena::mark_used(const ArenaExtent& e) {
    if (e.seg < 0 || static_cast<size_t>(e.seg) >= segs_.size() || e.off + e.cap > seg_bytes_) return Err::common("extent descriptor outside the arena");
    std::lock_guard<std::mutex> lk(mu_);
    const int64_t at = static_cast<int64_t>(e.seg) * seg_bytes_ + e.off, end = at + e.cap;
    if (at >= bump_) {  // beyond everything handed out so far: the gap becomes free space
        int64_t g = bump_;
        while (g < at) {  // never straddling a segment
            const int64_t stop = std::min(at, (g / seg_bytes_ + 1) * seg_bytes_);
            free_[g] = stop - g;
            g = stop;
        }
        bump_ = end;
        used_ += e.cap;
        return Err::ok();
    }
    auto it = free_.upper_bound(at);
    if (it == free_.begin()) return Err::common("extent descriptor overlaps another block");
    --it;
    const int64_t fa = it->first, fl = it->second;
    if (fa > at || fa + fl < end) return Err::common("extent descriptor overlaps another block");
    free_.erase(it);
    if (fa < at) free_[fa] = at - fa;
    if (fa + fl > end) free_[end] = fa + fl - end;
    used_ += e.cap;
    return Err::ok();
}

}  // namespace cv
