// Arena-backed mem tier (B200-native; no reference counterpart).
//
// The reference keeps a mem-tier block as one tmpfs file per block (block_meta.rs:199-237, SURVEY.md A12).  For a GPU
// client that is the wrong granularity: the copy engine can only DMA out of memory that was pinned and mapped for the
// device (cudaHostRegister), pinning costs ~1 GB/s per thread on 4 KiB tmpfs pages, and a file that did not exist when
// the client started can only be pinned on the read path -- so the first read of every file is a CPU copy through a
// pinned ring or pays the pinning inline (round 1: 20-32 GB/s cold against 55 GB/s warm).
//
// Here a `[MEM:cap]` data dir is ONE tmpfs arena of `cap` bytes, cut into a few large segment files
// (<base>/arena/seg_NNNN), created and populated when the worker starts.  Blocks are extents inside a segment.  A GPU
// client maps and pins the segments once, at mount time, off the read path; after that EVERY block the worker ever
// stores there -- including files written later -- is DMA-able at once: there is no per-file or per-block client state,
// so a never-read file streams at the same rate as a re-read.  The worker serves framed reads by sendfile(2) out of the
// segment file (tools/loopback_probe.cc compares it with send(2) from a mapping of the segment: the copy into socket buffers
// costs more than the page references sendfile takes).
//
// On-disk state (survives a worker restart like the reference's block files do): the reference path
// <base>/active/bX/bY/blk_<id> holds a one-line extent descriptor "CVARENA1 <seg> <off> <len>\n" instead of the bytes;
// BlockStore::scan_dir rebuilds the allocation map from the descriptors.
#pragma once
#include <deque>
#include <map>
#include <memory>
#include <mutex>
#include <vector>

#include "common.h"

namespace cv {

struct ArenaExtent {
    int32_t seg = -1;
    int64_t off = 0;  // inside the segment
    int64_t cap = 0;  // bytes reserved (page-rounded)
};

class MemArena {
   public:
    ~MemArena();
    // dir = <data_dir>/<cluster_id>/arena.  capacity 0 -> one segment to start with, grown a segment at a time.
    // cpus: populate (first-touch) the segments from threads bound to these CPUs (NUMA placement); empty = unbound.
    Err init(const std::string& dir, int64_t capacity, int64_t seg_bytes, const std::vector<int>& cpus);
    Err alloc(int64_t bytes, ArenaExtent* out);  // 4 KiB granules; never straddles a segment
    // The space is quarantined for reuse_delay_ms before it can be handed out again: a short-circuit client may still
    // have a DMA in flight out of an extent whose block was just deleted (it holds no descriptor the worker could wait on).
    void free(const ArenaExtent& e);
    int64_t reuse_delay_ms = 1000;
    void release_now(const ArenaExtent& e);  // no quarantine: for extents nobody can have been reading (never committed)
    void shrink(ArenaExtent* e, int64_t used);  // give the tail beyond `used` bytes back
    Err mark_used(const ArenaExtent& e);         // rescan: re-establish an allocation read from a descriptor
    int64_t seg_bytes() const { return seg_bytes_; }
    std::string seg_path(int32_t seg) const;
    uint8_t* base(int32_t seg) const { return segs_[static_cast<size_t>(seg)].base; }
    int fd(int32_t seg) const { return segs_[static_cast<size_t>(seg)].fd; }  // kept open: framed reads sendfile(2) out of the segment
    uint8_t* ptr(const ArenaExtent& e) const { return base(e.seg) + e.off; }
    size_t num_segments() const { return segs_.size(); }
    int64_t used_bytes() const;
    double populate_sec = 0;

    static constexpr int64_t kGranule = 4096;
    static constexpr const char* kMagic = "CVARENA1";
    static std::string encode_descriptor(const ArenaExtent& e, int64_t len);
    static bool decode_descriptor(const std::string& text, ArenaExtent* e, int64_t* len);

   private:
    struct Seg {
        uint8_t* base = nullptr;
        int fd = -1;
    };
    Err add_segments(size_t n);
    void release_locked(const ArenaExtent& e);
    bool drain_quarantine_locked(bool wait_one);
    std::deque<std::pair<double, ArenaExtent>> quarantine_;
    std::string dir_;
    int64_t seg_bytes_ = 0, capacity_ = 0;
    std::vector<int> cpus_;
    std::vector<Seg> segs_;
    mutable std::mutex mu_;
    int64_t bump_ = 0;                   // linear offset (seg * seg_bytes + off) of the never-used tail
    std::map<int64_t, int64_t> free_;    // linear offset -> length, coalesced, never straddling a segment
    int64_t used_ = 0;
};

// Keeps an extent allocated while anything still reads it: the BlockStore entry holds one reference, every worker-side
// read context another; the extent goes back to the arena (into quarantine) when the last one drops.
struct ExtentHold {
    std::shared_ptr<MemArena> arena;
    ArenaExtent ext;
    ExtentHold(std::shared_ptr<MemArena> a, const ArenaExtent& e) : arena(std::move(a)), ext(e) {}
    ~ExtentHold() { arena->free(ext); }
    ExtentHold(const ExtentHold&) = delete;
    ExtentHold& operator=(const ExtentHold&) = delete;
    uint8_t* ptr() const { return arena->ptr(ext); }
};

}  // namespace cv
