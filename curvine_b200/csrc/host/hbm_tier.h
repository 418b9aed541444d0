// HBM as a worker tier (SURVEY.md 8f-2, the worker-side CUDA counterpart of ReadHandler): blocks resident in device
// memory are served to remote clients as orpc frames that were PACKED ON THE GPU (K4: prefixes written, payload copied
// behind them, CRC computed at the source) and moved D2H once per block.
//
// Reference shape it mirrors: ReadHandler::{open,read} (curvine-server/src/worker/handler/read_handler.rs:60-183) +
// RpcFrame::send (orpc/src/handler/rpc_frame.rs:205-220); the tier sits beside Mem/Ssd/Hdd
// (curvine-common/src/state/storage_info.rs:36-49).
#pragma once
#include <atomic>
#include <condition_variable>
#include <deque>
#include <functional>
#include <list>
#include <thread>
#include <unordered_set>
#include <vector>
#include <memory>
#include <mutex>
#include <unordered_map>

#include "common.h"
#include "packed_frames.h"

namespace cv {

// One resident block.  Shared ownership: the tier's table holds one reference, every open read context that serves from the block
// holds another, so an eviction (or a re-load of the same id) while a reader is packing frames from it only drops the table's
// reference -- the device memory goes away with the last reader.
struct HbmBuf {
    uint8_t* d_ptr = nullptr;
    int64_t len = 0;
    int device = 0;
    ~HbmBuf();
};
using HbmBlock = std::shared_ptr<const HbmBuf>;

// Admission / eviction (the tier sits beside Mem/Ssd/Hdd; the reference's tiers are capacity-bounded directories chosen by
// storage policy, worker/storage/policy.rs:56-105 -- here the policy is LRU over resident blocks):
//   capacity      bytes of HBM the tier may hold; 0 = unbounded (blocks stay until the worker stops)
//   load()        admits a block, evicting least-recently-read blocks nobody is reading until it fits; a block larger than the
//                 capacity, or one that does not fit because everything resident is being read, is refused (kind Common)
//   promote_after a block read remotely (framed) this many times from its file is loaded on the next remote Open and that very read
//                 is served from HBM; 0 = manual loads only
class HbmTier {
   public:
    void configure(int64_t capacity_bytes, int promote_after, int device);
    Err load(int64_t block_id, const void* host_bytes, int64_t len, int device);
    bool get(int64_t block_id, HbmBlock* out);  // LRU touch
    void evict(int64_t block_id);               // the block was rewritten or removed: its resident copy must not be served again
    // a remote read of a block that is not resident is about to be served from its file: true = promote it first
    bool should_promote(int64_t block_id);
    // Asynchronous promotion: the read that crossed the threshold is served from the store as usual while a promoter thread
    // reads the block (`fetch` fills a buffer with its bytes; it owns whatever keeps them alive) and loads it; the NEXT read
    // finds it resident.  At most one promotion per block is in flight; the queue is bounded (a full queue drops the request --
    // the block asks again on its next read).
    void promote_async(int64_t block_id, int64_t len, std::function<bool(std::vector<char>*)> fetch);
    void drain();  // test/measurement hook: wait until no promotion is queued or running
    ~HbmTier();
    int device() const { return device_; }
    size_t size() const;
    void stats(int64_t out[6]) const;  // resident blocks, resident bytes, capacity, evictions, promotions, refused loads
    void note_promotion() { promotions_++; }
    // K4 over [off, off+n) of a resident block: prefixes (code 81, status Running|Success, req_id, seq first_seq..) + payload
    Err pack(const HbmBlock& b, int64_t off, int64_t n, int64_t chunk, int64_t req_id, int32_t first_seq, PackedStream* out) const;

   private:
    mutable std::mutex mu_;
    std::list<int64_t> lru_;  // front = most recently read
    struct Entry {
        HbmBlock buf;
        std::list<int64_t>::iterator pos;
    };
    std::unordered_map<int64_t, Entry> blocks_;
    std::unordered_map<int64_t, int> remote_reads_;  // non-resident blocks: framed reads served from the file so far
    int64_t capacity_ = 0, bytes_ = 0;
    int promote_after_ = 0, device_ = 0;
    std::atomic<int64_t> evictions_{0}, promotions_{0}, refused_{0};
    struct Promo {
        int64_t id, len;
        std::function<bool(std::vector<char>*)> fetch;
    };
    void promoter_loop();
    std::mutex pmu_;
    std::condition_variable pcv_, pidle_;
    std::deque<Promo> pq_;
    std::unordered_set<int64_t> pending_;
    std::thread promoter_;
    bool pstop_ = false, pbusy_ = false;
};

}  // namespace cv
