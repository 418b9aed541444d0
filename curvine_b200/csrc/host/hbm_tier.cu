#include "hbm_tier.h"

#include <cuda_runtime.h>

#include <vector>

#include "wire.h"

namespace cv {

HbmBuf::~HbmBuf() {
    if (!d_ptr) return;
    cudaSetDevice(device);
    cudaFree(d_ptr);
}

void HbmTier::configure(int64_t capacity_bytes, int promote_after, int device) {
    std::lock_guard<std::mutex> lk(mu_);
    capacity_ = std::max<int64_t>(capacity_bytes, 0), promote_after_ = std::max(promote_after, 0), device_ = device;
}

Err HbmTier::load(int64_t block_id, const void* host_bytes, int64_t len, int device) {
    std::vector<HbmBlock> dropped;  // released outside the lock (cudaFree)
    {
        // make room first: never hold more than `capacity` bytes, not even transiently
        std::lock_guard<std::mutex> lk(mu_);
        auto old = blocks_.find(block_id);
        if (old != blocks_.end()) {  // re-load: the old copy leaves the table (readers of it keep it alive)
            bytes_ -= old->second.buf->len;
            dropped.push_back(old->second.buf);
            lru_.erase(old->second.pos);
            blocks_.erase(old);
        }
        if (capacity_ > 0) {
            if (len > capacity_) {
                refused_++;
                return Err::common(str_printf("block of %lld bytes exceeds the HBM tier capacity %lld", (long long)len, (long long)capacity_));
            }
            auto it = lru_.end();
            while (bytes_ + len > capacity_ && it != lru_.begin()) {
                --it;  // walk from the cold end, skipping blocks somebody is reading
                auto e = blocks_.find(*it);
                if (e->second.buf.use_count() > 1) continue;
                bytes_ -= e->second.buf->len;
                dropped.push_back(e->second.buf);
                blocks_.erase(e);
                it = lru_.erase(it);
                evictions_++;
            }
            if (bytes_ + len > capacity_) {
                refused_++;
                return Err::common("the HBM tier is full of blocks that are being read");
            }
        }
        bytes_ += len;  // reserved
    }
    dropped.clear();
    auto fail = [&](Err e) {
        std::lock_guard<std::mutex> lk(mu_);
        bytes_ -= len;
        return e;
    };
    if (cudaSetDevice(device) != cudaSuccess) return fail(Err::io("cudaSetDevice failed"));
    std::shared_ptr<HbmBuf> b(new HbmBuf());
    b->len = len, b->device = device;
    cudaError_t ce = cudaMalloc(&b->d_ptr, static_cast<size_t>(std::max<int64_t>(len, 1)));
    if (ce == cudaSuccess) ce = cudaMemcpy(b->d_ptr, host_bytes, static_cast<size_t>(len), cudaMemcpyHostToDevice);
    if (ce != cudaSuccess) return fail(Err::io(str_printf("HBM tier load: %s", cudaGetErrorString(ce))));
    std::lock_guard<std::mutex> lk(mu_);
    auto dup = blocks_.find(block_id);
    if (dup != blocks_.end()) {  // two loads of one id raced: the later one wins
        bytes_ -= dup->second.buf->len;
        lru_.erase(dup->second.pos);
        blocks_.erase(dup);
    }
    lru_.push_front(block_id);
    blocks_[block_id] = Entry{b, lru_.begin()};
    remote_reads_.erase(block_id);
    return Err::ok();
}

bool HbmTier::get(int64_t block_id, HbmBlock* out) {
    std::lock_guard<std::mutex> lk(mu_);
    auto it = blocks_.find(block_id);
    if (it == blocks_.end()) return false;
    lru_.splice(lru_.begin(), lru_, it->second.pos);
    *out = it->second.buf;
    return true;
}

void HbmTier::evict(int64_t block_id) {
    HbmBlock dropped;  // released outside the lock; a reader that still packs frames from it keeps it alive
    std::lock_guard<std::mutex> lk(mu_);
    remote_reads_.erase(block_id);
    auto it = blocks_.find(block_id);
    if (it == blocks_.end()) return;
    bytes_ -= it->second.buf->len;
    dropped = it->second.buf;
    lru_.erase(it->second.pos);
    blocks_.erase(it);
}

bool HbmTier::should_promote(int64_t block_id) {
    std::lock_guard<std::mutex> lk(mu_);
    if (promote_after_ <= 0) return false;
    int& n = remote_reads_[block_id];
    if (n >= promote_after_) return true;
    n++;
    return false;
}

HbmTier::~HbmTier() {
    {
        std::lock_guard<std::mutex> lk(pmu_);
        pstop_ = true;
        pq_.clear();
        pcv_.notify_all();
    }
    if (promoter_.joinable()) promoter_.join();
}

void HbmTier::promote_async(int64_t block_id, int64_t len, std::function<bool(std::vector<char>*)> fetch) {
    std::lock_guard<std::mutex> lk(pmu_);
    if (pstop_ || pq_.size() >= 64 || !pending_.insert(block_id).second) return;
    pq_.push_back(Promo{block_id, len, std::move(fetch)});
    if (!promoter_.joinable()) promoter_ = std::thread([this] { promoter_loop(); });
    pcv_.notify_one();
}

void HbmTier::promoter_loop() {
    for (;;) {
        Promo p;
        {
            std::unique_lock<std::mutex> lk(pmu_);
            pcv_.wait(lk, [&] { return pstop_ || !pq_.empty(); });
            if (pstop_) return;
            p = std::move(pq_.front());
            pq_.pop_front();
            pbusy_ = true;
        }
        std::vector<char> buf;
        if (p.fetch(&buf) && static_cast<int64_t>(buf.size()) == p.len && !load(p.id, buf.data(), p.len, device_)) promotions_++;
        std::lock_guard<std::mutex> lk(pmu_);
        pending_.erase(p.id);
        pbusy_ = false;
        if (pq_.empty()) pidle_.notify_all();
    }
}

void HbmTier::drain() {
    std::unique_lock<std::mutex> lk(pmu_);
    pidle_.wait(lk, [&] { return pstop_ || (pq_.empty() && !pbusy_); });
}

size_t HbmTier::size() const {
    std::lock_guard<std::mutex> lk(mu_);
    return blocks_.size();
}

void HbmTier::stats(int64_t out[6]) const {
    std::lock_guard<std::mutex> lk(mu_);
    out[0] = static_cast<int64_t>(blocks_.size()), out[1] = bytes_, out[2] = capacity_;
    out[3] = evictions_.load(), out[4] = promotions_.load(), out[5] = refused_.load();
}

Err HbmTier::pack(const HbmBlock& blk, int64_t off, int64_t n, int64_t chunk, int64_t req_id, int32_t first_seq, PackedStream* out) const {
    const HbmBuf& b = *blk;
    CU_TRY(cudaSetDevice(b.device));
    out->off0 = off, out->total = n, out->chunk = chunk, out->req_id = req_id, out->first_seq = first_seq;
    cudaStream_t st;
    CU_TRY(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
    Err e = pack_running_frames(b.d_ptr + off, n, chunk, kCodeReadBlock, static_cast<uint8_t>(status_encode(kReqRunning, kRespSuccess)), req_id,
                                first_seq, st, out);
    cudaStreamDestroy(st);
    return e;
}

}  // namespace cv
