#include "writer.h"

#include "../../../include/curvine_b200.h"
#include "../crc_gf.h"
#include "block_store.h"
#include "net.h"

namespace cv {

uint32_t host_crc_update(int poly, uint32_t crc, const uint8_t* buf, size_t len) {
    // CRC(A||B) = combine(CRC(A), CRC(B), |B|)
    const uint32_t c = cv_host_crc(poly, buf, len);
    return crc_combine(crc, c, len, poly_of(poly));
}

FsWriter::~FsWriter() {
    if (client_) ctx_->release(std::move(client_));
}

Err FsWriter::create(FsContext* ctx, const std::string& path, int64_t inode_id, int64_t block_size, int32_t storage_type, const WorkerAddress& worker,
                     int64_t chunk_size, std::unique_ptr<FsWriter>* out) {
    if (block_size <= 0 || chunk_size <= 0 || chunk_size > kMaxDataSize) return Err(kInvalidFileSize, "bad block or chunk size");
    std::unique_ptr<FsWriter> w(new FsWriter());
    w->ctx_ = ctx, w->worker_ = worker, w->block_size_ = block_size, w->chunk_size_ = chunk_size, w->storage_type_ = storage_type;
    w->fb_.status.id = inode_id, w->fb_.status.path = path, w->fb_.status.block_size = block_size;
    if (Err e = ctx->acquire_read(worker, &w->client_)) {
        ctx->add_failed_worker(worker);  // batch_block_writer.rs:143-175: a worker that cannot be written to is excluded for failed_worker_ttl
        return e;
    }
    *out = std::move(w);
    return Err::ok();
}

Err FsWriter::open_block() {
    LocatedBlock lb;
    CV_RETURN_IF_ERR(create_block_id(fb_.status.id, static_cast<int64_t>(fb_.block_locs.size()), &lb.block.id));
    lb.block.storage_type = storage_type_;
    lb.locs.push_back(worker_);
    req_id_ = new_req_id(), seq_ = 0, block_pos_ = 0, crc32_ = 0, crc32c_ = 0;
    BlockWriteRequest r;
    r.block.id = lb.block.id, r.block.block_size = 0, r.block.storage_type = storage_type_;
    r.off = 0, r.block_size = block_size_, r.chunk_size = static_cast<int32_t>(chunk_size_), r.client_name = "curvine-b200";
    Protocol resp;
    std::string rh, rd;
    CV_RETURN_IF_ERR(client_->rpc(request_proto(kCodeWriteBlock, kReqOpen, req_id_, 0), r.encode(), &resp, &rh, &rd));
    BlockWriteResponse wr;
    CV_RETURN_IF_ERR(BlockWriteResponse::decode(reinterpret_cast<const uint8_t*>(rh.data()), rh.size(), &wr));
    if (wr.block_size != block_size_)
        return Err::common(str_printf("Abnormal block size, expected length %lld, actual length %lld", (long long)block_size_, (long long)wr.block_size));
    lb.block.storage_type = wr.storage_type;
    fb_.block_locs.push_back(lb);
    block_open_ = true;
    return Err::ok();
}

Err FsWriter::commit_block(bool cancel) {
    if (!block_open_) return Err::ok();
    LocatedBlock& lb = fb_.block_locs.back();
    lb.block.len = block_pos_, lb.crc32 = crc32_, lb.crc32c = crc32c_, lb.has_crc = true;
    BlockWriteRequest r;  // write_commit: block.len = bytes written, off = pos (block_client.rs:190-219)
    r.block.id = lb.block.id, r.block.block_size = block_pos_, r.block.storage_type = storage_type_;
    r.off = block_pos_, r.block_size = block_size_, r.client_name = "curvine-b200";
    Protocol resp;
    std::string rh, rd;
    CV_RETURN_IF_ERR(client_->rpc(request_proto(kCodeWriteBlock, cancel ? kReqCancel : kReqComplete, req_id_, ++seq_), r.encode(), &resp, &rh, &rd));
    block_open_ = false;
    if (cancel) fb_.block_locs.pop_back();
    return Err::ok();
}

// one Running request carrying `n` payload bytes, then its (empty) success response
Err FsWriter::send_running(const uint8_t* payload, int64_t n) {
    const Protocol req = request_proto(kCodeWriteBlock, kReqRunning, req_id_, ++seq_);
    std::string prefix;
    BlockClient::append_frame(req, std::string(), &prefix, static_cast<int32_t>(n));
    Err e = send_all(client_->fd(), prefix.data(), prefix.size());
    if (!e) e = send_all(client_->fd(), payload, static_cast<size_t>(n));
    if (e) client_->broken = true;
    Protocol resp;
    std::string rh, rd;
    if (!e) e = client_->recv_answer(req, &resp, &rh, &rd);
    if (e && client_->broken) ctx_->add_failed_worker(worker_);  // a well-formed error answer leaves the worker off the list
    return e;
}

Err FsWriter::write(const uint8_t* buf, int64_t n) {
    if (done_) return Err::common("writer is closed");
    while (n > 0) {
        if (block_open_ && block_pos_ == block_size_) CV_RETURN_IF_ERR(commit_block(false));
        if (!block_open_) CV_RETURN_IF_ERR(open_block());
        const int64_t take = std::min(n, std::min(chunk_size_, block_size_ - block_pos_));
        CV_RETURN_IF_ERR(send_running(buf, take));
        crc32_ = host_crc_update(0, crc32_, buf, static_cast<size_t>(take));
        crc32c_ = host_crc_update(1, crc32c_, buf, static_cast<size_t>(take));
        buf += take, n -= take, block_pos_ += take, pos_ += take;
    }
    return Err::ok();
}

Err FsWriter::write_device(const void* d_src, int64_t n, void* stream) {
    if (done_) return Err::common("writer is closed");
    const uint8_t* src = static_cast<const uint8_t*>(d_src);
    while (n > 0) {
        if (block_open_ && block_pos_ == block_size_) CV_RETURN_IF_ERR(commit_block(false));
        if (!block_open_) CV_RETURN_IF_ERR(open_block());
        const int64_t take = std::min(n, block_size_ - block_pos_);  // the rest of this block in one K4 launch
        const uint32_t nf = static_cast<uint32_t>((take + chunk_size_ - 1) / chunk_size_);
        const size_t wire_bytes = static_cast<size_t>(take) + size_t(nf) * kProtocolSize;
        uint32_t crc32 = 0;
        CV_RETURN_IF_ERR(pack_running_frames(src, take, chunk_size_, kCodeWriteBlock, static_cast<uint8_t>(status_encode(kReqRunning, kRespUndefined)),
                                             req_id_, seq_ + 1, stream, &packed_, &crc32));
        // all Running frames of this range in one write, then their responses (the worker serves them in order)
        Err e = send_all(client_->fd(), packed_.wire, wire_bytes);
        Protocol resp;
        std::string rh, rd;
        for (uint32_t f = 0; f < nf && !e; f++)
            e = client_->recv_answer(request_proto(kCodeWriteBlock, kReqRunning, req_id_, seq_ + 1 + static_cast<int32_t>(f)), &resp, &rh, &rd);
        if (e) {
            client_->broken = true;
            return e;
        }
        seq_ += static_cast<int32_t>(nf);
        crc32c_ = crc_combine(crc32c_, packed_.crc32c, static_cast<uint64_t>(take), kPolyCastagnoli);
        crc32_ = crc_combine(crc32_, crc32, static_cast<uint64_t>(take), kPolyIeee);
        src += take, n -= take, block_pos_ += take, pos_ += take;
    }
    return Err::ok();
}

Err FsWriter::complete() {
    if (done_) return Err::ok();
    CV_RETURN_IF_ERR(commit_block(false));
    done_ = true;
    fb_.status.len = pos_;
    fb_.build_index();
    ctx_->ns.put(fb_);
    return Err::ok();
}

Err FsWriter::cancel() {
    if (done_) return Err::ok();
    done_ = true;
    return commit_block(true);
}

std::string FsWriter::manifest() const {
    Namespace ns;
    ns.put(fb_);
    return ns.dump();
}

}  // namespace cv
