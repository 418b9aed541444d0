#include "worker.h"

#include <errno.h>
#include <fcntl.h>
#include <poll.h>
#include <sys/eventfd.h>
#include <sys/socket.h>
#include <sys/stat.h>
#include <sys/vfs.h>
#include <unistd.h>

#include "net.h"

namespace cv {

static Protocol response_proto(const Protocol& req, int8_t resp_status) {
    Protocol p = req;
    p.resp_status = resp_status;
    p.header_len = p.data_len = 0;
    return p;
}

ReadHandler::~ReadHandler() { close_fd(fd_); }

Err ReadHandler::handle(const RpcRequest& req, RpcResponse* resp) {
    switch (req.proto.req_status) {
        case kReqOpen: return open(req, resp);
        case kReqRunning: return read(req, resp);
        case kReqComplete: return complete(req, resp);
        default: return Err::common("Unsupported request type");
    }
}

Err ReadHandler::open(const RpcRequest& req, RpcResponse* resp) {
    BlockReadRequest c;
    CV_RETURN_IF_ERR(BlockReadRequest::decode(reinterpret_cast<const uint8_t*>(req.header.data()), req.header.size(), &c));
    BlockMeta meta;
    CV_RETURN_IF_ERR(store_->get_block(c.id, &meta));
    if (c.off > meta.len)
        return Err::common(str_printf("The length of the requested data exceeds the maximum length of the block file, request off %lld, file len %lld",
                                      (long long)c.off, (long long)meta.len));
    if (c.chunk_size <= 0) return Err::common("chunk_size must be greater than 0");
    if (c.enable_read_ahead && c.read_ahead_len > 16 * 1024 * 1024)
        return Err::common(str_printf("The pre-read size exceeds the maximum value allowed by the system.The current value is %lld. The maximum allowed value is: %d",
                                      (long long)c.read_ahead_len, 16 * 1024 * 1024));
    const bool short_circuit = c.short_circuit && meta.storage_type != kStorageSpdkDisk;
    if (short_circuit && meta.in_arena() && !c.accept_arena)
        return Err(kUnsupported, str_printf("block %lld lives in the worker's mem arena: a short-circuit read needs an arena-aware client "
                                            "(BlockReadRequest.accept_arena); read it with short_circuit = false", (long long)c.id));
    close_fd(fd_);
    fd_ = -1;
    meta_ = meta;
    hbm_block_.reset();
    from_hbm_ = !short_circuit && hbm_ && hbm_->get(c.id, &hbm_block_);
    if (from_hbm_ && hbm_block_->len != meta.len) {  // the block changed under the resident copy: drop it, serve from the store
        hbm_->evict(c.id);
        hbm_block_.reset();
        from_hbm_ = false;
    }
    if (!from_hbm_ && !short_circuit && hbm_ && hbm_->should_promote(c.id)) {
        // read often enough from its file / extent: a promoter thread loads it into the HBM tier (evicting colder blocks) while THIS
        // read is served from the store as usual; the next remote read of the block is served from HBM.  A refusal (tier full of blocks
        // being read, block larger than the tier) just leaves the block where it is.
        const BlockMeta m = meta;  // an arena block's meta keeps its extent allocated until the promoter is done with it
        hbm_->promote_async(c.id, meta.len, [m](std::vector<char>* buf) {
            buf->resize(static_cast<size_t>(m.len));
            if (m.in_arena()) {
                memcpy(buf->data(), m.mem(), buf->size());
                return true;
            }
            const int pfd = ::open(m.path.c_str(), O_RDONLY | O_CLOEXEC);
            bool ok = pfd >= 0;
            for (size_t got = 0; ok && got < buf->size();) {
                const ssize_t r = pread(pfd, buf->data() + got, buf->size() - got, static_cast<off_t>(got));
                if (r < 0 && errno == EINTR) continue;
                if (r <= 0) ok = false;
                else got += static_cast<size_t>(r);
            }
            close_fd(pfd);
            return ok;
        });
    }
    if (from_hbm_) {
        // the block is resident in HBM: pack the whole response stream on the GPU now (K4), serve Running requests from it
        len_ = hbm_block_->len, pos_ = c.off, next_seq_ = req.proto.seq_id + 1;
        CV_RETURN_IF_ERR(hbm_->pack(hbm_block_, c.off, len_ - c.off, c.chunk_size, req.proto.req_id, next_seq_, &packed_));
        metrics_->read_blocks_hbm++;
        metrics_->hbm_packed_bytes += len_ - c.off;
    } else if (!short_circuit && meta.in_arena()) {
        len_ = meta.len, pos_ = c.off;  // served from the mapping; nothing to open
    } else if (!short_circuit) {
        fd_ = ::open(meta.path.c_str(), O_RDONLY | O_CLOEXEC);
        if (fd_ < 0) return Err::io(str_printf("open %s: %s", meta.path.c_str(), strerror(errno)));
        struct stat st;
        fstat(fd_, &st);
        len_ = st.st_size;
        pos_ = c.off;
        struct statfs sfs;
        is_tmpfs_ = fstatfs(fd_, &sfs) == 0 && sfs.f_type == 0x01021994;  // TMPFS_MAGIC (sys_libc.rs:320-339)
        last_ahead_ = -1;
    }
    path_ = meta.path;
    ctx_ = c;
    ctx_req_id_ = req.proto.req_id;
    has_ctx_ = true;
    if (!from_hbm_) (short_circuit ? metrics_->read_blocks_local : metrics_->read_blocks_remote)++;
    BlockReadResponse r;
    r.id = c.id, r.len = meta.len, r.has_path = short_circuit, r.path = meta.path, r.storage_type = meta.storage_type;
    if (short_circuit && meta.in_arena()) r.has_arena = true, r.arena_off = meta.hold->ext.off, r.arena_seg_len = meta.hold->arena->seg_bytes();
    resp->proto = response_proto(req.proto, kRespSuccess);
    resp->header = r.encode();
    return Err::ok();
}

// cache_manager.rs:99-147 / local_file.rs:202-213: fadvise(WILLNEED) ahead of a sequential cursor; never on tmpfs
void ReadHandler::read_ahead() {
    if (!ctx_.enable_read_ahead || is_tmpfs_ || len_ < 256 * 1024 || ctx_.read_ahead_len <= 0) return;
    if (last_ahead_ < 0 || pos_ >= last_ahead_ + ctx_.read_ahead_len / 2) {
        posix_fadvise(fd_, pos_, ctx_.read_ahead_len, POSIX_FADV_WILLNEED);
        last_ahead_ = pos_;
    }
}

Err ReadHandler::read(const RpcRequest& req, RpcResponse* resp) {
    if (from_hbm_ && has_ctx_) {
        if (!req.header.empty()) {  // seek: re-pack from the new offset
            DataHeaderProto h;
            CV_RETURN_IF_ERR(DataHeaderProto::decode(reinterpret_cast<const uint8_t*>(req.header.data()), req.header.size(), &h));
            if (h.offset != pos_) {
                if (h.offset < 0 || h.offset > len_) return Err::io("seek out of range");
                pos_ = h.offset;
                CV_RETURN_IF_ERR(hbm_->pack(hbm_block_, pos_, len_ - pos_, ctx_.chunk_size, ctx_req_id_, req.proto.seq_id, &packed_));
            }
        }
        const int64_t chunk = std::min<int64_t>(ctx_.chunk_size, len_ - pos_);
        if (chunk <= 0) return Err::common(str_printf("offset exceeds file length, length=%lld, offset=%lld", (long long)len_, (long long)pos_));
        const int64_t f = (pos_ - packed_.off0) / packed_.chunk;
        uint8_t* frame = packed_.wire + f * (kProtocolSize + packed_.chunk);
        // the prefix was packed with the expected echoes; patch them if this request carries different ones
        if (static_cast<int32_t>(get_be32(frame + 18)) != req.proto.seq_id) put_be32(frame + 18, static_cast<uint32_t>(req.proto.seq_id));
        if (static_cast<int64_t>(get_be64(frame + 10)) != req.proto.req_id) put_be64(frame + 10, static_cast<uint64_t>(req.proto.req_id));
        resp->proto = response_proto(req.proto, kRespSuccess);
        resp->raw = frame, resp->raw_len = static_cast<size_t>(kProtocolSize + chunk);
        pos_ += chunk;
        metrics_->read_bytes += chunk;
        metrics_->read_count++;
        return Err::ok();
    }
    const bool arena = has_ctx_ && meta_.in_arena() && !ctx_.short_circuit;
    if (fd_ < 0 && !arena) return Err::common("self.file is none");
    if (!has_ctx_) return Err::common("self.context is none");
    if (!req.header.empty()) {
        DataHeaderProto h;
        CV_RETURN_IF_ERR(DataHeaderProto::decode(reinterpret_cast<const uint8_t*>(req.header.data()), req.header.size(), &h));
        if (h.offset != pos_) {  // local files: the header offset is absolute inside the block file
            if (h.offset < 0) return Err::io("seek to negative offset");
            pos_ = h.offset;
        }
    }
    const double t0 = now_sec();
    if (!arena) read_ahead();
    const int64_t chunk = std::min<int64_t>(ctx_.chunk_size, len_ - pos_);
    if (chunk <= 0) return Err::common(str_printf("offset exceeds file length, length=%lld, offset=%lld", (long long)len_, (long long)pos_));
    resp->proto = response_proto(req.proto, kRespSuccess);
    if (arena && enable_send_file_) {  // sendfile(2) out of the segment file
        resp->file_fd = meta_.hold->arena->fd(meta_.hold->ext.seg), resp->file_off = meta_.hold->ext.off + pos_, resp->file_len = static_cast<int32_t>(chunk);
    } else if (arena) {  // enable_send_file = false: send(2) from the worker's mapping of the segment
        resp->mem = meta_.mem() + pos_, resp->mem_len = static_cast<int32_t>(chunk);
    } else if (enable_send_file_) {
        resp->file_fd = fd_, resp->file_off = pos_, resp->file_len = static_cast<int32_t>(chunk);
    } else {
        resp->data.resize(static_cast<size_t>(chunk));
        int64_t got = 0;
        while (got < chunk) {
            const ssize_t r = pread(fd_, &resp->data[got], static_cast<size_t>(chunk - got), pos_ + got);
            if (r < 0 && errno == EINTR) continue;
            if (r <= 0) return Err::io(str_printf("pread %s: %s", path_.c_str(), r == 0 ? "unexpected eof" : strerror(errno)));
            got += r;
        }
    }
    pos_ += chunk;
    metrics_->read_bytes += chunk;
    metrics_->read_time_us += static_cast<int64_t>((now_sec() - t0) * 1e6);
    metrics_->read_count++;
    return Err::ok();
}

Err ReadHandler::complete(const RpcRequest& req, RpcResponse* resp) {
    if (has_ctx_ && ctx_req_id_ != req.proto.req_id)
        return Err::common(str_printf("Request id mismatch, expected %lld, actual %lld", (long long)ctx_req_id_, (long long)req.proto.req_id));
    close_fd(fd_);
    fd_ = -1;
    hbm_block_.reset();  // the read context's reference on the resident block
    meta_ = BlockMeta();  // ... and on the arena extent
    resp->proto = response_proto(req.proto, kRespSuccess);
    return Err::ok();
}

// ------------------------------------------------------------------ WriteHandler

WriteHandler::~WriteHandler() { close_fd(fd_); }  // an open arena extent stays findable in the BlockStore (Complete / Cancel / re-Open)

Err WriteHandler::handle(const RpcRequest& req, RpcResponse* resp) {
    switch (req.proto.req_status) {
        case kReqOpen: return open(req, resp);
        case kReqRunning: return write(req, resp);
        case kReqComplete: return complete(req, resp, true);
        case kReqCancel: return complete(req, resp, false);
        default: return Err::common("Unsupported request type");
    }
}

Err WriteHandler::open(const RpcRequest& req, RpcResponse* resp) {
    BlockWriteRequest c;
    CV_RETURN_IF_ERR(BlockWriteRequest::decode(reinterpret_cast<const uint8_t*>(req.header.data()), req.header.size(), &c));
    if (c.off > c.block_size) return Err::common(str_printf("Invalid write offset: %lld, block size: %lld", (long long)c.off, (long long)c.block_size));
    CV_RETURN_IF_ERR(store_->open_block(c.block.id, c.block.storage_type, c.block_size, &target_));
    target_open_ = true;
    const bool short_circuit = c.short_circuit;
    if (short_circuit && target_.arena) {
        store_->abort_block(c.block.id, &target_), target_open_ = false;
        return Err(kUnsupported, "short-circuit writes into the mem arena are not supported: write through the worker (short_circuit = false)");
    }
    close_fd(fd_);
    fd_ = -1;
    if (!short_circuit && !target_.arena) {
        fd_ = ::open(target_.path.c_str(), O_WRONLY | O_CREAT | O_CLOEXEC, 0644);
        if (fd_ < 0) return Err::io(str_printf("open %s: %s", target_.path.c_str(), strerror(errno)));
    }
    pos_ = c.off;
    ctx_ = c, ctx_req_id_ = req.proto.req_id, has_ctx_ = true, is_commit_ = false;
    metrics_->write_blocks++;
    BlockWriteResponse r;
    r.id = c.block.id, r.has_path = short_circuit, r.path = target_.path, r.off = c.off, r.block_size = c.block_size, r.storage_type = target_.dir_storage_type;
    resp->proto = response_proto(req.proto, kRespSuccess);
    resp->header = r.encode();
    return Err::ok();
}

Err WriteHandler::write(const RpcRequest& req, RpcResponse* resp) {
    if (fd_ < 0 && !(target_open_ && target_.arena)) return Err::common("self.file is none");
    if (!has_ctx_) return Err::common("self.context is none");
    if (ctx_req_id_ != req.proto.req_id)
        return Err::common(str_printf("Request id mismatch, expected %lld, actual %lld", (long long)ctx_req_id_, (long long)req.proto.req_id));
    if (!req.header.empty()) {
        DataHeaderProto h;
        CV_RETURN_IF_ERR(DataHeaderProto::decode(reinterpret_cast<const uint8_t*>(req.header.data()), req.header.size(), &h));
        if (!h.flush) {  // a flush must not seek (write_handler.rs:168-186)
            if (h.offset < 0 || h.offset >= ctx_.block_size)
                return Err::common(str_printf("Invalid seek offset: %lld, block length: %lld", (long long)h.offset, (long long)ctx_.block_size));
            pos_ = h.offset;
        }
    }
    const int64_t n = static_cast<int64_t>(req.data.size());
    if (n > 0) {
        if (pos_ + n > ctx_.block_size)
            return Err::common(str_printf("Write range [%lld, %lld) exceeds block size %lld", (long long)pos_, (long long)(pos_ + n), (long long)ctx_.block_size));
        const double t0 = now_sec();
        if (target_.arena) {
            memcpy(target_.mem() + pos_, req.data.data(), static_cast<size_t>(n));
        } else {
            int64_t done = 0;
            while (done < n) {
                const ssize_t w = pwrite(fd_, req.data.data() + done, static_cast<size_t>(n - done), pos_ + done);
                if (w < 0 && errno == EINTR) continue;
                if (w <= 0) return Err::io(str_printf("write %s: %s", target_.path.c_str(), strerror(errno)));
                done += w;
            }
        }
        pos_ += n;
        metrics_->write_bytes += n;
        metrics_->write_time_us += static_cast<int64_t>((now_sec() - t0) * 1e6);
        metrics_->write_count++;
    }
    resp->proto = response_proto(req.proto, kRespSuccess);
    return Err::ok();
}

Err WriteHandler::complete(const RpcRequest& req, RpcResponse* resp, bool commit) {
    resp->proto = response_proto(req.proto, kRespSuccess);
    if (is_commit_) {
        if (!req.data.empty()) return Err::common("The block has been committed and data cannot be written anymore.");
        return Err::ok();
    }
    if (has_ctx_ && ctx_req_id_ != req.proto.req_id)
        return Err::common(str_printf("Request id mismatch, expected %lld, actual %lld", (long long)ctx_req_id_, (long long)req.proto.req_id));
    has_ctx_ = false;
    BlockWriteRequest c;
    CV_RETURN_IF_ERR(BlockWriteRequest::decode(reinterpret_cast<const uint8_t*>(req.header.data()), req.header.size(), &c));
    close_fd(fd_);
    fd_ = -1;
    if (c.block.block_size > c.block_size)
        return Err::common(str_printf("Invalid write offset: %lld, block size: %lld", (long long)c.block.block_size, (long long)c.block_size));
    if (!target_open_) {  // Complete/Cancel without a live Open on this connection (write_handler.rs:246-259 re-derives the path)
        CV_RETURN_IF_ERR(store_->open_block(c.block.id, c.block.storage_type, c.block_size, &target_));
        target_open_ = true;
    }
    if (commit) {  // finalize: the block's length is what the client committed
        int64_t len = c.block.block_size;
        if (!target_.arena) {
            if (truncate(target_.path.c_str(), len) != 0 && errno != ENOENT) return Err::io(str_printf("truncate %s: %s", target_.path.c_str(), strerror(errno)));
            struct stat st;
            if (stat(target_.path.c_str(), &st) != 0) return Err::io(str_printf("finalize %s: %s", target_.path.c_str(), strerror(errno)));
            len = st.st_size;
        }
        CV_RETURN_IF_ERR(store_->commit_block(c.block.id, &target_, len));
        if (hbm_) hbm_->evict(c.block.id);  // a resident copy of the previous bytes must not be served any more
    } else {  // abort
        store_->abort_block(c.block.id, &target_);
    }
    target_open_ = false;
    is_commit_ = true;
    return Err::ok();
}

Worker::~Worker() { stop(); }

Err Worker::start(const std::vector<std::string>& data_dirs, const std::string& cluster_id, const std::string& host, int port, bool enable_send_file,
                  const ArenaOpts& arena) {
    CV_RETURN_IF_ERR(store_.init(data_dirs, cluster_id, arena));
    enable_send_file_ = enable_send_file;
    wake_fd_ = eventfd(0, EFD_CLOEXEC);
    if (wake_fd_ < 0) return Err::io(str_printf("eventfd: %s", strerror(errno)));
    if (Err e = tcp_listen(host, port, &listen_fd_, &port_)) {
        close_fd(wake_fd_);
        wake_fd_ = -1;
        return e;
    }
    // non-blocking listeners: a connection reset between poll() and accept() must not leave accept() blocked where stop() cannot reach it
    fcntl(listen_fd_, F_SETFL, fcntl(listen_fd_, F_GETFL) | O_NONBLOCK);
    stopping_ = false;
    accept_thread_ = std::thread([this] { accept_loop(listen_fd_); });
    if (!unix_listen(local_socket_name(port_), &unix_fd_)) {
        fcntl(unix_fd_, F_SETFL, fcntl(unix_fd_, F_GETFL) | O_NONBLOCK);
        unix_accept_thread_ = std::thread([this] { accept_loop(unix_fd_); });
    } else {
        unix_fd_ = -1;  // no same-host transport (name taken): TCP serves everyone
    }
    return Err::ok();
}

void Worker::stop() {
    if (listen_fd_ < 0) return;
    stopping_ = true;
    // the eventfd wakes both accept loops' poll(); shutdown() of a listening socket alone does not wake a waiter on every kernel / sandbox
    const uint64_t one = 1;
    const ssize_t w = ::write(wake_fd_, &one, sizeof(one));  // fails only on a full counter, which is readable anyway
    (void)w;
    ::shutdown(listen_fd_, SHUT_RDWR);
    if (unix_fd_ >= 0) ::shutdown(unix_fd_, SHUT_RDWR);
    if (accept_thread_.joinable()) accept_thread_.join();
    if (unix_accept_thread_.joinable()) unix_accept_thread_.join();
    close_fd(listen_fd_);
    close_fd(unix_fd_);
    close_fd(wake_fd_);
    listen_fd_ = unix_fd_ = wake_fd_ = -1;
    {
        std::lock_guard<std::mutex> lk(conn_mu_);
        for (int fd : conn_fds_) ::shutdown(fd, SHUT_RDWR);
    }
    while (live_conns_.load() > 0) usleep(1000);
}

void Worker::accept_loop(int lfd) {
    while (!stopping_) {
        pollfd p[2] = {{lfd, POLLIN, 0}, {wake_fd_, POLLIN, 0}};
        if (::poll(p, 2, -1) < 0) {
            if (errno == EINTR) continue;
            break;
        }
        if (p[1].revents) break;  // stop()
        if (!(p[0].revents & POLLIN)) break;  // the listening socket failed
        const int fd = ::accept4(lfd, nullptr, nullptr, 0);  // blocking connection socket: accept4 does not pass O_NONBLOCK on
        if (fd < 0) {
            if (errno == EINTR || errno == EAGAIN || errno == EWOULDBLOCK || errno == ECONNABORTED) continue;  // reset or taken meanwhile
            break;
        }
        set_sock_opts(fd);
        {
            std::lock_guard<std::mutex> lk(conn_mu_);
            conn_fds_.push_back(fd);
        }
        live_conns_++;
        std::thread([this, fd] {
            serve(fd);
            {
                std::lock_guard<std::mutex> lk(conn_mu_);
                for (auto& f : conn_fds_)
                    if (f == fd) {
                        f = conn_fds_.back();
                        conn_fds_.pop_back();
                        break;
                    }
            }
            close_fd(fd);
            live_conns_--;
        }).detach();
    }
}

// StreamHandler::run + WorkerHandler::handle for one connection
void Worker::serve(int fd) {
    std::unique_ptr<ReadHandler> handler;
    std::unique_ptr<WriteHandler> whandler;
    uint8_t prefix[kProtocolSize];
    RpcRequest req;
    for (;;) {
        if (recv_exact(fd, prefix, kProtocolSize)) return;  // peer closed
        if (decode_protocol(prefix, &req.proto)) return;    // malformed frame ends the connection
        if (req.proto.header_len < 0) return;
        req.header.resize(static_cast<size_t>(req.proto.header_len));
        if (req.proto.header_len && recv_exact(fd, &req.header[0], req.header.size())) return;
        req.data.resize(static_cast<size_t>(req.proto.data_len));
        if (req.proto.data_len && recv_exact(fd, &req.data[0], req.data.size())) return;
        if (req.proto.is_heartbeat()) continue;

        RpcResponse resp;
        Err e;
        if (req.proto.code == kCodeWriteBlock) {
            handler.reset();  // handler_matches_code (worker_handler.rs:89-98): a different code replaces the live handler
            if (!whandler || req.proto.req_status != kReqRunning) whandler.reset(new WriteHandler(&store_, &metrics_, &hbm_));
            e = whandler->handle(req, &resp);
        } else if (req.proto.code != kCodeReadBlock) {
            e = Err::common(str_printf("Unsupported request type: %d", int(req.proto.code)));
        } else {
            whandler.reset();
            // worker_handler.rs:71-88: a fresh handler unless this is a Running message for the live one
            if (!handler || req.proto.req_status != kReqRunning) handler.reset(new ReadHandler(&store_, &metrics_, enable_send_file_, &hbm_));
            e = handler->handle(req, &resp);
        }
        if (e) {  // block_handler.rs:57-60 -> msg.error_ext(&e)
            resp = RpcResponse();
            resp.proto = response_proto(req.proto, kRespError);
            resp.data = encode_error_body(e.kind, e.msg);
        }
        if (!e && resp.raw) {  // a GPU-packed frame: prefix and payload already in wire order
            if (send_all(fd, resp.raw, resp.raw_len)) return;
            if (req.proto.req_status == kReqCancel || req.proto.req_status == kReqComplete) handler.reset(), whandler.reset();
            continue;
        }
        resp.proto.header_len = static_cast<int32_t>(resp.header.size());
        resp.proto.data_len = resp.mem ? resp.mem_len : resp.file_fd >= 0 ? resp.file_len : static_cast<int32_t>(resp.data.size());
        uint8_t out[kProtocolSize];
        encode_protocol(resp.proto, out);
        // prefix + header in one write, then the payload region (rpc_frame.rs:205-220)
        std::string head(reinterpret_cast<char*>(out), kProtocolSize);
        head += resp.header;
        if (resp.file_fd < 0 && !resp.mem) head += resp.data;
        if (resp.mem) {  // prefix and payload leave in one segment train (MSG_MORE), payload straight out of the arena mapping
            if (send_more(fd, head.data(), head.size()) || send_all(fd, resp.mem, static_cast<size_t>(resp.mem_len))) return;
            if (req.proto.req_status == kReqCancel || req.proto.req_status == kReqComplete) handler.reset(), whandler.reset();
            continue;
        }
        if (resp.file_fd >= 0 ? send_more(fd, head.data(), head.size()) : send_all(fd, head.data(), head.size())) return;
        if (resp.file_fd >= 0 && send_file_full(fd, resp.file_fd, resp.file_off, static_cast<size_t>(resp.file_len))) return;
        if (req.proto.req_status == kReqCancel || req.proto.req_status == kReqComplete) handler.reset(), whandler.reset();
    }
}

}  // namespace cv
